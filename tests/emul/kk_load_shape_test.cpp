// Host driver of the load-shape resolver (kk_plan.cpp: resolve_load_shape) — test infrastructure only.  No CUDA (no GPU needed).
// Reads one case per line from stdin, "mode fanout flags part_index part_count n_devices peer_ok", and prints one JSON line per case:
// the status and message the resolver throws, or the shape it resolves.
#include <cstdio>
#include <string>

#include "kk_json.hpp"
#include "kk_plan.hpp"

using namespace kk;

static const char* order_name(LoadOrder o) {
  switch (o) {
    case LoadOrder::kOwn: return "own";
    case LoadOrder::kReplicas: return "replicas";
    case LoadOrder::kPush: return "push";
    case LoadOrder::kNvls: return "nvls";
    case LoadOrder::kRaw: return "raw";
    case LoadOrder::kPull: return "pull";
  }
  return "?";
}

int main() {
  kk_load_opts o{};
  int n_devices, peer_ok;
  while (scanf("%d %d %u %d %d %d %d", &o.mode, &o.fanout, &o.flags, &o.part_index, &o.part_count, &n_devices, &peer_ok) == 7) {
    try {
      const LoadShape S = resolve_load_shape(o, n_devices, peer_ok != 0);
      std::string parts;
      for (int p : S.local_parts) parts += (parts.empty() ? "" : ",") + std::to_string(p);
      printf("{\"status\":0,\"order\":\"%s\",\"multi_proc\":%d,\"rank\":%d,\"n_parts\":%d,\"local_parts\":[%s],\"every_part\":%d,\"xdst\":%d,"
             "\"peer_ok\":%d,\"two_stage\":%d}\n",
             order_name(S.order), S.multi_proc, S.rank, S.n_parts, parts.c_str(), S.every_part, S.xdst, S.peer_ok, S.two_stage);
    } catch (const Error& e) {
      printf("{\"status\":%d,\"error\":\"%s\"}\n", e.code, json_escape(e.what()).c_str());
    }
  }
  return 0;
}
