// Mutation fuzzer for the checkpoint parsers and the planner (host code only), built with ASan + UBSan:
//   make -C tools/fuzz && tools/fuzz/_build/fuzz_index tests/golden 20000
// Every mutated file must either index + plan cleanly or be rejected with a kk::Error — never crash, hang or trip a sanitizer.
#include <dirent.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <random>
#include <string>
#include <vector>

#include "../../kukeon_b200/csrc/kk_index.hpp"
#include "../../kukeon_b200/csrc/kk_plan.hpp"

namespace kk {
static thread_local std::string g_err;
void set_last_error(const std::string& s) { g_err = s; }
const char* get_last_error() { return g_err.c_str(); }
}  // namespace kk

static std::vector<uint8_t> slurp(const std::string& p) {
  std::ifstream f(p, std::ios::binary);
  return std::vector<uint8_t>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}

int main(int argc, char** argv) {
  if (argc < 3) { fprintf(stderr, "usage: %s <seed-dir> <iterations> [rng-seed]\n", argv[0]); return 2; }
  const std::string dir = argv[1];
  const long iters = atol(argv[2]);
  std::mt19937_64 rng(argc > 3 ? strtoull(argv[3], nullptr, 10) : 12345);
  std::vector<std::pair<std::string, std::vector<uint8_t>>> seeds;
  DIR* d = opendir(dir.c_str());
  if (!d) { perror("opendir"); return 2; }
  while (dirent* e = readdir(d)) {
    std::string n = e->d_name;
    auto ends_with = [&](const char* suf) { const size_t k = strlen(suf); return n.size() > k && n.compare(n.size() - k, k, suf) == 0; };
    struct stat st;
    if ((ends_with(".gguf") || ends_with(".safetensors")) && stat((dir + "/" + n).c_str(), &st) == 0 && S_ISREG(st.st_mode))
      seeds.emplace_back(n, slurp(dir + "/" + n));
  }
  closedir(d);
  if (seeds.empty()) { fprintf(stderr, "no seed files\n"); return 2; }
  char tmpl[] = "/tmp/kkfuzzXXXXXX";
  const std::string work = mkdtemp(tmpl);
  long ok = 0, rejected = 0;
  for (long it = 0; it < iters; ++it) {
    auto& seed = seeds[rng() % seeds.size()];
    std::vector<uint8_t> b = seed.second;
    const int nmut = 1 + (int)(rng() % 4);
    for (int k = 0; k < nmut && !b.empty(); ++k) {
      // bias mutations towards the header (first 1 KiB), where the structure lives
      size_t pos = (rng() % 4) ? rng() % std::min<size_t>(b.size(), 1024) : rng() % b.size();
      switch (rng() % 6) {
        case 0: b[pos] ^= (uint8_t)(1u << (rng() % 8)); break;
        case 1: b[pos] = (uint8_t)rng(); break;
        case 2: b.resize(pos); break;                                   // truncate
        case 3: b.insert(b.begin() + pos, (size_t)(rng() % 9), (uint8_t)rng()); break;
        case 4: if (pos + 8 <= b.size()) { uint64_t v = rng() % 3 ? (rng() % 100000) : rng(); memcpy(&b[pos], &v, 8); } break;
        case 5: if (b.size() > 16) b.erase(b.begin() + pos, b.begin() + std::min(b.size(), pos + 1 + (size_t)(rng() % 16))); break;
      }
    }
    const bool gguf = seed.first.rfind(".gguf") == seed.first.size() - 5;
    const std::string path = work + (gguf ? "/m.gguf" : "/m.safetensors");
    { std::ofstream f(path, std::ios::binary | std::ios::trunc); f.write((const char*)b.data(), (std::streamsize)b.size()); }
    try {
      kk::Index ix = kk::index_path(path);
      for (int mode = 0; mode < 3; ++mode) {
        const int parts = mode == 0 ? 1 : 1 + (int)(rng() % 8);
        try {
          kk::Plan P = kk::build_plan(ix, mode, (uint32_t)(rng() % 16) & ~4u, parts, (1ull << 20) * (1 + rng() % 4));
          (void)kk::plan_to_json(P);
        } catch (const kk::Error&) {}
        // the HF view reads the GGUF metadata keys and the tensor names and shapes the mutations reach
        try {
          kk::Plan P = kk::build_plan(kk::to_hf_layout(ix, KK_LOAD_HF_LAYOUT), mode, KK_LOAD_HF_LAYOUT | ((uint32_t)(rng() % 16) & ~4u), parts,
                                      (1ull << 20) * (1 + rng() % 4));
          (void)kk::plan_to_json(P);
        } catch (const kk::Error&) {}
      }
      ++ok;
    } catch (const kk::Error&) {
      ++rejected;
    }
    unlink(path.c_str());
  }
  rmdir(work.c_str());
  printf("iterations %ld: %ld indexed+planned, %ld rejected, 0 crashes\n", iters, ok, rejected);
  return 0;
}
