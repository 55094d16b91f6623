// PEFT LoRA adapters: config and tensor parsing, matching against a load's plan, the describe JSON and the host read of A and B.
// The format is PEFT's saved form (save_pretrained): adapter_config.json plus adapter_model.safetensors with keys
// base_model.model.<M>.lora_A.weight [r, C] and base_model.model.<M>.lora_B.weight [R, r].
#include "kk_adapter.hpp"

#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <map>
#include <set>
#include <sstream>

#include "kk_json.hpp"
#include "kk_lora.cuh"
#include "kk_read.hpp"

namespace kk {

namespace {

bool is_dir(const std::string& p) {
  struct stat st;
  return stat(p.c_str(), &st) == 0 && S_ISDIR(st.st_mode);
}
bool is_file(const std::string& p) {
  struct stat st;
  return stat(p.c_str(), &st) == 0 && S_ISREG(st.st_mode);
}
bool ends_with(const std::string& s, const char* suf) {
  const size_t n = strlen(suf);
  return s.size() >= n && s.compare(s.size() - n, n, suf) == 0;
}
std::string absolute(const std::string& p) {
  char buf[PATH_MAX];
  return realpath(p.c_str(), buf) ? std::string(buf) : p;
}

std::string read_text(const std::string& path) {
  const int fd = ::open(path.c_str(), O_RDONLY | O_CLOEXEC);
  if (fd < 0) fail(errno == ENOENT ? KK_ENOENT : KK_EIO, "adapter: open %s: %s", path.c_str(), strerror(errno));
  std::string s;
  char buf[65536];
  for (;;) {
    const ssize_t n = ::read(fd, buf, sizeof buf);
    if (n < 0 && errno == EINTR) continue;
    if (n < 0) { const int e = errno; ::close(fd); fail(KK_EIO, "adapter: read %s: %s", path.c_str(), strerror(e)); }
    if (n == 0) break;
    s.append(buf, (size_t)n);
    if (s.size() > (64u << 20)) { ::close(fd); fail(KK_EFORMAT, "adapter: %s is larger than 64 MiB", path.c_str()); }
  }
  ::close(fd);
  return s;
}

// A boolean config key: absent = false.
bool config_bool(const JsonValue& cfg, const char* key) {
  const JsonValue* v = cfg.find(key);
  if (!v || v->kind == JsonValue::Null) return false;
  if (v->kind != JsonValue::Bool) fail(KK_EFORMAT, "adapter_config.json: \"%s\" is not a boolean", key);
  return v->b;
}

constexpr const char* kPrefix = "base_model.model.";

// A transpose (KK_LOAD_GPT2_CONV1D_T) writes the tensor at p in the pool of placement set `part`.  Checked on the ops, as a square
// Conv1D weight keeps its shape.
bool transposed(const Plan& P, int part, const Placement& p) {
  for (size_t q = 0; q < P.parts.size(); ++q) {
    if (P.placements.size() > 1 && (int)q != part) continue;
    for (const KKSeg& s : P.parts[q].segs)
      if (kk_is_transpose(s.op) && s.dst_off >= p.pool_offset && s.dst_off < p.pool_offset + p.nbytes) return true;
  }
  return false;
}

}  // namespace

void check_adapter_opts(const kk_load_opts& opts) {
  if (opts.fanout == KK_FANOUT_NVLS && opts.mode == KK_MODE_BROADCAST)
    fail(KK_EUNSUPPORTED, "adapter: KK_FANOUT_NVLS pools cannot be merged into (multicast pools are written through the switch only)");
  if (opts.part_count > 1 && opts.mode == KK_MODE_BROADCAST)
    fail(KK_EUNSUPPORTED, "adapter: a multi-process BROADCAST pool also receives the other ranks' stores, so no rank knows when to merge it");
  if (opts.part_count > 1 && opts.mode == KK_MODE_SCATTER && (opts.flags & KK_LOAD_SCATTER_EXCHANGE))
    fail(KK_EUNSUPPORTED, "adapter: with KK_LOAD_SCATTER_EXCHANGE a rank's pool also receives the other ranks' rows, so no rank knows when to merge it");
}

uint32_t lora_out_of(uint32_t dt) { return dt == KK_F16 ? KK_LORA_F16 : dt == KK_F32 ? KK_LORA_F32 : KK_LORA_BF16; }

Adapter match_adapter(const std::string& adapter_path, const std::string& ckpt_path, uint32_t flags, const Plan& P) {
  Adapter A;
  A.path = absolute(adapter_path);
  std::string dir;
  if (is_dir(A.path)) {
    dir = A.path;
    A.file = dir + "/adapter_model.safetensors";
    if (!is_file(A.file)) {
      if (is_file(dir + "/adapter_model.bin")) fail(KK_EUNSUPPORTED, "adapter: %s holds adapter_model.bin (a pickle); save the adapter as safetensors", dir.c_str());
      fail(KK_ENOENT, "adapter: %s has no adapter_model.safetensors", dir.c_str());
    }
  } else if (is_file(A.path)) {
    if (!ends_with(A.path, ".safetensors")) fail(KK_EUNSUPPORTED, "adapter: %s is not a safetensors file (adapter_model.bin is not read)", A.path.c_str());
    A.file = A.path;
    const size_t k = A.path.find_last_of('/');
    dir = k == std::string::npos ? "." : A.path.substr(0, k);
  } else {
    fail(KK_ENOENT, "adapter: %s does not exist", adapter_path.c_str());
  }

  // ---- config
  const std::string text = read_text(dir + "/adapter_config.json");
  JsonValue cfg;
  try {
    cfg = JsonParser(text.data(), text.size()).parse_document();
  } catch (const Error& e) {
    fail(KK_EFORMAT, "adapter_config.json: %s", e.what());
  }
  if (cfg.kind != JsonValue::Object) fail(KK_EFORMAT, "adapter_config.json is not a JSON object");
  const JsonValue* alpha = cfg.find("lora_alpha");
  if (!alpha || (alpha->kind != JsonValue::Int && alpha->kind != JsonValue::Double) || !std::isfinite(alpha->d))
    fail(KK_EFORMAT, "adapter_config.json: \"lora_alpha\" is missing or not a finite number");
  A.alpha = alpha->d;
  A.rslora = config_bool(cfg, "use_rslora");
  if (const JsonValue* ap = cfg.find("alpha_pattern")) {
    if (ap->kind != JsonValue::Null && ap->kind != JsonValue::Object) fail(KK_EFORMAT, "adapter_config.json: \"alpha_pattern\" is not an object");
    if (ap->kind == JsonValue::Object && !ap->obj.empty()) fail(KK_EUNSUPPORTED, "adapter: a non-empty alpha_pattern (per-module alpha) is not supported");
  }
  if (config_bool(cfg, "use_dora")) fail(KK_EUNSUPPORTED, "adapter: DoRA (use_dora) is not supported");
  if (config_bool(cfg, "fan_in_fan_out")) fail(KK_EUNSUPPORTED, "adapter: fan_in_fan_out (GPT-2 Conv1D targets) is not supported");
  if (const JsonValue* b = cfg.find("bias")) {
    if (b->kind != JsonValue::String) fail(KK_EFORMAT, "adapter_config.json: \"bias\" is not a string");
    if (b->s != "none") fail(KK_EUNSUPPORTED, "adapter: bias \"%s\" is not supported (only \"none\")", b->s.c_str());
  }

  // ---- tensors: every key is half of a pair, or a refusal
  std::vector<TensorRec> recs;
  index_safetensors_file(A.file, 0, recs, nullptr);
  struct Half { const TensorRec* a = nullptr; const TensorRec* b = nullptr; };
  std::map<std::string, Half> mods;
  for (const TensorRec& t : recs) {
    const std::string& n = t.name;
    if (n.find("lora_embedding_") != std::string::npos) fail(KK_EUNSUPPORTED, "adapter: embedding LoRA (%s) is not supported", n.c_str());
    if (n.find("lora_magnitude_vector") != std::string::npos) fail(KK_EUNSUPPORTED, "adapter: DoRA (%s) is not supported", n.c_str());
    if (n.find("modules_to_save") != std::string::npos) fail(KK_EUNSUPPORTED, "adapter: modules_to_save tensors (%s) are not supported", n.c_str());
    if (ends_with(n, ".bias")) fail(KK_EUNSUPPORTED, "adapter: bias tensors (%s) are not supported", n.c_str());
    const bool is_a = ends_with(n, ".lora_A.weight"), is_b = ends_with(n, ".lora_B.weight");
    if (n.compare(0, strlen(kPrefix), kPrefix) != 0 || (!is_a && !is_b)) fail(KK_EFORMAT, "adapter: tensor %s is not a PEFT LoRA key", n.c_str());
    if (t.dtype != KK_F32 && t.dtype != KK_BF16 && t.dtype != KK_F16)
      fail(KK_EUNSUPPORTED, "adapter: tensor %s is %s (F32, BF16 or F16 only)", n.c_str(), dtype_info(t.dtype)->name);
    const std::string mod = n.substr(strlen(kPrefix), n.size() - strlen(kPrefix) - strlen(".lora_A.weight"));
    (is_a ? mods[mod].a : mods[mod].b) = &t;
  }
  if (mods.empty()) fail(KK_EFORMAT, "adapter: %s holds no lora_A / lora_B tensors", A.file.c_str());

  // ---- match: the plan's index is the load's view (HF names under KK_LOAD_HF_LAYOUT) cut to its stage
  std::map<std::string, uint32_t> by_name;
  for (size_t i = 0; i < P.index.tensors.size(); ++i) by_name[P.index.tensors[i].name] = (uint32_t)i;
  std::set<std::string> whole;  // names of the whole checkpoint's view, asked only for a name the stage lacks
  bool whole_known = false;
  for (auto& kv : mods) {
    const std::string& mod = kv.first;
    if (!kv.second.a || !kv.second.b) fail(KK_EFORMAT, "adapter: %s has lora_%s but no lora_%s", mod.c_str(), kv.second.a ? "A" : "B", kv.second.a ? "B" : "A");
    const TensorRec& a = *kv.second.a;
    const TensorRec& b = *kv.second.b;
    const std::string target = mod + ".weight";
    auto it = by_name.find(target);
    if (it == by_name.end()) {
      if (P.index.layer_end && !whole_known) {
        for (auto& t : to_hf_layout(index_path(ckpt_path), flags).tensors) whole.insert(t.name);
        whole_known = true;
      }
      if (whole.count(target)) { A.skipped.push_back(target); continue; }
      fail(KK_ENOENT, "adapter: target %s is not a tensor of the checkpoint", target.c_str());
    }
    const TensorRec& w = P.index.tensors[it->second];
    if (w.shape.size() != 2) fail(KK_EUNSUPPORTED, "adapter: target %s has %zu dimensions (2 only)", target.c_str(), w.shape.size());
    for (size_t part = 0; part < P.placements.size(); ++part) {
      const Placement& p = P.placements[part][it->second];
      if (p.dtype != KK_BF16 && p.dtype != KK_F16 && p.dtype != KK_F32)
        fail(KK_EUNSUPPORTED, "adapter: target %s is %s in the pool (bf16, f16 or F32 only)", target.c_str(), dtype_info(p.dtype)->name);
      bool same = p.shape.size() == 2;
      for (size_t d = 0; same && d < 2; ++d) same = d == p.slice_dim || p.shape[d] == w.shape[d];
      if (!same || transposed(P, (int)part, p)) fail(KK_EUNSUPPORTED, "adapter: target %s is transposed in the pool (GPT-2 Conv1D)", target.c_str());
    }
    if (a.shape.size() != 2 || b.shape.size() != 2) fail(KK_EFORMAT, "adapter: lora_A / lora_B of %s are not 2-D", mod.c_str());
    const uint64_t r = a.shape[0];
    if (b.shape[1] != r) fail(KK_EFORMAT, "adapter: %s: lora_A is [%llu, %llu] and lora_B [%llu, %llu]", mod.c_str(), (unsigned long long)a.shape[0],
                              (unsigned long long)a.shape[1], (unsigned long long)b.shape[0], (unsigned long long)b.shape[1]);
    if (r < 1 || r > KK_LORA_MAX_R) fail(KK_EUNSUPPORTED, "adapter: %s has rank %llu (1..%u)", mod.c_str(), (unsigned long long)r, KK_LORA_MAX_R);
    if (b.shape[0] != w.shape[0] || a.shape[1] != w.shape[1])
      fail(KK_EFORMAT, "adapter: %s: B.A is [%llu, %llu], the target [%llu, %llu]", mod.c_str(), (unsigned long long)b.shape[0],
           (unsigned long long)a.shape[1], (unsigned long long)w.shape[0], (unsigned long long)w.shape[1]);
    if (w.shape[0] >= (1ull << 31) || w.shape[1] >= (1ull << 31)) fail(KK_EUNSUPPORTED, "adapter: target %s is too large", target.c_str());
    LoraPair pr;
    pr.module = mod;
    pr.tensor = it->second;
    pr.a = a;
    pr.b = b;
    pr.r = (uint32_t)r;
    pr.s = (float)(A.rslora ? A.alpha / std::sqrt((double)r) : A.alpha / (double)r);
    A.pairs.push_back(std::move(pr));
  }
  std::sort(A.pairs.begin(), A.pairs.end(), [](const LoraPair& x, const LoraPair& y) { return x.tensor < y.tensor; });
  return A;
}

std::string adapter_to_json(const Adapter& A, const Plan& P) {
  std::ostringstream o;
  char sbuf[32];
  snprintf(sbuf, sizeof sbuf, "%.17g", A.alpha);
  o << "{\"adapter\":\"" << json_escape(A.path) << "\",\"file\":\"" << json_escape(A.file) << "\",\"lora_alpha\":" << sbuf
    << ",\"use_rslora\":" << (A.rslora ? "true" : "false") << ",\"n_targets\":" << A.pairs.size() << ",\"targets\":[";
  for (size_t i = 0; i < A.pairs.size(); ++i) {
    const LoraPair& p = A.pairs[i];
    const TensorRec& w = P.index.tensors[p.tensor];
    snprintf(sbuf, sizeof sbuf, "%.9g", (double)p.s);
    o << (i ? "," : "") << "{\"name\":\"" << json_escape(w.name) << "\",\"dtype\":\"" << dtype_info(P.placements[0][p.tensor].dtype)->name
      << "\",\"shape\":[" << w.shape[0] << "," << w.shape[1] << "],\"r\":" << p.r << ",\"scaling\":" << sbuf << ",\"lora_A\":\""
      << json_escape(p.a.name) << "\",\"lora_A_dtype\":\"" << dtype_info(p.a.dtype)->name << "\",\"lora_B\":\"" << json_escape(p.b.name)
      << "\",\"lora_B_dtype\":\"" << dtype_info(p.b.dtype)->name << "\"}";
  }
  o << "],\"skipped\":[";
  for (size_t i = 0; i < A.skipped.size(); ++i) o << (i ? "," : "") << "\"" << json_escape(A.skipped[i]) << "\"";
  o << "]}";
  return o.str();
}

std::vector<float> read_adapter_f32(const Adapter& A, std::vector<uint64_t>& a_off, std::vector<uint64_t>& b_off) {
  uint64_t n = 0;
  a_off.clear();
  b_off.clear();
  for (const LoraPair& p : A.pairs) {
    a_off.push_back(n);
    n += p.a.n_elems();
    b_off.push_back(n);
    n += p.b.n_elems();
  }
  std::vector<float> out(n ? n : 1);
  const int fd = ::open(A.file.c_str(), O_RDONLY | O_CLOEXEC);
  if (fd < 0) fail(errno == ENOENT ? KK_ENOENT : KK_EIO, "adapter: open %s: %s", A.file.c_str(), strerror(errno));
  std::vector<uint8_t> raw;
  try {
    for (size_t i = 0; i < A.pairs.size(); ++i)
      for (const TensorRec* t : {&A.pairs[i].a, &A.pairs[i].b}) {
        raw.resize(t->nbytes);
        pread_full(fd, raw.data(), t->nbytes, t->file_offset, A.file);
        float* dst = out.data() + (t == &A.pairs[i].a ? a_off[i] : b_off[i]);
        const uint64_t ne = t->n_elems();
        if (t->dtype == KK_F32) {
          memcpy(dst, raw.data(), ne * 4);
        } else {
          for (uint64_t e = 0; e < ne; ++e) {
            uint16_t h;
            memcpy(&h, raw.data() + 2 * e, 2);
            dst[e] = t->dtype == KK_F16 ? kk_lora_f16_f32(h) : kk_lora_bf16_f32(h);
          }
        }
      }
  } catch (...) {
    ::close(fd);
    throw;
  }
  ::close(fd);
  return out;
}

}  // namespace kk
