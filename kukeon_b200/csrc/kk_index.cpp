// Checkpoint indexing: safetensors + GGUF header parsing (host only, no CUDA).
//
// Format rules implemented here were probed against the format owners' libraries installed in the
// image (safetensors 0.7.0, gguf 0.19.0) — SURVEY.md §8(c), Appendix C.3/C.4 — because the reference
// has no loader to follow.  The validation set is the one safetensors' reader enforces:
// contiguous, sorted, hole-free data_offsets that cover the data section exactly; size == shape x dtype.
#include "kk_index.hpp"

#include <dirent.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <climits>
#include <cstdlib>
#include <cstring>
#include <map>
#include <set>

#include "kk_json.hpp"

namespace kk {

// ---------------------------------------------------------------------------------------------
// dtype table
// ---------------------------------------------------------------------------------------------
namespace {
struct DtRow { uint32_t dt; DtypeInfo info; uint32_t bits; };
// bits: storage bits per element for plain types (sub-byte types sized in bits like safetensors does).
const DtRow kDt[] = {
    {KK_BOOL, {"BOOL", 1, 1, false}, 8},       {KK_F4, {"F4", 2, 1, false}, 4},
    {KK_F6_E2M3, {"F6_E2M3", 4, 3, false}, 6}, {KK_F6_E3M2, {"F6_E3M2", 4, 3, false}, 6},
    {KK_U8, {"U8", 1, 1, false}, 8},           {KK_I8, {"I8", 1, 1, false}, 8},
    {KK_F8_E5M2, {"F8_E5M2", 1, 1, false}, 8}, {KK_F8_E4M3, {"F8_E4M3", 1, 1, false}, 8},
    {KK_F8_E8M0, {"F8_E8M0", 1, 1, false}, 8}, {KK_I16, {"I16", 1, 2, false}, 16},
    {KK_U16, {"U16", 1, 2, false}, 16},        {KK_F16, {"F16", 1, 2, true}, 16},
    {KK_BF16, {"BF16", 1, 2, true}, 16},       {KK_I32, {"I32", 1, 4, false}, 32},
    {KK_U32, {"U32", 1, 4, false}, 32},        {KK_F32, {"F32", 1, 4, true}, 32},
    {KK_C64, {"C64", 1, 8, false}, 64},        {KK_F64, {"F64", 1, 8, false}, 64},
    {KK_I64, {"I64", 1, 8, false}, 64},        {KK_U64, {"U64", 1, 8, false}, 64},
    {KK_Q4_0, {"Q4_0", 32, 18, true}, 0},      {KK_Q4_1, {"Q4_1", 32, 20, true}, 0},
    {KK_Q5_0, {"Q5_0", 32, 22, true}, 0},      {KK_Q5_1, {"Q5_1", 32, 24, true}, 0},
    {KK_Q8_0, {"Q8_0", 32, 34, true}, 0},      {KK_Q2_K, {"Q2_K", 256, 84, true}, 0},
    {KK_Q3_K, {"Q3_K", 256, 110, true}, 0},    {KK_Q4_K, {"Q4_K", 256, 144, true}, 0},
    {KK_Q5_K, {"Q5_K", 256, 176, true}, 0},    {KK_Q6_K, {"Q6_K", 256, 210, true}, 0},
    {KK_Q8_K, {"Q8_K", 256, 292, true}, 0},    {KK_IQ4_NL, {"IQ4_NL", 32, 18, true}, 0},
    {KK_IQ4_XS, {"IQ4_XS", 256, 136, true}, 0}, {KK_MXFP4, {"MXFP4", 32, 17, true}, 0},
    {KK_IQ2_XXS, {"IQ2_XXS", 256, 66, true}, 0}, {KK_IQ2_XS, {"IQ2_XS", 256, 74, true}, 0},
    {KK_IQ2_S, {"IQ2_S", 256, 82, true}, 0}, {KK_IQ3_XXS, {"IQ3_XXS", 256, 98, true}, 0},
    {KK_IQ3_S, {"IQ3_S", 256, 110, true}, 0}, {KK_IQ1_S, {"IQ1_S", 256, 50, true}, 0},
    {KK_IQ1_M, {"IQ1_M", 256, 56, true}, 0}, {KK_TQ1_0, {"TQ1_0", 256, 54, true}, 0},
    {KK_TQ2_0, {"TQ2_0", 256, 66, true}, 0}, {KK_NVFP4, {"NVFP4", 64, 36, true}, 0},
};
const DtRow* dt_row(uint32_t dt) {
  for (auto& r : kDt)
    if (r.dt == dt) return &r;
  return nullptr;
}
}  // namespace

const DtypeInfo* dtype_info(uint32_t dt) {
  const DtRow* r = dt_row(dt);
  return r ? &r->info : nullptr;
}

int dtype_from_safetensors(const std::string& s) {
  for (auto& r : kDt)
    if (r.dt < 32 && s == r.info.name) return (int)r.dt;
  return -1;
}

int dtype_from_ggml(uint32_t t) {
  switch (t) {  // ggml_type ids, gguf-py constants.py GGMLQuantizationType
    case 0: return KK_F32;   case 1: return KK_F16;   case 2: return KK_Q4_0;  case 3: return KK_Q4_1;
    case 6: return KK_Q5_0;  case 7: return KK_Q5_1;  case 8: return KK_Q8_0;  case 10: return KK_Q2_K;
    case 11: return KK_Q3_K; case 12: return KK_Q4_K; case 13: return KK_Q5_K; case 14: return KK_Q6_K;
    case 20: return KK_IQ4_NL; case 23: return KK_IQ4_XS; case 39: return KK_MXFP4;
    case 16: return KK_IQ2_XXS; case 17: return KK_IQ2_XS; case 22: return KK_IQ2_S; case 18: return KK_IQ3_XXS; case 21: return KK_IQ3_S;
    case 19: return KK_IQ1_S; case 29: return KK_IQ1_M; case 34: return KK_TQ1_0; case 35: return KK_TQ2_0; case 40: return KK_NVFP4;
    case 15: return KK_Q8_K; case 24: return KK_I8;   case 25: return KK_I16;  case 26: return KK_I32;
    case 27: return KK_I64;  case 28: return KK_F64;  case 30: return KK_BF16;
    default: return -1;
  }
}

// ---------------------------------------------------------------------------------------------
// small file helpers
// ---------------------------------------------------------------------------------------------
namespace {

struct MappedFile {
  const uint8_t* p = nullptr;
  uint64_t n = 0;
  int fd = -1;
  explicit MappedFile(const std::string& path) {
    fd = ::open(path.c_str(), O_RDONLY | O_CLOEXEC);
    if (fd < 0) fail(errno == ENOENT ? KK_ENOENT : KK_EIO, "open %s: %s", path.c_str(), strerror(errno));
    struct stat st;
    if (fstat(fd, &st) != 0) { int e = errno; ::close(fd); fail(KK_EIO, "stat %s: %s", path.c_str(), strerror(e)); }
    if (!S_ISREG(st.st_mode)) { ::close(fd); fail(KK_EFORMAT, "%s: not a regular file", path.c_str()); }
    n = (uint64_t)st.st_size;
    if (n) {
      void* m = mmap(nullptr, n, PROT_READ, MAP_PRIVATE, fd, 0);
      if (m == MAP_FAILED) { int e = errno; ::close(fd); fail(KK_EIO, "mmap %s: %s", path.c_str(), strerror(e)); }
      p = (const uint8_t*)m;
    }
  }
  ~MappedFile() {
    if (p) munmap((void*)p, n);
    if (fd >= 0) ::close(fd);
  }
  MappedFile(const MappedFile&) = delete;
  MappedFile& operator=(const MappedFile&) = delete;
};

bool is_dir(const std::string& p) {
  struct stat st;
  return stat(p.c_str(), &st) == 0 && S_ISDIR(st.st_mode);
}
bool is_file(const std::string& p) {
  struct stat st;
  return stat(p.c_str(), &st) == 0 && S_ISREG(st.st_mode);
}
bool ends_with(const std::string& s, const char* suf) {
  size_t n = strlen(suf);
  return s.size() >= n && memcmp(s.data() + s.size() - n, suf, n) == 0;
}
std::string abspath(const std::string& p) {
  char buf[PATH_MAX];
  if (realpath(p.c_str(), buf)) return buf;
  return p;
}
std::string dirname_of(const std::string& p) {
  size_t k = p.find_last_of('/');
  if (k == std::string::npos) return ".";
  if (k == 0) return "/";
  return p.substr(0, k);
}
std::vector<std::string> list_dir(const std::string& d, const char* suffix) {
  std::vector<std::string> out;
  DIR* dir = opendir(d.c_str());
  if (!dir) fail(KK_ENOENT, "opendir %s: %s", d.c_str(), strerror(errno));
  while (struct dirent* e = readdir(dir)) {
    std::string n = e->d_name;
    if (ends_with(n, suffix) && is_file(d + "/" + n)) out.push_back(n);
  }
  closedir(dir);
  std::sort(out.begin(), out.end());
  return out;
}

bool mul_overflow(uint64_t a, uint64_t b, uint64_t* r) { return __builtin_mul_overflow(a, b, r); }

}  // namespace

// ---------------------------------------------------------------------------------------------
// safetensors
// ---------------------------------------------------------------------------------------------
void index_safetensors_file(const std::string& file, uint32_t shard, std::vector<TensorRec>& out,
                            uint64_t* file_bytes) {
  MappedFile mf(file);
  if (file_bytes) *file_bytes = mf.n;
  if (mf.n < 8) fail(KK_EFORMAT, "%s: header too small", file.c_str());
  uint64_t hn;
  memcpy(&hn, mf.p, 8);  // little-endian host assumed (x86-64)
  if (hn > 100000000ull) fail(KK_EFORMAT, "%s: header too large", file.c_str());
  if (hn > mf.n - 8) fail(KK_EFORMAT, "%s: invalid header length", file.c_str());
  const char* hp = (const char*)mf.p + 8;
  if (hn == 0 || hp[0] != '{') fail(KK_EFORMAT, "%s: invalid header start", file.c_str());
  JsonValue doc;
  try {
    doc = JsonParser(hp, (size_t)hn).parse_document();
  } catch (Error& e) {
    fail(KK_EFORMAT, "%s: invalid header deserialization: %s", file.c_str(), e.what());
  }
  if (doc.kind != JsonValue::Object) fail(KK_EFORMAT, "%s: header is not a JSON object", file.c_str());

  struct Ent { std::string name; uint32_t dt; std::vector<uint64_t> shape; uint64_t b, e; };
  std::vector<Ent> ents;
  std::set<std::string> seen;
  for (auto& kv : doc.obj) {
    if (kv.first == "__metadata__") {
      if (kv.second.kind != JsonValue::Object) fail(KK_EFORMAT, "%s: __metadata__ is not an object", file.c_str());
      for (auto& m : kv.second.obj)
        if (m.second.kind != JsonValue::String)
          fail(KK_EFORMAT, "%s: __metadata__ value for \"%s\" is not a string", file.c_str(), m.first.c_str());
      continue;
    }
    const JsonValue& t = kv.second;
    if (t.kind != JsonValue::Object) fail(KK_EFORMAT, "%s: tensor entry \"%s\" is not an object", file.c_str(), kv.first.c_str());
    if (!seen.insert(kv.first).second) fail(KK_EFORMAT, "%s: duplicate tensor \"%s\"", file.c_str(), kv.first.c_str());
    const JsonValue* jd = t.find("dtype");
    const JsonValue* js = t.find("shape");
    const JsonValue* jo = t.find("data_offsets");
    if (!jd || jd->kind != JsonValue::String) fail(KK_EFORMAT, "%s: tensor \"%s\": missing dtype", file.c_str(), kv.first.c_str());
    if (!js || js->kind != JsonValue::Array) fail(KK_EFORMAT, "%s: tensor \"%s\": missing shape", file.c_str(), kv.first.c_str());
    if (!jo || jo->kind != JsonValue::Array || jo->arr.size() != 2 || !jo->arr[0].is_uint() || !jo->arr[1].is_uint())
      fail(KK_EFORMAT, "%s: tensor \"%s\": bad data_offsets", file.c_str(), kv.first.c_str());
    int dt = dtype_from_safetensors(jd->s);
    if (dt < 0) fail(KK_EFORMAT, "%s: tensor \"%s\": unknown variant `%s` for dtype", file.c_str(), kv.first.c_str(), jd->s.c_str());
    Ent e;
    e.name = kv.first;
    e.dt = (uint32_t)dt;
    for (auto& d : js->arr) {
      if (!d.is_uint()) fail(KK_EFORMAT, "%s: tensor \"%s\": bad shape entry", file.c_str(), kv.first.c_str());
      e.shape.push_back(d.u);
    }
    e.b = jo->arr[0].u;
    e.e = jo->arr[1].u;
    ents.push_back(std::move(e));
  }
  // safetensors sorts by data_offsets and then demands a gap-free cover of the data section.
  std::stable_sort(ents.begin(), ents.end(), [](const Ent& a, const Ent& b) {
    if (a.b != b.b) return a.b < b.b;
    return a.e < b.e;
  });
  const uint64_t data_start = 8 + hn;
  uint64_t cur = 0;
  for (auto& e : ents) {
    if (e.b != cur || e.e < e.b) fail(KK_EFORMAT, "%s: invalid offset for tensor `%s`", file.c_str(), e.name.c_str());
    cur = e.e;
    uint64_t nel = 1;
    for (auto d : e.shape)
      if (mul_overflow(nel, d, &nel)) fail(KK_EFORMAT, "%s: tensor `%s`: shape overflows", file.c_str(), e.name.c_str());
    const DtRow* r = dt_row(e.dt);
    uint64_t nbits;
    if (mul_overflow(nel, (uint64_t)r->bits, &nbits)) fail(KK_EFORMAT, "%s: tensor `%s`: size overflows", file.c_str(), e.name.c_str());
    if (nbits % 8 != 0) fail(KK_EFORMAT, "%s: tensor `%s`: misaligned slice (sub-byte dtype)", file.c_str(), e.name.c_str());
    if (nbits / 8 != e.e - e.b)
      fail(KK_EFORMAT, "%s: invalid shape, data type, or offset for tensor `%s`", file.c_str(), e.name.c_str());
    if (e.name.size() >= KK_NAME_MAX) fail(KK_EUNSUPPORTED, "%s: tensor name longer than %d bytes", file.c_str(), KK_NAME_MAX - 1);
    if (e.shape.size() > KK_MAX_DIMS) fail(KK_EUNSUPPORTED, "%s: tensor `%s` has %zu dims (max %d)", file.c_str(), e.name.c_str(), e.shape.size(), KK_MAX_DIMS);
  }
  if (data_start + cur != mf.n) fail(KK_EFORMAT, "%s: incomplete metadata, file not fully covered", file.c_str());
  for (auto& e : ents) {
    TensorRec t;
    t.name = std::move(e.name);
    t.dtype = e.dt;
    t.shape = std::move(e.shape);
    t.shard = shard;
    t.file_offset = data_start + e.b;
    t.nbytes = e.e - e.b;
    out.push_back(std::move(t));
  }
}

// ---------------------------------------------------------------------------------------------
// GGUF
// ---------------------------------------------------------------------------------------------
namespace {
struct Cursor {
  const uint8_t* p;
  uint64_t n;
  uint64_t off = 0;
  const std::string& file;
  void need(uint64_t k) const {
    if (k > n - off) fail(KK_EFORMAT, "%s: truncated GGUF header at byte %llu", file.c_str(), (unsigned long long)off);
  }
  template <class T>
  T get() {
    need(sizeof(T));
    T v;
    memcpy(&v, p + off, sizeof(T));
    off += sizeof(T);
    return v;
  }
  std::string str() {
    uint64_t len = get<uint64_t>();
    if (len > (1ull << 30)) fail(KK_EFORMAT, "%s: GGUF string too long", file.c_str());
    need(len);
    std::string s((const char*)p + off, (size_t)len);
    off += len;
    return s;
  }
  void skip(uint64_t k) { need(k); off += k; }
};

uint64_t gguf_scalar_size(uint32_t vt) {
  switch (vt) {
    case 0: case 1: case 7: return 1;
    case 2: case 3: return 2;
    case 4: case 5: case 6: return 4;
    case 10: case 11: case 12: return 8;
    default: return 0;
  }
}

void gguf_skip_value(Cursor& c, uint32_t vt, int depth) {
  if (depth > 4) fail(KK_EFORMAT, "%s: GGUF array nesting too deep", c.file.c_str());
  if (vt == 8) { c.str(); return; }
  if (vt == 9) {
    uint32_t et = c.get<uint32_t>();
    uint64_t cnt = c.get<uint64_t>();
    uint64_t sz = gguf_scalar_size(et);
    if (sz) {
      uint64_t tot;
      if (mul_overflow(sz, cnt, &tot)) fail(KK_EFORMAT, "%s: GGUF array too large", c.file.c_str());
      c.skip(tot);
    } else if (et == 8 || et == 9) {
      for (uint64_t i = 0; i < cnt; ++i) gguf_skip_value(c, et, depth + 1);
    } else fail(KK_EFORMAT, "%s: GGUF unknown array element type %u", c.file.c_str(), et);
    return;
  }
  uint64_t sz = gguf_scalar_size(vt);
  if (!sz) fail(KK_EFORMAT, "%s: GGUF unknown value type %u", c.file.c_str(), vt);
  c.skip(sz);
}

// Reads the value of metadata key `key` (type vt) into a GgufKey: a string, or an integer of any GGUF integer type in 1..65535.  A value
// of another type is recorded as unusable, not refused: only a load that needs it fails.  A malformed value is refused like any other.
GgufKey gguf_read_key(Cursor& c, const std::string& key, uint32_t vt, bool string) {
  GgufKey k;
  k.seen = true;
  char why[160];
  if (string && vt == 8) {
    k.s = c.str();
    return k;
  }
  if (!string && vt <= 11 && vt != 6 && vt != 7 && vt != 8 && vt != 9) {
    const bool sgn = vt == 1 || vt == 3 || vt == 5 || vt == 11;
    const uint64_t sz = gguf_scalar_size(vt);
    c.need(sz);
    uint64_t raw = 0;
    memcpy(&raw, c.p + c.off, (size_t)sz);  // little-endian
    c.off += sz;
    int64_t v = (int64_t)raw;
    if (sgn && sz < 8 && (raw >> (sz * 8 - 1)) & 1) v = (int64_t)(raw | (~0ull << (sz * 8)));  // sign-extend
    if ((sgn && v < 1) || (!sgn && raw < 1) || (sgn ? (uint64_t)v : raw) > 65535) {
      snprintf(why, sizeof why, "%s = %lld is out of range 1..65535", key.c_str(), sgn ? (long long)v : (long long)std::min<uint64_t>(raw, INT64_MAX));
      k.err = KK_EFORMAT;
      k.why = why;
    } else {
      k.u = sgn ? (uint64_t)v : raw;
    }
    return k;
  }
  gguf_skip_value(c, vt, 0);
  if (!string && vt == 9) {
    snprintf(why, sizeof why, "%s is a per-layer array, which is not supported", key.c_str());
    k.err = KK_EUNSUPPORTED;
  } else {
    snprintf(why, sizeof why, "%s has GGUF value type %u, not %s", key.c_str(), vt, string ? "a string" : "an integer");
    k.err = KK_EFORMAT;
  }
  k.why = why;
  return k;
}
}  // namespace

void index_gguf_file(const std::string& file, uint32_t shard, std::vector<TensorRec>& out, uint64_t* file_bytes, GgufMeta* meta) {
  MappedFile mf(file);
  if (file_bytes) *file_bytes = mf.n;
  Cursor c{mf.p, mf.n, 0, file};
  if (mf.n < 24) fail(KK_EFORMAT, "%s: too small for a GGUF header", file.c_str());
  uint32_t magic = c.get<uint32_t>();
  if (magic != 0x46554747u) fail(KK_EFORMAT, "%s: GGUF magic invalid", file.c_str());
  uint32_t version = c.get<uint32_t>();
  if ((version & 0xFFFF) == 0) fail(KK_EUNSUPPORTED, "%s: big-endian GGUF is not supported", file.c_str());
  if (version != 2 && version != 3) fail(KK_EUNSUPPORTED, "%s: GGUF version %u not supported", file.c_str(), version);
  uint64_t n_tensors = c.get<uint64_t>();
  uint64_t n_kv = c.get<uint64_t>();
  if (n_tensors > (1ull << 24) || n_kv > (1ull << 24)) fail(KK_EFORMAT, "%s: implausible GGUF counts", file.c_str());
  uint64_t alignment = 32;
  std::set<std::string> keys;
  GgufMeta m;
  std::map<std::string, GgufKey> per_arch;  // <any>.attention.head_count(_kv) / <any>.expert_count: general.architecture may come later
  for (uint64_t i = 0; i < n_kv; ++i) {
    std::string key = c.str();
    if (!keys.insert(key).second) fail(KK_EFORMAT, "%s: duplicate GGUF key %s", file.c_str(), key.c_str());
    uint32_t vt = c.get<uint32_t>();
    if (key == "general.alignment") {
      if (vt != 4) fail(KK_EFORMAT, "%s: bad type for general.alignment field", file.c_str());
      alignment = c.get<uint32_t>();
      if (alignment == 0 || (alignment & (alignment - 1)) != 0)
        fail(KK_EFORMAT, "%s: invalid alignment: must be a non-zero power of two", file.c_str());
    } else if (key == "general.architecture") {
      m.arch = gguf_read_key(c, key, vt, true);
    } else if (ends_with(key, ".attention.head_count") || ends_with(key, ".attention.head_count_kv") || ends_with(key, ".expert_count")) {
      per_arch[key] = gguf_read_key(c, key, vt, false);
    } else {
      gguf_skip_value(c, vt, 0);
    }
  }
  if (meta) {
    if (m.arch.seen && !m.arch.err) {
      auto take = [&](const char* suffix, GgufKey& k) {
        auto it = per_arch.find(m.arch.s + suffix);
        if (it != per_arch.end()) k = it->second;
      };
      take(".attention.head_count", m.head_count);
      take(".attention.head_count_kv", m.head_count_kv);
      take(".expert_count", m.expert_count);
    }
    *meta = m;
  }
  struct Ent { TensorRec t; uint64_t rel; };
  std::vector<Ent> ents;
  std::set<std::string> names;
  for (uint64_t i = 0; i < n_tensors; ++i) {
    Ent e;
    e.t.name = c.str();
    if (!names.insert(e.t.name).second) fail(KK_EFORMAT, "%s: found duplicated tensor with name %s", file.c_str(), e.t.name.c_str());
    if (e.t.name.size() >= KK_NAME_MAX) fail(KK_EUNSUPPORTED, "%s: tensor name longer than %d bytes", file.c_str(), KK_NAME_MAX - 1);
    uint32_t nd = c.get<uint32_t>();
    if (nd > KK_MAX_DIMS) fail(KK_EUNSUPPORTED, "%s: tensor %s has %u dims (max %d)", file.c_str(), e.t.name.c_str(), nd, KK_MAX_DIMS);
    std::vector<uint64_t> ne(nd);
    for (uint32_t d = 0; d < nd; ++d) ne[d] = c.get<uint64_t>();
    uint32_t gt = c.get<uint32_t>();
    e.rel = c.get<uint64_t>();
    int dt = dtype_from_ggml(gt);
    if (dt < 0) fail(KK_EUNSUPPORTED, "%s: tensor %s: ggml type %u not supported", file.c_str(), e.t.name.c_str(), gt);
    e.t.dtype = (uint32_t)dt;
    const DtypeInfo* di = dtype_info((uint32_t)dt);
    uint64_t nel = 1;
    for (auto d : ne)
      if (mul_overflow(nel, d, &nel)) fail(KK_EFORMAT, "%s: tensor %s: shape overflows", file.c_str(), e.t.name.c_str());
    if (di->block_elems > 1) {
      if (nd == 0 || ne[0] % di->block_elems != 0)
        fail(KK_EFORMAT, "%s: tensor %s: row length %llu is not a multiple of the %s block size %u", file.c_str(),
             e.t.name.c_str(), (unsigned long long)(nd ? ne[0] : 0), di->name, di->block_elems);
    }
    uint64_t nb;
    if (mul_overflow(nel / di->block_elems, (uint64_t)di->block_bytes, &nb)) fail(KK_EFORMAT, "%s: tensor %s: size overflows", file.c_str(), e.t.name.c_str());
    e.t.nbytes = nb;
    e.t.shape.assign(ne.rbegin(), ne.rend());  // ggml ne[] is innermost-first
    e.t.shard = shard;
    ents.push_back(std::move(e));
  }
  uint64_t data_start = align_up(c.off, alignment);
  for (auto& e : ents) {
    if (e.rel % alignment != 0) fail(KK_EFORMAT, "%s: tensor %s: data offset %llu not aligned to %llu", file.c_str(),
                                     e.t.name.c_str(), (unsigned long long)e.rel, (unsigned long long)alignment);
    uint64_t abs_off;
    if (__builtin_add_overflow(data_start, e.rel, &abs_off) || abs_off > mf.n || e.t.nbytes > mf.n - abs_off)
      fail(KK_EFORMAT, "%s: tensor %s: data out of file bounds", file.c_str(), e.t.name.c_str());
    e.t.file_offset = abs_off;
    out.push_back(std::move(e.t));
  }
}

// ---------------------------------------------------------------------------------------------
// path resolution
// ---------------------------------------------------------------------------------------------
namespace {
void sort_index(Index& ix) {
  std::stable_sort(ix.tensors.begin(), ix.tensors.end(), [](const TensorRec& a, const TensorRec& b) {
    if (a.shard != b.shard) return a.shard < b.shard;
    if (a.file_offset != b.file_offset) return a.file_offset < b.file_offset;
    if (a.nbytes != b.nbytes) return a.nbytes < b.nbytes;
    return a.name < b.name;
  });
  std::set<std::string> names;
  for (auto& t : ix.tensors)
    if (!names.insert(t.name).second) fail(KK_EFORMAT, "tensor \"%s\" appears in more than one shard", t.name.c_str());
}

Index index_sharded_safetensors(const std::string& index_json) {
  MappedFile mf(index_json);
  JsonValue doc = JsonParser((const char*)mf.p, (size_t)mf.n).parse_document();
  const JsonValue* wm = doc.kind == JsonValue::Object ? doc.find("weight_map") : nullptr;
  if (!wm || wm->kind != JsonValue::Object) fail(KK_EFORMAT, "%s: no weight_map object", index_json.c_str());
  std::set<std::string> files;
  for (auto& kv : wm->obj) {
    if (kv.second.kind != JsonValue::String) fail(KK_EFORMAT, "%s: weight_map[\"%s\"] is not a string", index_json.c_str(), kv.first.c_str());
    if (kv.second.s.find('/') != std::string::npos) fail(KK_EFORMAT, "%s: shard name \"%s\" escapes the directory", index_json.c_str(), kv.second.s.c_str());
    files.insert(kv.second.s);
  }
  if (files.empty()) fail(KK_EFORMAT, "%s: empty weight_map", index_json.c_str());
  Index ix;
  ix.format = "safetensors";
  std::string dir = dirname_of(index_json);
  std::map<std::string, uint32_t> shard_of;
  for (auto& f : files) {  // std::set iterates in name order => shard numbering is by file name
    uint32_t sid = (uint32_t)ix.shards.size();
    shard_of[f] = sid;
    ix.shards.push_back(dir + "/" + f);
    uint64_t fb = 0;
    index_safetensors_file(ix.shards.back(), sid, ix.tensors, &fb);
    ix.shard_bytes.push_back(fb);
  }
  std::map<std::string, uint32_t> where;
  for (auto& t : ix.tensors) where[t.name] = t.shard;
  for (auto& kv : wm->obj) {
    auto it = where.find(kv.first);
    if (it == where.end()) fail(KK_EFORMAT, "%s: weight_map names \"%s\" but %s does not contain it", index_json.c_str(), kv.first.c_str(), kv.second.s.c_str());
    if (it->second != shard_of[kv.second.s]) fail(KK_EFORMAT, "%s: weight_map puts \"%s\" in %s but it lives in another shard", index_json.c_str(), kv.first.c_str(), kv.second.s.c_str());
  }
  sort_index(ix);
  return ix;
}

Index index_files(const std::string& dir, const std::vector<std::string>& names, bool gguf) {
  Index ix;
  ix.format = gguf ? "gguf" : "safetensors";
  for (auto& f : names) {
    uint32_t sid = (uint32_t)ix.shards.size();
    ix.shards.push_back(dir.empty() ? f : dir + "/" + f);
    uint64_t fb = 0;
    if (gguf) {
      GgufMeta m;
      index_gguf_file(ix.shards.back(), sid, ix.tensors, &fb, &m);
      if (sid == 0) ix.gguf = m;
      else {  // the keys are the first shard's; a later shard that repeats one must agree, a disagreement is raised by a load that needs it
        GgufKey* first[] = {&ix.gguf.arch, &ix.gguf.head_count, &ix.gguf.head_count_kv, &ix.gguf.expert_count};
        const GgufKey* later[] = {&m.arch, &m.head_count, &m.head_count_kv, &m.expert_count};
        for (int k = 0; k < 4; ++k)
          if (later[k]->seen && first[k]->seen && !(*later[k] == *first[k]) && first[k]->err == 0) {
            first[k]->seen = true;
            first[k]->err = KK_EFORMAT;
            first[k]->why = "shard " + ix.shards.back() + " disagrees with the first shard on a metadata key the HF layout reads";
          }
      }
    } else {
      index_safetensors_file(ix.shards.back(), sid, ix.tensors, &fb);
    }
    ix.shard_bytes.push_back(fb);
  }
  sort_index(ix);
  return ix;
}
}  // namespace

Index index_path(const std::string& path_in) {
  if (path_in.empty()) fail(KK_EINVAL, "empty path");
  std::string path = abspath(path_in);
  if (is_dir(path)) {
    std::string idx = path + "/model.safetensors.index.json";
    if (is_file(idx)) return index_sharded_safetensors(idx);
    if (is_file(path + "/model.safetensors")) return index_files(path, {"model.safetensors"}, false);
    auto st = list_dir(path, ".safetensors");
    if (!st.empty()) return index_files(path, st, false);
    auto gg = list_dir(path, ".gguf");
    if (!gg.empty()) return index_files(path, gg, true);
    fail(KK_ENOENT, "%s: no model.safetensors.index.json, *.safetensors or *.gguf inside", path.c_str());
  }
  if (!is_file(path)) fail(KK_ENOENT, "%s: no such file or directory", path.c_str());
  if (ends_with(path, ".index.json")) return index_sharded_safetensors(path);
  if (ends_with(path, ".gguf")) return index_files("", {path}, true);
  if (ends_with(path, ".safetensors")) return index_files("", {path}, false);
  // sniff
  {
    MappedFile mf(path);
    if (mf.n >= 4 && memcmp(mf.p, "GGUF", 4) == 0) return index_files("", {path}, true);
  }
  return index_files("", {path}, false);
}

// ---------------------------------------------------------------------------------------------
// Views of an index: the Hugging Face layout and a pipeline stage
// ---------------------------------------------------------------------------------------------
namespace {

// Layer of a tensor: the first dotted component pair "<container>.<N>." with <container> one of layers / h / blk and N all digits.
// stack receives the name up to and including "<container>.", which names the numbered stack the layer belongs to.
bool layer_of(const std::string& n, uint64_t& layer, std::string& stack) {
  size_t c = 0;  // start of the current component
  while (c < n.size()) {
    const size_t dot = n.find('.', c);
    if (dot == std::string::npos) return false;
    const std::string comp = n.substr(c, dot - c);
    if (comp == "layers" || comp == "h" || comp == "blk") {
      const size_t d0 = dot + 1, d1 = n.find('.', d0);
      if (d1 != std::string::npos && d1 > d0 &&
          std::all_of(n.begin() + (long)d0, n.begin() + (long)d1, [](char ch) { return ch >= '0' && ch <= '9'; })) {
        layer = 0;
        for (size_t i = d0; i < d1; ++i) layer = std::min<uint64_t>(layer * 10 + (uint64_t)(n[i] - '0'), 0xFFFFFFFFull);  // beyond any layer_end
        stack = n.substr(0, dot + 1);
        return true;
      }
    }
    c = dot + 1;
  }
  return false;
}

}  // namespace

Index select_layers(Index ix, uint32_t begin, uint32_t end) {
  if (end == 0 && begin == 0) return ix;
  if (end == 0) fail(KK_EINVAL, "layer range [%u, 0): layer_end 0 selects the whole checkpoint and takes layer_begin 0", begin);
  if (begin >= end) fail(KK_EINVAL, "layer range [%u, %u) is empty", begin, end);
  std::string stack;
  uint64_t n_layers = 0;
  bool has_head = false;
  std::vector<uint64_t> layer(ix.tensors.size(), UINT64_MAX);  // UINT64_MAX: outer tensor
  for (size_t i = 0; i < ix.tensors.size(); ++i) {
    const std::string& n = ix.tensors[i].name;
    std::string s;
    if (layer_of(n, layer[i], s)) {
      if (stack.empty()) stack = s;
      else if (s != stack)
        fail(KK_EUNSUPPORTED, "the checkpoint has two numbered layer stacks, \"%s\" and \"%s\" (tensor %s): a layer range cannot tell which to cut",
             stack.c_str(), s.c_str(), n.c_str());
      n_layers = std::max(n_layers, layer[i] + 1);
    }
    has_head = has_head || ends_with(n, "lm_head.weight") || n == "output.weight";
  }
  if (stack.empty()) fail(KK_EUNSUPPORTED, "layer range [%u, %u): the checkpoint has no tensor with a layer index (layers.N. / h.N. / blk.N.)", begin, end);
  if (end > n_layers) fail(KK_EINVAL, "layer range [%u, %u) exceeds the checkpoint's %llu layers", begin, end, (unsigned long long)n_layers);
  const bool first = begin == 0, last = end == n_layers;
  auto any_suffix = [](const std::string& n, std::initializer_list<const char*> sufs) {
    for (auto s : sufs)
      if (ends_with(n, s)) return true;
    return false;
  };
  std::vector<TensorRec> kept;
  for (size_t i = 0; i < ix.tensors.size(); ++i) {
    const std::string& n = ix.tensors[i].name;
    bool keep;
    if (layer[i] != UINT64_MAX) keep = layer[i] >= begin && layer[i] < end;
    else if (any_suffix(n, {"embed_tokens.weight", "token_embd.weight", "wte.weight"})) keep = first || (last && !has_head);  // tied head
    else if (ends_with(n, "wpe.weight")) keep = first;
    else if (n == "output.weight" || any_suffix(n, {"lm_head.weight", "lm_head.bias", "norm.weight", "norm.bias", "ln_f.weight", "ln_f.bias"}))
      keep = last;
    else keep = true;  // e.g. GGUF rope_freqs.weight: every stage
    if (keep) kept.push_back(std::move(ix.tensors[i]));
  }
  ix.tensors = std::move(kept);
  ix.layer_begin = begin;
  ix.layer_end = end;
  ix.n_layers = n_layers;
  return ix;
}

namespace {

uint32_t need_key(const GgufKey& k, const char* key) {
  if (!k.seen) fail(KK_EFORMAT, "KK_LOAD_HF_LAYOUT: the GGUF metadata has no %s", key);
  if (k.err) fail(k.err, "KK_LOAD_HF_LAYOUT: %s", k.why.c_str());
  return (uint32_t)k.u;
}

// The rename table, restated from gguf-py's tensor_mapping for llama / qwen2 / qwen3: per-layer GGUF base name -> HF name under
// model.layers.N., and which architectures carry it.
struct HfName { const char* gguf; const char* hf; bool llama, qwen2, qwen3; };
const HfName kLayerNames[] = {
    {"attn_norm", "input_layernorm", true, true, true},        {"ffn_norm", "post_attention_layernorm", true, true, true},
    {"attn_q", "self_attn.q_proj", true, true, true},          {"attn_k", "self_attn.k_proj", true, true, true},
    {"attn_v", "self_attn.v_proj", true, true, true},          {"attn_output", "self_attn.o_proj", true, true, true},
    {"attn_q_norm", "self_attn.q_norm", false, false, true},   {"attn_k_norm", "self_attn.k_norm", false, false, true},
    {"ffn_gate", "mlp.gate_proj", true, true, true},           {"ffn_up", "mlp.up_proj", true, true, true},
    {"ffn_down", "mlp.down_proj", true, true, true},           {"ffn_gate_inp", "block_sparse_moe.gate", true, false, false},
};
// Mixtral's expert stacks: GGUF base name -> the per-expert HF name (HF's Mixtral files: w1 gate, w3 up, w2 down).
const HfName kExpertNames[] = {
    {"ffn_gate_exps", "w1", true, false, false}, {"ffn_up_exps", "w3", true, false, false}, {"ffn_down_exps", "w2", true, false, false}};

}  // namespace

Index to_hf_layout(Index ix, uint32_t flags) {
  if (!(flags & KK_LOAD_HF_LAYOUT)) return ix;
  if (ix.format != "gguf") fail(KK_EINVAL, "KK_LOAD_HF_LAYOUT applies to GGUF checkpoints only (this one is %s)", ix.format.c_str());
  const GgufMeta& M = ix.gguf;
  if (!M.arch.seen) fail(KK_EFORMAT, "KK_LOAD_HF_LAYOUT: the GGUF metadata has no general.architecture");
  if (M.arch.err) fail(M.arch.err, "KK_LOAD_HF_LAYOUT: %s", M.arch.why.c_str());
  const std::string& arch = M.arch.s;
  const bool llama = arch == "llama", qwen2 = arch == "qwen2", qwen3 = arch == "qwen3";
  if (!llama && !qwen2 && !qwen3)
    fail(KK_EUNSUPPORTED, "KK_LOAD_HF_LAYOUT: architecture \"%s\" is not supported (llama, qwen2 and qwen3 are)", arch.c_str());
  uint32_t n_head = 0, n_head_kv = 0;
  if (llama) {  // the Q/K row permutation is llama.cpp's for the llama architecture only; qwen's NEOX rotary keeps the rows
    n_head = need_key(M.head_count, (arch + ".attention.head_count").c_str());
    n_head_kv = M.head_count_kv.seen ? need_key(M.head_count_kv, (arch + ".attention.head_count_kv").c_str()) : n_head;
  }
  std::vector<TensorRec> out;
  out.reserve(ix.tensors.size());
  std::set<std::string> names;
  for (TensorRec& t : ix.tensors) {
    const std::string& n = t.name;
    std::string hf;
    if (n == "token_embd.weight") hf = "model.embed_tokens.weight";
    else if (n == "output_norm.weight") hf = "model.norm.weight";
    else if (n == "output.weight") hf = "lm_head.weight";
    else if (n == "rope_freqs.weight") hf = n;
    else {
      // blk.N.<base>.weight|bias
      const size_t d0 = 4, d1 = n.find('.', d0);
      const size_t sfx = n.rfind('.');
      const bool layered = n.compare(0, 4, "blk.") == 0 && d1 != std::string::npos && d1 > d0 && sfx > d1 + 1 &&
                           std::all_of(n.begin() + (long)d0, n.begin() + (long)d1, [](char ch) { return ch >= '0' && ch <= '9'; });
      const std::string suffix = layered ? n.substr(sfx) : "";
      if (layered && (suffix == ".weight" || suffix == ".bias")) {
        const std::string layer = n.substr(d0, d1 - d0), base = n.substr(d1 + 1, sfx - d1 - 1);
        const std::string prefix = "model.layers." + layer + ".";
        auto in_arch = [&](const HfName& e) { return (llama && e.llama) || (qwen2 && e.qwen2) || (qwen3 && e.qwen3); };
        for (auto& e : kLayerNames)
          if (base == e.gguf && in_arch(e)) hf = prefix + e.hf + suffix;
        bool split = false;
        for (auto& e : kExpertNames) {
          if (base != e.gguf || !in_arch(e) || suffix != ".weight") continue;
          if (t.shape.size() != 3 || t.shape[0] == 0)
            fail(KK_EFORMAT, "KK_LOAD_HF_LAYOUT: expert stack %s is not [experts, rows, cols]", n.c_str());
          const uint64_t E = t.shape[0];
          if (M.expert_count.seen && need_key(M.expert_count, (arch + ".expert_count").c_str()) != E)
            fail(KK_EFORMAT, "KK_LOAD_HF_LAYOUT: expert stack %s has %llu experts, %s.expert_count says %llu", n.c_str(), (unsigned long long)E,
                 arch.c_str(), (unsigned long long)M.expert_count.u);
          for (uint64_t x = 0; x < E; ++x) {  // each expert is a whole number of rows, so a contiguous byte range of the stack
            TensorRec r;
            r.name = prefix + "block_sparse_moe.experts." + std::to_string(x) + "." + e.hf + ".weight";
            r.dtype = t.dtype;
            r.shape = {t.shape[1], t.shape[2]};
            r.shard = t.shard;
            r.nbytes = t.nbytes / E;
            r.file_offset = t.file_offset + x * r.nbytes;
            if (!names.insert(r.name).second) fail(KK_EFORMAT, "KK_LOAD_HF_LAYOUT: two tensors map to %s", r.name.c_str());
            out.push_back(std::move(r));
          }
          split = true;
        }
        if (split) continue;
        const bool q = base == "attn_q", k = base == "attn_k";
        if (llama && (q || k) && !hf.empty()) {
          const uint32_t heads = q ? n_head : n_head_kv;
          const uint64_t rows = t.shape.empty() ? 0 : t.shape[0];
          if (t.shape.empty() || t.shape.size() > 2 || rows % (2ull * heads) != 0)
            fail(KK_EFORMAT, "KK_LOAD_HF_LAYOUT: %s has %llu rows, not a multiple of 2 * %u heads", n.c_str(), (unsigned long long)rows, heads);
          // the rows are moved one by one, so each must be a whole number of the op's source units: a block-quantised row holds whole
          // blocks (a 1-D block-quantised tensor, whose rows are single elements, cannot be un-permuted)
          const DtypeInfo* di = dtype_info(t.dtype);
          const uint64_t row_elems = t.shape.size() == 2 ? t.shape[1] : 1;
          if (!di || di->block_bytes == 0 || row_elems % di->block_elems != 0)
            fail(KK_EUNSUPPORTED, "KK_LOAD_HF_LAYOUT: %s (%s, shape of %zu dims) has rows that are not whole %s blocks; its rows cannot be un-permuted",
                 n.c_str(), di ? di->name : "?", t.shape.size(), di ? di->name : "?");
          t.rope_heads = heads;
        }
      }
    }
    if (hf.empty()) fail(KK_EUNSUPPORTED, "KK_LOAD_HF_LAYOUT: tensor %s has no Hugging Face name for architecture %s", n.c_str(), arch.c_str());
    if (!names.insert(hf).second) fail(KK_EFORMAT, "KK_LOAD_HF_LAYOUT: two tensors map to %s", hf.c_str());
    t.name = std::move(hf);
    out.push_back(std::move(t));
  }
  ix.tensors = std::move(out);
  ix.hf_arch = arch;
  return ix;
}

Index index_for_load(const std::string& path, uint32_t flags, uint32_t layer_begin, uint32_t layer_end) {
  return select_layers(to_hf_layout(index_path(path), flags), layer_begin, layer_end);
}
}  // namespace kk
