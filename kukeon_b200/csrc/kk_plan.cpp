// Load planning: decides where every tensor lives in the pool, which op moves it, and how the
// checkpoint's bytes are cut into staging chunks per ingesting rank.  Pure host code.
#include "kk_plan.hpp"

#include <algorithm>
#include <cstring>
#include <set>
#include <sstream>

#include "kk_json.hpp"

namespace kk {

namespace {

bool ends_with(const std::string& s, const char* suf) {
  size_t n = strlen(suf);
  return s.size() >= n && memcmp(s.data() + s.size() - n, suf, n) == 0;
}
bool contains(const std::string& s, const char* sub) { return s.find(sub) != std::string::npos; }

struct OpInfo {
  uint32_t op;
  uint32_t pool_dtype;
  uint64_t src_unit_bytes;  // source bytes per op unit
  uint64_t out_unit_bytes;  // pool bytes per op unit
  uint64_t tile_units;      // op units per tile (split granule)
};

// op for a non-transposed tensor of file dtype dt.  Every float output is bf16, or fp16 under KK_LOAD_F16 (out): the op codes are the
// same, the launch's output format (KK_LAUNCH_F16) picks the kernel.  Under it the 16-bit roles swap: F16 is the verbatim copy and BF16
// takes the 16-bit cast.
OpInfo op_for(uint32_t dt, uint32_t flags, const std::string& name) {
  const bool f16 = (flags & KK_LOAD_F16) != 0;
  const uint32_t out = f16 ? KK_F16 : KK_BF16;
  switch (dt) {
    case KK_BF16:
    case KK_F16:
      if (dt == out) return {KK_OP_COPY, out, 1, 1, KK_TILE_SRC_BYTES};
      return {KK_OP_F16_BF16, out, 2, 2, KK_TILE_SRC_BYTES / 2};
    case KK_F32:
      if (flags & KK_LOAD_KEEP_F32) return {KK_OP_COPY, KK_F32, 1, 1, KK_TILE_SRC_BYTES};
      return {KK_OP_F32_BF16, out, 4, 2, KK_TILE_SRC_BYTES / 4};
    case KK_F8_E4M3:
      if (flags & KK_LOAD_F8_TO_BF16) return {KK_OP_F8E4M3_BF16, out, 1, 2, KK_TILE_SRC_BYTES};
      break;
    case KK_F8_E5M2:
      if (flags & KK_LOAD_F8_TO_BF16) return {KK_OP_F8E5M2_BF16, out, 1, 2, KK_TILE_SRC_BYTES};
      break;
    default: break;
  }
  // block-quantised GGUF types -> bf16 / fp16 (geometry shared with the kernel: kk_ops.h)
  uint32_t qop = KK_OP_COUNT;
  switch (dt) {
    case KK_Q4_0: qop = KK_OP_Q4_0_BF16; break;
    case KK_Q4_1: qop = KK_OP_Q4_1_BF16; break;
    case KK_Q5_0: qop = KK_OP_Q5_0_BF16; break;
    case KK_Q5_1: qop = KK_OP_Q5_1_BF16; break;
    case KK_Q8_0: qop = KK_OP_Q8_0_BF16; break;
    case KK_Q2_K: qop = KK_OP_Q2K_BF16; break;
    case KK_Q3_K: qop = KK_OP_Q3K_BF16; break;
    case KK_Q4_K: qop = KK_OP_Q4K_BF16; break;
    case KK_Q5_K: qop = KK_OP_Q5K_BF16; break;
    case KK_Q6_K: qop = KK_OP_Q6K_BF16; break;
    case KK_IQ4_NL: qop = KK_OP_IQ4NL_BF16; break;
    case KK_IQ4_XS: qop = KK_OP_IQ4XS_BF16; break;
    case KK_MXFP4: qop = KK_OP_MXFP4_BF16; break;
    case KK_IQ2_XXS: qop = KK_OP_IQ2XXS_BF16; break;
    case KK_IQ2_XS: qop = KK_OP_IQ2XS_BF16; break;
    case KK_IQ2_S: qop = KK_OP_IQ2S_BF16; break;
    case KK_IQ3_XXS: qop = KK_OP_IQ3XXS_BF16; break;
    case KK_IQ3_S: qop = KK_OP_IQ3S_BF16; break;
    case KK_IQ1_S: qop = KK_OP_IQ1S_BF16; break;
    case KK_IQ1_M: qop = KK_OP_IQ1M_BF16; break;
    case KK_TQ1_0: qop = KK_OP_TQ1_0_BF16; break;
    case KK_TQ2_0: qop = KK_OP_TQ2_0_BF16; break;
    case KK_NVFP4: qop = KK_OP_NVFP4_BF16; break;
    default: break;
  }
  if (qop != KK_OP_COUNT) {
    const KKBlockGeom g = kk_block_geom(qop);
    return {qop, out, g.block_bytes, g.out_bytes, g.tile_blocks};
  }
  const DtypeInfo* di = dtype_info(dt);
  if (!di) fail(KK_EINVAL, "tensor %s: unknown dtype %u", name.c_str(), dt);
  if (di->block_elems > 1 && dt >= 32)
    fail(KK_EUNSUPPORTED, "tensor %s: %s -> bf16 dequantisation is not implemented (every GGUF weight type except Q8_K / Q8_1 is)", name.c_str(), di->name);
  return {KK_OP_COPY, dt, 1, 1, KK_TILE_SRC_BYTES};  // integers, bool, fp8, f64, sub-byte: verbatim bytes
}

struct Piece {
  uint32_t shard;
  uint64_t file_off;   // first source byte
  uint64_t run_bytes;  // bytes per run (whole piece when n_runs == 1)
  uint64_t n_runs;
  uint64_t stride;     // file distance between runs
  OpInfo oi;
  uint64_t units;      // total op units (transposes: source rows)
  uint64_t dst_off;
  uint32_t p0 = 0, p1 = 0;  // transposes: C, R
  bool transpose = false;
  uint64_t row_src_bytes = 0;  // transposes: C * es
  bool rowsplit = false;       // SCATTER exchange: whole rows in, column slices out to every pool
  uint32_t rs_row_bytes = 0, rs_slice_bytes = 0, rs_first_row = 0;
};

struct ChunkBuilder {
  PartPlan& pp;
  uint64_t cap;
  Chunk cur;
  uint64_t pos = 0;
  bool open = false;

  explicit ChunkBuilder(PartPlan& p, uint64_t c) : pp(p), cap(c) {}

  void begin(uint32_t shard) {
    cur = Chunk();
    cur.shard = shard;
    cur.seg_begin = (uint32_t)pp.segs.size();
    pos = 0;
    open = true;
  }
  void flush() {
    if (!open) return;
    if (cur.seg_count) {
      cur.buf_bytes = pos;
      pp.src_bytes += cur.src_bytes;
      pp.out_bytes += cur.out_bytes;
      pp.chunks.push_back(std::move(cur));
    }
    open = false;
  }
  // Reserve room for `len` bytes read from file_off; returns the buffer offset.
  uint64_t add_read(uint64_t file_off, uint64_t len) {
    if (!cur.reads.empty()) {
      ReadOp& l = cur.reads.back();
      if (l.file_off + l.len == file_off && l.buf_off + l.len == pos) {
        l.len += len;
        uint64_t at = pos;
        pos += len;
        cur.src_bytes += len;
        return at;
      }
    }
    uint64_t at = align_up(pos, 16);
    cur.reads.push_back({file_off, len, at});
    pos = at + len;
    cur.src_bytes += len;
    return at;
  }
  void add_seg(const Piece& pc, uint64_t src_off, uint64_t units, uint64_t units_done) {
    KKSeg s{};
    s.src_off = src_off;
    s.units = units;
    s.op = pc.oi.op;
    s.tile_begin = cur.n_tiles;
    if (pc.transpose) {
      s.dst_off = pc.dst_off;
      s.p0 = pc.p0;
      s.p1 = pc.p1;
      s.p2 = (uint32_t)units_done;
      cur.out_bytes += units * pc.p0 * pc.oi.out_unit_bytes;
    } else if (pc.rowsplit) {
      s.dst_off = pc.dst_off;
      s.p0 = pc.rs_row_bytes;
      s.p1 = pc.rs_slice_bytes;
      s.p2 = pc.rs_first_row;
      s.p3 = (uint32_t)units_done;
      cur.out_bytes += units;
    } else {
      s.dst_off = pc.dst_off + units_done * pc.oi.out_unit_bytes;
      cur.out_bytes += units * pc.oi.out_unit_bytes;
    }
    uint64_t nt = kk_seg_tiles(s.op, s.units, s.p0);
    if (nt + cur.n_tiles > 0xFFFFFFF0ull) fail(KK_EUNSUPPORTED, "chunk has too many tiles");
    cur.n_tiles += (uint32_t)nt;
    cur.seg_count++;
    pp.segs.push_back(s);
  }

  void emit(const Piece& pc) {
    if (pc.units == 0) return;
    if (open && cur.shard != pc.shard) flush();
    if (!open) begin(pc.shard);
    if (pc.n_runs == 1) {
      const uint64_t ub = pc.transpose ? pc.row_src_bytes : pc.oi.src_unit_bytes;
      const uint64_t gran = pc.transpose ? KK_T_ROWS : pc.oi.tile_units;
      uint64_t done = 0;
      while (done < pc.units) {
        if (cur.seg_count >= kMaxSegsPerChunk) { flush(); begin(pc.shard); }
        const uint64_t start = align_up(pos, 16);
        const uint64_t space = cap > start ? cap - start : 0;
        uint64_t fit = ub ? space / ub : 0;
        const uint64_t rem = pc.units - done;
        uint64_t take;
        if (fit >= rem) take = rem;
        else take = fit / gran * gran;
        if (take == 0) {
          if (cur.seg_count == 0) fail(KK_EINVAL, "staging buffer (%llu B) smaller than one tile", (unsigned long long)cap);
          flush();
          begin(pc.shard);
          continue;
        }
        uint64_t at = add_read(pc.file_off + done * ub, take * ub);
        add_seg(pc, at, take, done);
        done += take;
      }
    } else {
      // strided rows packed back to back in the buffer; split on multiples of 16 rows
      const uint64_t units_per_run = pc.run_bytes / pc.oi.src_unit_bytes;
      uint64_t rdone = 0;
      while (rdone < pc.n_runs) {
        if (cur.seg_count >= kMaxSegsPerChunk) { flush(); begin(pc.shard); }
        const uint64_t start = align_up(pos, 16);
        const uint64_t space = cap > start ? cap - start : 0;
        uint64_t fit = space / pc.run_bytes;
        const uint64_t rem = pc.n_runs - rdone;
        uint64_t take = fit >= rem ? rem : fit / 16 * 16;
        if (take == 0) {
          if (cur.seg_count == 0) fail(KK_EINVAL, "staging buffer (%llu B) smaller than 16 slice rows", (unsigned long long)cap);
          flush();
          begin(pc.shard);
          continue;
        }
        uint64_t first_at = 0;
        for (uint64_t r = 0; r < take; ++r) {
          uint64_t at;
          if (r == 0) {
            at = align_up(pos, 16);
            cur.reads.push_back({pc.file_off + (rdone + r) * pc.stride, pc.run_bytes, at});
            first_at = at;
          } else {
            at = pos;
            cur.reads.push_back({pc.file_off + (rdone + r) * pc.stride, pc.run_bytes, at});
          }
          pos = at + pc.run_bytes;
          cur.src_bytes += pc.run_bytes;
        }
        add_seg(pc, first_at, take * units_per_run, rdone * units_per_run);
        rdone += take;
      }
    }
  }

  static constexpr uint32_t kMaxSegsPerChunk = 1024;
};

}  // namespace

bool is_gpt2_conv1d(const TensorRec& t) {
  if (t.shape.size() != 2) return false;
  return ends_with(t.name, "attn.c_attn.weight") || ends_with(t.name, "attn.c_proj.weight") ||
         ends_with(t.name, "mlp.c_fc.weight") || ends_with(t.name, "mlp.c_proj.weight");
}

uint64_t seg_out_extent(const KKSeg& s) {
  switch (s.op) {
    case KK_OP_ROWSPLIT: return 0;
    case KK_OP_COPY: return s.units;
    case KK_OP_F32_BF16: case KK_OP_F16_BF16: case KK_OP_F8E4M3_BF16: case KK_OP_F8E5M2_BF16: return s.units * 2;
    case KK_OP_T_B32: return (uint64_t)s.p0 * s.p1 * 4;
    case KK_OP_T_F32_BF16: case KK_OP_T_F16_BF16: case KK_OP_T_B16: return (uint64_t)s.p0 * s.p1 * 2;
    default: return s.units * kk_block_geom(s.op).out_bytes;  // block-dequantising ops
  }
}

uint32_t scatter_slice_dim(const TensorRec& t, int n_parts) {
  if (n_parts <= 1 || t.shape.size() != 2) return kNoSlice;
  const std::string& n = t.name;
  static const char* kDim0[] = {"q_proj.weight", "k_proj.weight", "v_proj.weight", "gate_proj.weight", "up_proj.weight",
                                "embed_tokens.weight", "lm_head.weight", "attn_q.weight", "attn_k.weight", "attn_v.weight",
                                "ffn_gate.weight", "ffn_up.weight", "token_embd.weight", "output.weight"};
  static const char* kDim1[] = {"o_proj.weight", "down_proj.weight", "attn_output.weight", "ffn_down.weight"};
  uint32_t dim = kNoSlice;
  for (auto s : kDim1)
    if (ends_with(n, s)) dim = 1;
  if (dim == kNoSlice)
    for (auto s : kDim0)
      if (ends_with(n, s) && !contains(n, "norm")) dim = 0;
  if (dim == kNoSlice) return kNoSlice;
  if (t.shape[0] == 0 || t.shape[1] == 0) return kNoSlice;  // empty tensors are "replicated" (nothing to slice)
  if (t.shape[dim] % (uint64_t)n_parts != 0) return kNoSlice;
  const DtypeInfo* di = dtype_info(t.dtype);
  // sub-byte safetensors dtypes (F4: 2 elements per byte, F6: 4 per 3 bytes) FIRST — their table rows also have block_elems > 1, so they used to
  // fall into the block-quantised branch below and a row of cols * bits not divisible by 8 was sliced mid-byte (ADVICE r1): never slice them
  if (t.dtype == KK_F4 || t.dtype == KK_F6_E2M3 || t.dtype == KK_F6_E3M2) return kNoSlice;
  if (di->block_bytes == 0) return kNoSlice;
  if (di->block_elems > 1) {
    // block-quantised rows: dim-0 slices stay whole rows of blocks; dim-1 slices would cut blocks.
    if (dim == 1) return kNoSlice;
  }
  return dim;
}

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

namespace {

// Pieces of a tensor whose rows llama.cpp interleaved per rotary half (TensorRec::rope_heads), for HF rows [r0, r1) of it with HF row r0 at
// pool offset dst.  HF row h*hd + k*hd/2 + i is file row h*hd + 2i + k, so the rows of one (head, half) group are one strided run of file rows.
// The pieces come in HF row order and tile [r0, r1) exactly: destination offsets never decrease in plan order (a part stays one pool range)
// and every pool byte of the slice is written once.  A slice boundary may cut a group (scatter does not need heads % ranks == 0).
void unpermuted_pieces(const TensorRec& t, const Piece& whole, uint64_t r0, uint64_t r1, uint64_t dst, std::vector<Piece>& out) {
  const uint64_t R = t.shape[0], half = R / t.rope_heads / 2, row_bytes = t.nbytes / R;
  const uint64_t row_units = row_bytes / whole.oi.src_unit_bytes, out_row = row_units * whole.oi.out_unit_bytes;
  if (row_bytes * R != t.nbytes || row_units * whole.oi.src_unit_bytes != row_bytes || row_units == 0)  // to_hf_layout refuses such tensors
    fail(KK_EUNSUPPORTED, "KK_LOAD_HF_LAYOUT: tensor %s: a row is not a whole number of source units", t.name.c_str());
  for (uint64_t g = r0 / half; g * half < r1; ++g) {
    const uint64_t a = std::max(r0, g * half), b = std::min(r1, (g + 1) * half);
    const uint64_t head = g / 2, k = g % 2, i0 = a - g * half;
    Piece pc = whole;
    pc.file_off = t.file_offset + (head * 2 * half + 2 * i0 + k) * row_bytes;
    pc.run_bytes = row_bytes;
    pc.n_runs = b - a;
    pc.stride = 2 * row_bytes;
    pc.units = (b - a) * row_units;
    pc.dst_off = dst + (a - r0) * out_row;
    // the consumers store whole 16-byte vectors from a segment's first output on
    if (pc.dst_off % 16 != 0)
      fail(KK_EUNSUPPORTED, "KK_LOAD_HF_LAYOUT: tensor %s: HF row %llu would start at pool offset %llu, off a 16-byte boundary (%llu B per row)",
           t.name.c_str(), (unsigned long long)a, (unsigned long long)pc.dst_off, (unsigned long long)out_row);
    out.push_back(pc);
  }
}

}  // namespace

Plan build_plan(Index index, int mode, uint32_t flags, int n_parts, uint64_t chunk_bytes) {
  if (n_parts < 1 || n_parts > KK_MAX_DEVICES) fail(KK_EINVAL, "n_parts %d out of range", n_parts);
  if (mode != KK_MODE_SINGLE && mode != KK_MODE_BROADCAST && mode != KK_MODE_SCATTER) fail(KK_EINVAL, "unknown mode %d", mode);
  if (mode == KK_MODE_SINGLE && n_parts != 1) fail(KK_EINVAL, "KK_MODE_SINGLE takes exactly one part");
  Plan P;
  P.index = std::move(index);
  P.mode = mode;
  P.flags = flags;
  P.n_parts = n_parts;
  const auto& T = P.index.tensors;
  for (auto& t : T) P.file_bytes += t.nbytes;

  const int n_layouts = mode == KK_MODE_SCATTER ? n_parts : 1;
  P.placements.assign((size_t)n_layouts, {});
  P.pool_bytes.assign((size_t)n_layouts, 0);

  // pieces[layout][tensor]
  std::vector<std::vector<Piece>> pieces((size_t)n_layouts);
  for (int L = 0; L < n_layouts; ++L) {
    uint64_t off = 0;
    auto& pl = P.placements[(size_t)L];
    pl.reserve(T.size());
    for (auto& t : T) {
      Placement p;
      Piece pc{};
      pc.shard = t.shard;
      pc.n_runs = 1;
      const bool tr = (flags & KK_LOAD_GPT2_CONV1D_T) && mode != KK_MODE_SCATTER && is_gpt2_conv1d(t) &&
                      (t.dtype == KK_F32 || t.dtype == KK_F16 || t.dtype == KK_BF16 || t.dtype == KK_I16 || t.dtype == KK_U16 ||
                       t.dtype == KK_I32 || t.dtype == KK_U32);
      if (tr) {
        const uint64_t R = t.shape[0], C = t.shape[1];
        if (R > 0xFFFFFFFFull || C > 0xFFFFFFFFull) fail(KK_EUNSUPPORTED, "tensor %s too large to transpose", t.name.c_str());
        uint32_t op, pdt;
        uint64_t es, oes;
        const uint32_t out = (flags & KK_LOAD_F16) ? KK_F16 : KK_BF16;  // the float output format, as in op_for
        if (t.dtype == KK_F32 && !(flags & KK_LOAD_KEEP_F32)) { op = KK_OP_T_F32_BF16; pdt = out; es = 4; oes = 2; }
        else if ((t.dtype == KK_F16 || t.dtype == KK_BF16) && t.dtype != out) { op = KK_OP_T_F16_BF16; pdt = out; es = 2; oes = 2; }
        else if (t.dtype == KK_F32 || t.dtype == KK_I32 || t.dtype == KK_U32) { op = KK_OP_T_B32; pdt = t.dtype; es = 4; oes = 4; }
        else { op = KK_OP_T_B16; pdt = t.dtype; es = 2; oes = 2; }
        pc.oi = {op, pdt, es, oes, KK_T_ROWS};
        pc.transpose = true;
        pc.row_src_bytes = C * es;
        pc.units = C ? R : 0;  // [R, 0]: nothing to move (found by the hypothesis test)
        pc.p0 = (uint32_t)C;
        pc.p1 = (uint32_t)R;
        pc.file_off = t.file_offset;
        pc.run_bytes = t.nbytes;
        p.dtype = pdt;
        p.shape = {C, R};
        p.nbytes = R * C * oes;
      } else {
        OpInfo oi = op_for(t.dtype, flags, t.name);
        pc.oi = oi;
        const DtypeInfo* di = dtype_info(t.dtype);
        uint32_t sd = mode == KK_MODE_SCATTER ? scatter_slice_dim(t, n_parts) : kNoSlice;
        p.dtype = oi.pool_dtype;
        p.shape = t.shape;
        if (sd == kNoSlice) {
          pc.file_off = t.file_offset;
          pc.run_bytes = t.nbytes;
          pc.units = t.nbytes / oi.src_unit_bytes;
          p.nbytes = pc.units * oi.out_unit_bytes;
        } else {
          const uint64_t R = t.shape[0], C = t.shape[1];
          p.slice_dim = sd;
          if (sd == 0) {
            const uint64_t rows = R / (uint64_t)n_parts;
            const uint64_t row_bytes = t.nbytes / R;  // whole rows (also for block-quantised types)
            p.slice_begin = rows * (uint64_t)L;
            p.shape[0] = rows;
            pc.file_off = t.file_offset + p.slice_begin * row_bytes;
            pc.run_bytes = rows * row_bytes;
            pc.units = pc.run_bytes / oi.src_unit_bytes;
          } else {
            const uint64_t cols = C / (uint64_t)n_parts;
            const uint64_t es = di->block_bytes;
            p.slice_begin = cols * (uint64_t)L;
            p.shape[1] = cols;
            const uint64_t row_bytes = C * es, slice_bytes = cols * es;
            const bool exchange = (flags & KK_LOAD_SCATTER_EXCHANGE) && oi.op == KK_OP_COPY && row_bytes <= 0xFFFFFFFFull &&
                                  R <= 0xFFFFFFFFull && (R / (uint64_t)n_parts + (uint64_t)n_parts) * row_bytes < 0xFFFFFFFFull;
            if (exchange) {
              // this rank ingests whole rows [r0, r1) and the kernel deals column slice j of every row to pool j
              const uint64_t per = R / (uint64_t)n_parts;
              const uint64_t r0 = per * (uint64_t)L, r1 = (L == n_parts - 1) ? R : per * (uint64_t)(L + 1);
              pc.rowsplit = true;
              pc.rs_row_bytes = (uint32_t)row_bytes;
              pc.rs_slice_bytes = (uint32_t)slice_bytes;
              pc.rs_first_row = (uint32_t)r0;
              pc.file_off = t.file_offset + r0 * row_bytes;
              pc.run_bytes = (r1 - r0) * row_bytes;
              pc.units = pc.run_bytes;
              pc.oi.op = KK_OP_ROWSPLIT;
              p.nbytes = R * slice_bytes;
            } else {
              pc.file_off = t.file_offset + p.slice_begin * es;
              pc.run_bytes = cols * es;
              pc.n_runs = R;
              pc.stride = C * es;
              pc.units = R * (pc.run_bytes / oi.src_unit_bytes);
            }
          }
          if (!pc.rowsplit) p.nbytes = pc.units * oi.out_unit_bytes;
        }
      }
      p.pool_offset = off;
      pc.dst_off = off;
      off = align_up(off + p.nbytes, KK_POOL_ALIGN);
      if (t.rope_heads && !tr && p.nbytes) {  // the same slot, filled in HF row order (a dim-0 slice keeps HF rows)
        const uint64_t r0 = p.slice_dim == 0 ? p.slice_begin : 0;
        unpermuted_pieces(t, pc, r0, r0 + p.shape[0], p.pool_offset, pieces[(size_t)L]);
      } else {
        pieces[(size_t)L].push_back(pc);
      }
      pl.push_back(std::move(p));
    }
    P.pool_bytes[(size_t)L] = off ? off : KK_POOL_ALIGN;
  }

  // chunk size: keep >= 8 chunks per part for balance on small checkpoints, never above the slot size
  uint64_t cb = chunk_bytes;
  {
    uint64_t want = P.file_bytes / ((uint64_t)n_parts * 8) + 1;
    want = align_up(want, 1u << 20);
    const uint64_t floor_b = 4ull << 20;
    if (want < floor_b) want = floor_b;
    if (want < cb) cb = want;
  }
  if (cb < KK_TILE_SRC_BYTES * 2ull) fail(KK_EINVAL, "staging buffer too small");
  cb -= 64;  // room for the 16-B aligned over-read of the last tile

  P.parts.assign((size_t)n_parts, {});
  if (mode == KK_MODE_SCATTER) {
    for (int g = 0; g < n_parts; ++g) {
      ChunkBuilder cbld(P.parts[(size_t)g], cb);
      for (auto& pc : pieces[(size_t)g]) cbld.emit(pc);
      cbld.flush();
    }
  } else {
    PartPlan all;
    {
      ChunkBuilder cbld(all, cb);
      for (auto& pc : pieces[0]) cbld.emit(pc);
      cbld.flush();
    }
    // contiguous split of the chunk list by cumulative source bytes
    uint64_t acc = 0;
    for (auto& c : all.chunks) {
      int g = all.src_bytes ? (int)((__uint128_t)acc * (uint64_t)n_parts / all.src_bytes) : 0;
      if (g >= n_parts) g = n_parts - 1;
      acc += c.src_bytes;
      PartPlan& pp = P.parts[(size_t)g];
      Chunk nc = c;
      nc.seg_begin = (uint32_t)pp.segs.size();
      for (uint32_t i = 0; i < c.seg_count; ++i) pp.segs.push_back(all.segs[c.seg_begin + i]);
      pp.src_bytes += nc.src_bytes;
      pp.out_bytes += nc.out_bytes;
      pp.chunks.push_back(std::move(nc));
    }
  }
  return P;
}

LoadShape resolve_load_shape(const kk_load_opts& opts, int n_devices, bool peer_ok) {
  LoadShape S;
  S.multi_proc = opts.part_count > 1;
  const int part_count = S.multi_proc ? opts.part_count : 1;
  S.rank = S.multi_proc ? opts.part_index : 0;
  if (S.rank < 0 || S.rank >= part_count || part_count > KK_MAX_DEVICES) fail(KK_EINVAL, "part %d of %d out of range", S.rank, part_count);
  if (opts.mode < KK_MODE_SINGLE || opts.mode > KK_MODE_SCATTER) fail(KK_EINVAL, "unknown mode %d", opts.mode);
  if (opts.fanout < KK_FANOUT_P2P || opts.fanout > KK_FANOUT_PULL) fail(KK_EINVAL, "unknown fanout %d", opts.fanout);
  const bool bcast = opts.mode == KK_MODE_BROADCAST;
  if (opts.fanout == KK_FANOUT_NVLS) {
    // every "cannot do NVLS here" is KK_EUNSUPPORTED (the contract since the first ABI version), whatever the reason
    if (!bcast) fail(KK_EUNSUPPORTED, "fan-out NVLS only applies to KK_MODE_BROADCAST");
    if (S.multi_proc) fail(KK_EUNSUPPORTED, "fan-out NVLS needs one process owning all devices (sharing a multicast object across processes is not implemented)");
    if (n_devices < 2) fail(KK_EUNSUPPORTED, "fan-out NVLS needs at least two devices in the context");
  }
  if (opts.fanout == KK_FANOUT_RAW && !bcast) fail(KK_EINVAL, "KK_FANOUT_RAW only applies to KK_MODE_BROADCAST");
  if (opts.fanout == KK_FANOUT_PULL && !bcast) fail(KK_EINVAL, "KK_FANOUT_PULL only applies to KK_MODE_BROADCAST");
  if (opts.fanout == KK_FANOUT_PULL && !S.multi_proc)
    fail(KK_EINVAL, "KK_FANOUT_PULL is for one-process-per-GPU operation (part_count > 1); one process owning the GPUs fans out with P2P stores");
  if (S.multi_proc && n_devices != 1) fail(KK_EINVAL, "multi-process parts need a one-device context (got %d devices)", n_devices);
  if (S.multi_proc && opts.mode == KK_MODE_SINGLE) fail(KK_EINVAL, "KK_MODE_SINGLE cannot be split into parts");

  S.n_parts = opts.mode == KK_MODE_SINGLE ? 1 : S.multi_proc ? part_count : n_devices;
  if (S.multi_proc || opts.mode == KK_MODE_SINGLE) S.local_parts = {S.rank};
  else
    for (int i = 0; i < n_devices; ++i) S.local_parts.push_back(i);
  S.xdst = opts.mode == KK_MODE_SCATTER && (opts.flags & KK_LOAD_SCATTER_EXCHANGE) && S.n_parts > 1;
  S.peer_ok = peer_ok;
  // one process, >= 2 devices and no stores between them: each device builds its whole pool itself
  const bool replicas = bcast && !S.multi_proc && n_devices > 1 && (opts.fanout == KK_FANOUT_NONE || !peer_ok);
  if (bcast) {
    if (opts.fanout == KK_FANOUT_RAW) S.order = LoadOrder::kRaw;
    else if (opts.fanout == KK_FANOUT_PULL) S.order = LoadOrder::kPull;
    else if (opts.fanout == KK_FANOUT_NVLS) S.order = LoadOrder::kNvls;
    else if (replicas) S.order = LoadOrder::kReplicas;
    else if (opts.fanout == KK_FANOUT_P2P && (S.multi_proc || n_devices > 1)) S.order = LoadOrder::kPush;
  }
  S.every_part = replicas && S.order != LoadOrder::kRaw;  // RAW's stage 1 gathers the parts; its stage 2 converts all of them anyway
  S.two_stage = S.multi_proc && (S.order == LoadOrder::kRaw || S.order == LoadOrder::kPull);
  return S;
}

std::string plan_to_json(const Plan& P) {
  std::ostringstream o;
  o << "{\"mode\":" << P.mode << ",\"flags\":" << P.flags << ",\"n_parts\":" << P.n_parts << ",\"file_bytes\":" << P.file_bytes
    << ",\"format\":\"" << P.index.format << "\"";
  if (!P.index.hf_arch.empty()) o << ",\"layout\":\"hf\",\"architecture\":\"" << json_escape(P.index.hf_arch) << "\"";
  if (P.index.layer_end) o << ",\"layers\":[" << P.index.layer_begin << "," << P.index.layer_end << "],\"n_layers\":" << P.index.n_layers;
  o << ",\"shards\":[";
  for (size_t i = 0; i < P.index.shards.size(); ++i) o << (i ? "," : "") << "\"" << json_escape(P.index.shards[i]) << "\"";
  o << "],\"layouts\":[";
  for (size_t L = 0; L < P.placements.size(); ++L) {
    o << (L ? "," : "") << "{\"pool_bytes\":" << P.pool_bytes[L] << ",\"tensors\":[";
    for (size_t i = 0; i < P.placements[L].size(); ++i) {
      const Placement& p = P.placements[L][i];
      const DtypeInfo* di = dtype_info(p.dtype);
      o << (i ? "," : "") << "{\"name\":\"" << json_escape(P.index.tensors[i].name) << "\",\"dtype\":\"" << (di ? di->name : "?")
        << "\",\"shape\":[";
      for (size_t d = 0; d < p.shape.size(); ++d) o << (d ? "," : "") << p.shape[d];
      o << "],\"pool_offset\":" << p.pool_offset << ",\"nbytes\":" << p.nbytes << ",\"slice_dim\":";
      if (p.slice_dim == kNoSlice) o << "null";
      else o << p.slice_dim;
      o << ",\"slice_begin\":" << p.slice_begin << "}";
    }
    o << "]}";
  }
  o << "],\"parts\":[";
  for (size_t g = 0; g < P.parts.size(); ++g) {
    const PartPlan& pp = P.parts[g];
    o << (g ? "," : "") << "{\"src_bytes\":" << pp.src_bytes << ",\"out_bytes\":" << pp.out_bytes << ",\"chunks\":[";
    for (size_t c = 0; c < pp.chunks.size(); ++c) {
      const Chunk& ch = pp.chunks[c];
      o << (c ? "," : "") << "{\"shard\":" << ch.shard << ",\"buf_bytes\":" << ch.buf_bytes << ",\"n_tiles\":" << ch.n_tiles
        << ",\"src_bytes\":" << ch.src_bytes << ",\"out_bytes\":" << ch.out_bytes << ",\"reads\":[";
      for (size_t r = 0; r < ch.reads.size(); ++r)
        o << (r ? "," : "") << "[" << ch.reads[r].file_off << "," << ch.reads[r].len << "," << ch.reads[r].buf_off << "]";
      o << "],\"segs\":[";
      for (uint32_t s = 0; s < ch.seg_count; ++s) {
        const KKSeg& sg = pp.segs[ch.seg_begin + s];
        o << (s ? "," : "") << "{\"src_off\":" << sg.src_off << ",\"dst_off\":" << sg.dst_off << ",\"units\":" << sg.units
          << ",\"op\":" << sg.op << ",\"tile_begin\":" << sg.tile_begin << ",\"p0\":" << sg.p0 << ",\"p1\":" << sg.p1
          << ",\"p2\":" << sg.p2 << ",\"p3\":" << sg.p3 << "}";
      }
      o << "]}";
    }
    o << "]}";
  }
  o << "]}";
  return o.str();
}

}  // namespace kk
