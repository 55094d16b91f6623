// Load planning: decides where every tensor lives in the pool, which op moves it, and how the
// checkpoint's bytes are cut into staging chunks per ingesting rank.  Pure host code.
#include "kk_plan.hpp"

#include <algorithm>
#include <cstring>
#include <sstream>

#include "kk_json.hpp"

namespace kk {

namespace {

bool ends_with(const std::string& s, const char* suf) {
  size_t n = strlen(suf);
  return s.size() >= n && memcmp(s.data() + s.size() - n, suf, n) == 0;
}
bool contains(const std::string& s, const char* sub) { return s.find(sub) != std::string::npos; }

// KK_LOAD_GPT2_CONV1D_T applies to t: a GPT-2 Conv1D weight ([in, out]) of a dtype the transposes move, in a load that does not scatter.
bool transposed(const TensorRec& t, uint32_t flags, int mode) {
  if (!(flags & KK_LOAD_GPT2_CONV1D_T) || mode == KK_MODE_SCATTER || t.shape.size() != 2) return false;
  if (!ends_with(t.name, "attn.c_attn.weight") && !ends_with(t.name, "attn.c_proj.weight") && !ends_with(t.name, "mlp.c_fc.weight") &&
      !ends_with(t.name, "mlp.c_proj.weight"))
    return false;
  switch (t.dtype) {
    case KK_F32: case KK_F16: case KK_BF16: case KK_I16: case KK_U16: case KK_I32: case KK_U32: return true;
    default: return false;
  }
}

struct OpInfo {
  uint32_t op;
  uint32_t pool_dtype;
  uint64_t src_unit_bytes;  // source bytes per op unit (a transpose's unit is one source row)
  uint64_t out_unit_bytes;  // pool bytes per op unit
  uint64_t tile_units;      // op units per tile (split granule)
};

// The op that moves tensor t (tr: transposed, see transposed()).  Every float output is bf16, or fp16 under KK_LOAD_F16 (out): the op codes
// are the same, the launch's output format (KK_LAUNCH_F16) picks the kernel.  Under it the 16-bit roles swap: F16 is the verbatim copy and
// BF16 takes the 16-bit cast.
OpInfo op_for(const TensorRec& t, uint32_t flags, bool tr) {
  const uint32_t dt = t.dtype;
  const uint32_t out = (flags & KK_LOAD_F16) ? KK_F16 : KK_BF16;
  const bool cast32 = dt == KK_F32 && !(flags & KK_LOAD_KEEP_F32), cast16 = (dt == KK_F16 || dt == KK_BF16) && dt != out;
  if (tr) {
    const uint64_t R = t.shape[0], C = t.shape[1], es = dtype_info(dt)->block_bytes;  // 2 or 4 for every transposed dtype
    if (R > 0xFFFFFFFFull || C > 0xFFFFFFFFull) fail(KK_EUNSUPPORTED, "tensor %s too large to transpose", t.name.c_str());
    const uint32_t op = cast32 ? KK_OP_T_F32_BF16 : cast16 ? KK_OP_T_F16_BF16 : es == 4 ? KK_OP_T_B32 : KK_OP_T_B16;
    return {op, cast32 || cast16 ? out : dt, C * es, C * (cast32 ? 2 : es), KK_T_ROWS};
  }
  if (cast32) return {KK_OP_F32_BF16, out, 4, 2, KK_TILE_SRC_BYTES / 4};
  if (cast16) return {KK_OP_F16_BF16, out, 2, 2, KK_TILE_SRC_BYTES / 2};
  if (flags & KK_LOAD_F8_TO_BF16) {
    if (dt == KK_F8_E4M3) return {KK_OP_F8E4M3_BF16, out, 1, 2, KK_TILE_SRC_BYTES};
    if (dt == KK_F8_E5M2) return {KK_OP_F8E5M2_BF16, out, 1, 2, KK_TILE_SRC_BYTES};
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
  if (!di) fail(KK_EINVAL, "tensor %s: unknown dtype %u", t.name.c_str(), dt);
  if (di->block_elems > 1 && dt >= 32)
    fail(KK_EUNSUPPORTED, "tensor %s: %s -> bf16 dequantisation is not implemented (every GGUF weight type except Q8_K / Q8_1 is)", t.name.c_str(), di->name);
  return {KK_OP_COPY, dt, 1, 1, KK_TILE_SRC_BYTES};  // verbatim bytes: the output format's own 16-bit floats, F32 under KEEP_F32, integers, ...
}

// Which dimension a tensor is sliced along in SCATTER mode (kNoSlice = replicate). [PROPOSED] rule of
// SURVEY.md §8(a3.S5): column-parallel weights along dim 0, row-parallel weights along dim 1.
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

// Source bytes that one op moves into one pool range, cut into steps: op units read as one contiguous range (stride 0), or runs of a slice
// read one by one, stride apart in the file.  A chunk takes whole steps; a piece split across chunks becomes one segment per chunk, each a
// copy of seg that starts done units into the piece.
struct Piece {
  uint32_t shard;
  uint64_t file_off;    // first source byte
  uint64_t step_bytes;  // source bytes per step
  uint64_t steps;
  uint64_t stride;      // 0: contiguous; else the file distance between runs
  uint64_t granule;     // steps per split: the op's tile units, or 16 runs
  uint64_t step_units;  // segment units per step
  KKSeg seg;            // the segments' op, dst_off and p0..p3
  uint32_t KKSeg::*done;  // the field that counts the units done (a transpose's p2, the row exchange's p3); nullptr: they advance dst_off
  uint64_t unit_out;    // pool bytes each unit accounts for
};

// Sets pc to read n_runs runs of run_bytes, stride apart, from file_off.  One run is read contiguously and split on the op's tiles; more
// runs are read one by one and split on 16 runs.
void set_runs(Piece& pc, const OpInfo& oi, uint64_t file_off, uint64_t run_bytes, uint64_t n_runs = 1, uint64_t stride = 0) {
  pc.file_off = file_off;
  if (n_runs == 1) {
    pc.step_bytes = oi.src_unit_bytes;
    pc.steps = oi.src_unit_bytes ? run_bytes / oi.src_unit_bytes : 0;  // a transposed [R, 0] tensor's rows are empty: nothing to move
    pc.stride = 0;
    pc.granule = oi.tile_units;
    pc.step_units = 1;
  } else {
    pc.step_bytes = run_bytes;
    pc.steps = n_runs;
    pc.stride = stride;
    pc.granule = 16;
    pc.step_units = run_bytes / oi.src_unit_bytes;
  }
}

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
  // Reserves room for n reads of len bytes, stride apart from file_off, packed back to back in the buffer; returns the buffer offset of
  // the first.  A contiguous read (stride 0) joins the previous read when the two are adjacent in the file and in the buffer; the runs of
  // a strided piece always open a new 16-byte aligned read, so the segment's src_off stays aligned.
  uint64_t add_reads(uint64_t file_off, uint64_t len, uint64_t n, uint64_t stride) {
    cur.src_bytes += n * len;
    if (!stride && !cur.reads.empty()) {
      ReadOp& l = cur.reads.back();
      if (l.file_off + l.len == file_off && l.buf_off + l.len == pos) {
        l.len += len;
        pos += len;
        return pos - len;
      }
    }
    const uint64_t at = align_up(pos, 16);
    for (uint64_t r = 0; r < n; ++r) cur.reads.push_back({file_off + r * stride, len, at + r * len});
    pos = at + n * len;
    return at;
  }
  void add_seg(const Piece& pc, uint64_t src_off, uint64_t units, uint64_t units_done) {
    KKSeg s = pc.seg;
    s.src_off = src_off;
    s.units = units;
    s.tile_begin = cur.n_tiles;
    if (pc.done) s.*pc.done = (uint32_t)units_done;
    else s.dst_off += units_done * pc.unit_out;
    cur.out_bytes += units * pc.unit_out;
    uint64_t nt = kk_seg_tiles(s.op, s.units, s.p0);
    if (nt + cur.n_tiles > 0xFFFFFFF0ull) fail(KK_EUNSUPPORTED, "chunk has too many tiles");
    cur.n_tiles += (uint32_t)nt;
    cur.seg_count++;
    pp.segs.push_back(s);
  }

  void emit(const Piece& pc) {
    if (pc.steps == 0) return;
    if (open && cur.shard != pc.shard) flush();
    if (!open) begin(pc.shard);
    for (uint64_t done = 0; done < pc.steps;) {
      if (cur.seg_count >= kMaxSegsPerChunk) { flush(); begin(pc.shard); }
      const uint64_t start = align_up(pos, 16);
      const uint64_t fit = cap > start ? (cap - start) / pc.step_bytes : 0;
      const uint64_t rem = pc.steps - done;
      const uint64_t take = fit >= rem ? rem : fit / pc.granule * pc.granule;
      if (take == 0) {
        if (cur.seg_count == 0)
          fail(KK_EINVAL, "staging buffer (%llu B) smaller than %s", (unsigned long long)cap, pc.stride ? "16 slice rows" : "one tile");
        flush();
        begin(pc.shard);
        continue;
      }
      const uint64_t at = pc.stride ? add_reads(pc.file_off + done * pc.stride, pc.step_bytes, take, pc.stride)
                                    : add_reads(pc.file_off + done * pc.step_bytes, take * pc.step_bytes, 1, 0);
      add_seg(pc, at, take * pc.step_units, done * pc.step_units);
      done += take;
    }
  }

  static constexpr uint32_t kMaxSegsPerChunk = 1024;
};

// Pieces of a tensor whose rows llama.cpp interleaved per rotary half (TensorRec::rope_heads), for HF rows [r0, r1) of it with HF row r0 at
// whole's destination.  HF row h*hd + k*hd/2 + i is file row h*hd + 2i + k, so the rows of one (head, half) group are one strided run of file
// rows.  The pieces come in HF row order and tile [r0, r1) exactly: destination offsets never decrease in plan order (a part stays one pool
// range) and every pool byte of the slice is written once.  A slice boundary may cut a group (scatter does not need heads % ranks == 0).
void unpermuted_pieces(const TensorRec& t, const OpInfo& oi, const Piece& whole, uint64_t r0, uint64_t r1, std::vector<Piece>& out) {
  const uint64_t R = t.shape[0], half = R / t.rope_heads / 2, row_bytes = t.nbytes / R;
  const uint64_t row_units = row_bytes / oi.src_unit_bytes, out_row = row_units * oi.out_unit_bytes;
  if (row_bytes * R != t.nbytes || row_units * oi.src_unit_bytes != row_bytes || row_units == 0)  // to_hf_layout refuses such tensors
    fail(KK_EUNSUPPORTED, "KK_LOAD_HF_LAYOUT: tensor %s: a row is not a whole number of source units", t.name.c_str());
  for (uint64_t g = r0 / half; g * half < r1; ++g) {
    const uint64_t a = std::max(r0, g * half), b = std::min(r1, (g + 1) * half);
    const uint64_t head = g / 2, k = g % 2, i0 = a - g * half;
    Piece pc = whole;
    set_runs(pc, oi, t.file_offset + (head * 2 * half + 2 * i0 + k) * row_bytes, row_bytes, b - a, 2 * row_bytes);
    pc.seg.dst_off = whole.seg.dst_off + (a - r0) * out_row;
    // the consumers store whole 16-byte vectors from a segment's first output on
    if (pc.seg.dst_off % 16 != 0)
      fail(KK_EUNSUPPORTED, "KK_LOAD_HF_LAYOUT: tensor %s: HF row %llu would start at pool offset %llu, off a 16-byte boundary (%llu B per row)",
           t.name.c_str(), (unsigned long long)a, (unsigned long long)pc.seg.dst_off, (unsigned long long)out_row);
    out.push_back(pc);
  }
}

// Places tensor t at pool offset off of layout L (a SCATTER rank, else 0) and appends the pieces that fill its slot.
Placement place(const Plan& P, const TensorRec& t, int L, uint64_t off, std::vector<Piece>& pieces) {
  const bool tr = transposed(t, P.flags, P.mode);
  const OpInfo oi = op_for(t, P.flags, tr);
  Placement p;
  p.dtype = oi.pool_dtype;
  p.shape = t.shape;
  p.pool_offset = off;
  p.slice_dim = P.mode == KK_MODE_SCATTER ? scatter_slice_dim(t, P.n_parts) : kNoSlice;
  Piece pc{};
  pc.shard = t.shard;
  pc.seg.op = oi.op;
  pc.seg.dst_off = off;
  pc.unit_out = oi.out_unit_bytes;
  set_runs(pc, oi, t.file_offset, t.nbytes);  // the whole tensor
  const uint64_t n = (uint64_t)P.n_parts;
  if (tr) {
    p.shape = {t.shape[1], t.shape[0]};
    pc.seg.p0 = (uint32_t)t.shape[1];  // C
    pc.seg.p1 = (uint32_t)t.shape[0];  // R
    pc.done = &KKSeg::p2;              // source rows already transposed
  } else if (p.slice_dim == 0) {
    const uint64_t rows = t.shape[0] / n, row_bytes = t.nbytes / t.shape[0];  // whole rows (also for block-quantised types)
    p.slice_begin = rows * (uint64_t)L;
    p.shape[0] = rows;
    set_runs(pc, oi, t.file_offset + p.slice_begin * row_bytes, rows * row_bytes);
  } else if (p.slice_dim == 1) {
    const uint64_t R = t.shape[0], C = t.shape[1], cols = C / n, es = dtype_info(t.dtype)->block_bytes;
    const uint64_t row_bytes = C * es, slice_bytes = cols * es;
    p.slice_begin = cols * (uint64_t)L;
    p.shape[1] = cols;
    const bool exchange = (P.flags & KK_LOAD_SCATTER_EXCHANGE) && oi.op == KK_OP_COPY && row_bytes <= 0xFFFFFFFFull && R <= 0xFFFFFFFFull &&
                          (R / n + n) * row_bytes < 0xFFFFFFFFull;
    if (exchange) {
      // this rank ingests whole rows [r0, r1) and the kernel deals column slice j of every row to pool j
      const uint64_t r0 = R / n * (uint64_t)L, r1 = (L == P.n_parts - 1) ? R : R / n * (uint64_t)(L + 1);
      set_runs(pc, oi, t.file_offset + r0 * row_bytes, (r1 - r0) * row_bytes);
      pc.seg.op = KK_OP_ROWSPLIT;
      pc.seg.p0 = (uint32_t)row_bytes;
      pc.seg.p1 = (uint32_t)slice_bytes;
      pc.seg.p2 = (uint32_t)r0;
      pc.done = &KKSeg::p3;  // bytes of the rows already dealt
      p.nbytes = R * slice_bytes;
      pieces.push_back(pc);
      return p;
    }
    set_runs(pc, oi, t.file_offset + p.slice_begin * es, slice_bytes, R, row_bytes);
  }
  p.nbytes = pc.steps * pc.step_units * pc.unit_out;
  if (t.rope_heads && p.nbytes) {  // the same slot, filled in HF row order (a dim-0 slice keeps HF rows)
    const uint64_t r0 = p.slice_dim == 0 ? p.slice_begin : 0;
    unpermuted_pieces(t, oi, pc, r0, r0 + p.shape[0], pieces);
  } else {
    pieces.push_back(pc);
  }
  return p;
}

}  // namespace

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
  std::vector<std::vector<Piece>> pieces((size_t)n_layouts);  // pieces[layout], in pool order
  for (int L = 0; L < n_layouts; ++L) {
    auto& pl = P.placements[(size_t)L];
    pl.reserve(T.size());
    uint64_t off = 0;
    for (auto& t : T) {
      pl.push_back(place(P, t, L, off, pieces[(size_t)L]));
      off = align_up(off + pl.back().nbytes, KK_POOL_ALIGN);
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
