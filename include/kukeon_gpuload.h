/*
 * kukeon_gpuload.h — C ABI of libkukeon_gpuload.so, the model-hub weight loader for NVIDIA H100 (sm_90a).
 *
 * This is the drop-in boundary of the hot path named by BASELINE.json's north_star: kukeond keeps a Go
 * API (modelhub.Pull / Load / Mount, gpupool, the Cell hooks) and every one of those calls bottoms
 * out in one of the functions below through cgo.  The reference (eminwux/kukeon @ 4be245a) has NO
 * loader and NO FFI today (SURVEY.md §0), so each entry point cites the nearest reference seam it
 * would be bound next to rather than a function it replaces:
 *
 *   kk_open / kk_close      pool lifetime == daemon lifetime.  internal/daemon/server.go:87 (NewServer)
 *                           and :242 (Stop); options threaded like runner.Options, runner/runner.go:173-194.
 *   kk_index                modelhub.Pull [NOT IN REFERENCE].  Nearest analogue: OCI image pull,
 *                           internal/ctr/image.go:91-157.  CPU only; no device is touched.
 *   kk_load / kk_load_ex    modelhub.Load [NOT IN REFERENCE].  Nearest analogue: ctr.LoadImage,
 *                           internal/ctr/image.go:166-188.  Called from runner.StartCell beside
 *                           attachableBuildOpts, internal/controller/runner/start.go:785-790 and
 *                           provision.go:1560-1570.
 *   kk_export               modelhub.Mount [NOT IN REFERENCE].  The manifest it renders is staged the way
 *                           secrets are (internal/ctr/secrets.go:105-127) and bind-mounted read-only through a
 *                           ctr.BuildOption (internal/ctr/spec.go:176), env named like kukeonDefaultEnv
 *                           (internal/ctr/spec.go:464-482).
 *   kk_acquire / kk_release per-Cell refcount ("N concurrent Sessions share one HBM copy").  Acquire in
 *                           StartCell (runner/start.go:252); release in KillCell (runner/kill.go:31),
 *                           StopCell (runner/stop.go:34), DeleteCell (runner/delete_cell.go:33).
 *   kk_last_error           errors surface as Go sentinels wrapped with %w, internal/errdefs/errdefs.go:23-.
 *
 * Contract (SURVEY.md §8(b)):
 *   - every function returns 0 (KK_OK) or a negative kk_status; kk_last_error() returns a thread-local,
 *     NUL-terminated description valid until the next failing call on the same thread;
 *   - no C++ exception crosses the boundary; all entry points are thread-safe (kukeond serves one
 *     goroutine per connection, internal/daemon/server.go:236, so calls arrive on arbitrary OS threads);
 *   - the caller owns every input buffer and every out-struct it passes; the library owns device memory,
 *     pinned buffers, streams and opaque handles until the matching kk_release / kk_close;
 *   - plain pointers and sizes only: no torch, no C++ types;
 *   - there is NO CPU fallback: a load on a machine without a usable CUDA device fails with KK_ECUDA.
 */
#ifndef KUKEON_GPULOAD_H
#define KUKEON_GPULOAD_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KK_ABI_VERSION 1
#define KK_MAX_DEVICES 8
#define KK_MAX_DIMS 8
#define KK_NAME_MAX 256
#define KK_IPC_HANDLE_BYTES 64 /* sizeof(cudaIpcMemHandle_t) */
#define KK_POOL_ALIGN 256      /* every tensor slot in a pool starts on a 256-byte boundary */

typedef enum kk_status {
  KK_OK = 0,
  KK_EINVAL = -1,       /* bad argument (NULL, out of range, unknown enum) */
  KK_ENOENT = -2,       /* path / shard / tensor not found */
  KK_EFORMAT = -3,      /* malformed safetensors / GGUF / index.json */
  KK_EIO = -4,          /* open/read failed or short read */
  KK_ENOMEM = -5,       /* host or device allocation failed, or pool budget exceeded */
  KK_ECUDA = -6,        /* CUDA runtime/driver error, or no usable device */
  KK_EUNSUPPORTED = -7, /* dtype / mode / fan-out not supported on this build or machine */
  KK_EBUSY = -8,        /* object still referenced */
  KK_ERANGE = -9,       /* caller buffer too small; required size is reported where documented */
  KK_ESTATE = -10       /* call not valid in the object's current state */
} kk_status;

/* File dtypes.  0..19 follow safetensors' Dtype enum order; 32.. are GGUF block-quantised types. */
typedef enum kk_dtype {
  KK_BOOL = 0, KK_F4 = 1, KK_F6_E2M3 = 2, KK_F6_E3M2 = 3, KK_U8 = 4, KK_I8 = 5, KK_F8_E5M2 = 6,
  KK_F8_E4M3 = 7, KK_F8_E8M0 = 8, KK_I16 = 9, KK_U16 = 10, KK_F16 = 11, KK_BF16 = 12, KK_I32 = 13,
  KK_U32 = 14, KK_F32 = 15, KK_C64 = 16, KK_F64 = 17, KK_I64 = 18, KK_U64 = 19,
  KK_Q4_0 = 32, KK_Q4_1 = 33, KK_Q5_0 = 34, KK_Q5_1 = 35, KK_Q8_0 = 36, KK_Q2_K = 37, KK_Q3_K = 38,
  KK_Q4_K = 39, KK_Q5_K = 40, KK_Q6_K = 41, KK_Q8_K = 42, KK_IQ4_NL = 43, KK_IQ4_XS = 44, KK_MXFP4 = 45,
  KK_IQ2_XXS = 46, KK_IQ2_XS = 47, KK_IQ2_S = 48, KK_IQ3_XXS = 49, KK_IQ3_S = 50, KK_IQ1_S = 51, KK_IQ1_M = 52, KK_TQ1_0 = 53, KK_TQ2_0 = 54, KK_NVFP4 = 55
} kk_dtype;

typedef enum kk_mode {
  KK_MODE_SINGLE = 0,    /* whole checkpoint into the pool of devices[0] */
  KK_MODE_BROADCAST = 1, /* every device ends with the whole pool: sharded ingest + fused P2P fan-out */
  KK_MODE_SCATTER = 2    /* device g keeps only its slice (dim0 for column-parallel, dim1 for row-parallel) */
} kk_mode;

typedef enum kk_fanout {
  KK_FANOUT_P2P = 0,  /* convert kernel stores every output vector to all peer-mapped pools (NVLink/NVSwitch) */
  KK_FANOUT_NVLS = 1, /* BROADCAST, one process owning >= 2 devices: the pools are VMM allocations bound to one NVSwitch multicast object and the
                         convert kernel stores every vector once with multimem.st.  KK_EUNSUPPORTED where the host does not expose NVLS, for
                         checkpoints with tensors that are not whole 16-byte vectors, and for kk_export's IPC handle (VMM memory has none):
                         the comparison the north_star names, not the default (an all-gather is ingress-bound either way) */
  KK_FANOUT_NONE = 2, /* local pool only; the caller runs its own collective (e.g. the NCCL comparison) */
  KK_FANOUT_RAW = 3,  /* BROADCAST only: all-gather the *file* bytes (e.g. q4_K blocks, 3.56x smaller than their bf16)
                         into a per-device raw image over NVLink, then every device converts everything locally */
  KK_FANOUT_PULL = 4  /* BROADCAST, one process per GPU only: every rank converts its part into its own pool AND into a slice buffer
                         (its 1/N of the pool, a separate allocation); peers map only the slice buffers — 1/N of the bytes a pool
                         mapping costs, which is what dominates time-to-ready in that deployment — and kk_convert_local pulls them
                         into the local pool with bulk loads over NVLink.  Same NVLink bytes as the push order. */
} kk_fanout;

/* kk_config.flags */
#define KK_CFG_ZEROCOPY 0x1u     /* convert kernels read the pinned host ring directly (no H2D copy engine hop) */
#define KK_CFG_NO_PEER_ACCESS 0x2u /* do not enable peer access between devices (forces replicas) */
#define KK_CFG_PEER_ALL 0x8u       /* kk_open enables peer access from the context's devices to EVERY visible GPU (one-rank-
                                      per-GPU deployments: moves the one-time peer setup out of the first kk_peer_attach) */
#define KK_CFG_NO_NUMA_PIN 0x4u    /* do not bind reader threads / pinned slots to the device's NUMA node */
#define KK_CFG_VMM_POOLS 0x10u     /* allocate pools with the driver's virtual-memory API (cuMemCreate) instead of cudaMalloc.  Such a pool is exported as a
                                      POSIX file descriptor (kk_export_fd) which the consumer maps READ-ONLY (kk_import_fd): agent cells that share one
                                      HBM copy can then not overwrite it.  A cudaIpcMemHandle (kk_export) always maps read-write in the opener — use VMM
                                      pools whenever the cells mounting a model do not trust each other.  Not available for one-process-per-GPU
                                      fan-out (kk_peer_attach takes IPC handles) */

/* kk_load_opts.flags */
#define KK_LOAD_GPT2_CONV1D_T 0x1u /* transpose HF GPT-2 Conv1D weights ([in,out] -> [out,in]) while loading */
#define KK_LOAD_KEEP_F32 0x2u      /* keep F32 tensors as F32 in the pool (default: convert to bf16) */
#define KK_LOAD_DEFER 0x4u         /* index + plan + allocate pools only; data moves on kk_load_part */
#define KK_LOAD_SCATTER_EXCHANGE 0x8u /* KK_MODE_SCATTER: row-parallel (dim-1 sliced) tensors are ingested as whole rows by
                                      the rank owning 1/N of the rows and split across the N pools by the kernel over NVLink
                                      (an all-to-all through NVSwitch) instead of every rank gathering 2-7 KB column runs
                                      from the file; needs peer access (one process) or attached peers (kk_peer_attach) */

#define KK_LOAD_F8_TO_BF16 0x10u    /* widen safetensors F8_E4M3 / F8_E5M2 tensors to bf16 (exact; NaN -> 0x7FFF).  Default: FP8 stays
                                      verbatim in the pool — FP8 engines want the bytes, and the per-block scale tensors that FP8
                                      checkpoints carry are model-specific and are not applied here */
/* 0x20 and 0x40 selected round 1's two candidate transpose geometries; the 8-row tiles won the A/B and are what KK_LOAD_GPT2_CONV1D_T uses now */
#define KK_LOAD_F16 0x80u           /* store every float output as IEEE binary16 (KK_F16) instead of bf16.  The pool's layout, sizes and
                                      offsets are exactly those of the same load without the flag; only the dtype of the float tensors differs:
                                        F16                 verbatim (a copy: NaN payloads kept byte for byte)
                                        BF16                cast to f16: round to nearest even, overflow -> +-inf, f16 subnormals kept
                                        F32                 cast to f16 likewise (still F32 under KK_LOAD_KEEP_F32)
                                        GGUF block types    the same fp32 arithmetic as the bf16 load, then one RNE rounding to f16
                                        F8_E4M3 / F8_E5M2   verbatim; f16 under KK_LOAD_F8_TO_BF16 (exact, the hardware's FP8 -> f16 pair conversion)
                                        GPT-2 transposes    F32 / BF16 -> f16, F16 moved verbatim
                                        integers, bool, F64, sub-byte: verbatim
                                      Every NaN a conversion produces is 0x7FFF.  Composes with every mode, fan-out, KK_LOAD_DEFER, parts,
                                      pipeline stages and VMM pools.  KK_LOAD_SCATTER_EXCHANGE keeps applying to the tensors the pool holds byte
                                      for byte, so under this flag an F16 checkpoint's row-parallel tensors use the exchange and a BF16
                                      checkpoint's are gathered (as F32 tensors are).  Flags are part of a model's identity: an f16 and a bf16
                                      load of one file are two models. */
#define KK_LOAD_HF_LAYOUT 0x100u    /* GGUF checkpoints only: load the checkpoint in Hugging Face layout, as transformers' safetensors files have it.
                                      The load sees the HF view of the file before it plans, and every other flag, mode, fan-out, DEFER, parts,
                                      pipeline stage (over the HF names) and VMM pools apply to that view unchanged.  Placements, kk_model_tensor,
                                      kk_model_get_info and the manifest speak HF names and shapes only (a GGUF name is KK_ENOENT); the manifest
                                      and kk_plan_describe add "layout":"hf" and "architecture".
                                        names        token_embd -> model.embed_tokens, output_norm -> model.norm, output -> lm_head,
                                                     blk.N.attn_norm -> model.layers.N.input_layernorm, blk.N.ffn_norm -> .post_attention_layernorm,
                                                     blk.N.attn_{q,k,v} -> .self_attn.{q,k,v}_proj, blk.N.attn_output -> .self_attn.o_proj,
                                                     blk.N.attn_{q,k}_norm -> .self_attn.{q,k}_norm (qwen3), blk.N.ffn_{gate,up,down} ->
                                                     .mlp.{gate,up,down}_proj, blk.N.ffn_gate_inp -> .block_sparse_moe.gate (llama); each keeps
                                                     its .weight / .bias; rope_freqs.weight keeps its name (HF engines compute it from the config)
                                        experts      (llama) blk.N.ffn_{gate,up,down}_exps.weight [E, r, c] -> E tensors
                                                     model.layers.N.block_sparse_moe.experts.e.{w1,w3,w2}.weight [r, c], expert e being bytes
                                                     [e * nbytes / E, (e + 1) * nbytes / E) of the stack
                                        Q / K rows   (llama: Llama, Mistral, Mixtral) llama.cpp's converter interleaves the two rotary halves of
                                                     every head of q_proj / k_proj (weight and bias); the load un-permutes them while staging:
                                                     HF row h*hd + k*hd/2 + i is file row h*hd + 2i + k, with head count
                                                     <arch>.attention.head_count for q and .head_count_kv (default: head_count) for k and
                                                     hd = rows / heads.  qwen2 / qwen3 use NEOX rotary and are not permuted.
                                      Architectures (general.architecture): llama, qwen2, qwen3; any other is KK_EUNSUPPORTED, and so is any
                                      tensor the table does not map (nothing is dropped).  KK_EINVAL on a safetensors checkpoint; KK_EFORMAT
                                      when a needed metadata key is missing or ill-typed (integers: any GGUF integer type in 1..65535; a
                                      per-layer array is KK_EUNSUPPORTED) or Q/K rows are not a multiple of 2 * heads; KK_EUNSUPPORTED when a
                                      Q/K row is not whole blocks of its type (a 1-D block-quantised bias) or a Q/K (head, half) row group would
                                      start off a 16-byte pool boundary.  Split GGUFs: the keys are the first shard's; a later shard that repeats
                                      one must agree (KK_EFORMAT).  All are raised before any device
                                      is touched.  Costs: Q/K rows are read one row per read and stage as (head, half) pieces. */

typedef struct kk_ctx kk_ctx;     /* one per process (kukeond lifetime) */
typedef struct kk_model kk_model; /* refcounted; one per (checkpoint identity, mode, flags, layer range) */

typedef struct kk_config {
  int32_t n_devices;                /* 1..KK_MAX_DEVICES */
  int32_t devices[KK_MAX_DEVICES];  /* CUDA ordinals */
  uint64_t pool_bytes_per_device;   /* budget across all resident models; 0 = no limit */
  uint32_t n_staging_buffers;       /* pinned ring slots per device; 0 = default (2 per reader thread) */
  uint64_t staging_buffer_bytes;    /* bytes per slot; 0 = default (16 MiB); rounded up to 2 MiB */
  uint32_t n_reader_threads;        /* host reader threads per device; 0 = default (16) */
  uint32_t flags;                   /* KK_CFG_* */
} kk_config;

typedef struct kk_tensor_meta {
  char name[KK_NAME_MAX];
  uint32_t dtype;             /* kk_dtype as stored in the file */
  uint32_t n_dims;
  uint64_t shape[KK_MAX_DIMS]; /* row-major, outermost first (GGUF ne[] is reversed into this order) */
  uint32_t shard;             /* index into the shard list (kk_index_shard) */
  uint32_t reserved;
  uint64_t file_offset;       /* absolute byte offset of the tensor's data inside its shard file */
  uint64_t nbytes;            /* bytes in the file */
} kk_tensor_meta;

typedef struct kk_placement {
  int32_t device;             /* CUDA ordinal */
  uint32_t dtype;             /* dtype in the pool (KK_BF16 for every float tensor by default, KK_F16 under KK_LOAD_F16; KK_F32 under KK_LOAD_KEEP_F32) */
  uint64_t pool_offset;       /* byte offset inside that device's pool, multiple of KK_POOL_ALIGN */
  uint64_t nbytes;            /* bytes in the pool */
  uint32_t n_dims;
  uint32_t slice_dim;         /* KK_MODE_SCATTER: dimension sliced, or 0xFFFFFFFF when replicated/whole */
  uint64_t shape[KK_MAX_DIMS]; /* shape in the pool (after transpose / slice) */
  uint64_t slice_begin;       /* first index kept along slice_dim (0 when not sliced) */
} kk_placement;

typedef struct kk_load_opts {
  int32_t mode;      /* kk_mode */
  int32_t fanout;    /* kk_fanout */
  uint32_t flags;    /* KK_LOAD_* */
  /* Multi-process operation (one rank per GPU, e.g. under torchrun): this process ingests part
   * `part_index` of `part_count` of the checkpoint and, in BROADCAST mode, fans it out to the pools
   * attached with kk_peer_attach.  part_count <= 1 means "this process ingests everything its ctx's
   * devices need". In SCATTER mode part_index/part_count select which slice this rank keeps. */
  int32_t part_index;
  int32_t part_count;
  /* Pipeline stage: load only layers [layer_begin, layer_end) of the checkpoint.  layer_end == 0 loads the whole checkpoint.
   * A stage is a model of its own (a context may hold several stages of one file); kk_plan_describe takes the same range.
   * The range is part of the model's identity as given: [0, n_layers) holds the same tensors as the whole checkpoint but is a
   * separate model (its own pool, and a manifest with the stage keys), so a caller should use one form per checkpoint.
   *   - The layer of a tensor is N in its first dotted component pair "<container>.<N>." with <container> one of layers / h / blk
   *     and N all digits (model.layers.3.mlp.up_proj.weight, transformer.h.0.attn.c_attn.weight, blk.7.ffn_down_exps.weight).
   *     The checkpoint has n_layers = 1 + the largest N.  Every layered tensor must belong to one stack (the same text up to and
   *     including "<container>.") — two numbered stacks, e.g. model.layers. and vision_tower.encoder.layers., are KK_EUNSUPPORTED.
   *   - A layered tensor is kept iff layer_begin <= N < layer_end.  Tensors without a layer go by name suffix:
   *     embed_tokens.weight, token_embd.weight, wte.weight, wpe.weight to the first stage (layer_begin == 0);
   *     lm_head.weight, lm_head.bias, the name output.weight, *norm.weight, *norm.bias, ln_f.weight, ln_f.bias to the last stage
   *     (layer_end == n_layers); with no lm_head.weight and no output.weight (tied embeddings) the token embedding (not wpe)
   *     goes to the last stage as well; every other tensor (e.g. rope_freqs.weight) to every stage.
   *   - KK_EINVAL: layer_begin != 0 with layer_end == 0, layer_begin >= layer_end, layer_end > n_layers.  KK_EUNSUPPORTED: a range
   *     on a checkpoint without layered tensors.  All are raised before any device is touched.
   * The stage's tensors then load exactly as a checkpoint of only those tensors would, in every mode, fan-out and flag: shards and
   * file offsets are unchanged, and no byte outside the stage is read.  Deployments: one process per GPU passes its stage plus its
   * part_index / part_count within the stage's group and attaches that group's peers only; one process opens one kk_ctx per stage
   * group, over disjoint devices. */
  uint32_t layer_begin;
  uint32_t layer_end;
  uint32_t reserved;
} kk_load_opts;

typedef struct kk_model_info {
  uint64_t n_tensors;
  uint64_t n_shards;
  uint64_t file_bytes;   /* sum of tensor bytes in the files */
  uint64_t pool_bytes;   /* bytes of one device's pool (max over devices for SCATTER) */
  int32_t n_devices;
  int32_t devices[KK_MAX_DEVICES];
  int32_t mode;
  int32_t refcount;
  int32_t loaded;        /* 1 once every pool holds its data */
  int32_t reserved;
} kk_model_info;

/* ---- lifecycle ------------------------------------------------------------------------------ */
int kk_abi_version(void);
const char* kk_last_error(void);
const char* kk_status_name(int status);

int kk_open(const kk_config* cfg, kk_ctx** out);
int kk_close(kk_ctx* ctx); /* KK_EBUSY while any model is still referenced */

/* ---- Pull: index a checkpoint (CPU only; ctx may be NULL) ------------------------------------ */
/* path: a directory (model.safetensors.index.json | model.safetensors | *.gguf inside) or one file.
 * Records come back sorted by (shard, file_offset).  Free with kk_free_index. */
int kk_index(kk_ctx* ctx, const char* path, kk_tensor_meta** out, size_t* n);
int kk_free_index(kk_tensor_meta* recs);
/* Shard file names (absolute paths) of the last-level index of `path`; *n_out receives the count.
 * buf receives name `i`; returns KK_ERANGE if cap is too small. */
int kk_index_shard(kk_ctx* ctx, const char* path, size_t i, char* buf, size_t cap, size_t* n_out);

/* Describe, without touching a device, what a load would do: pool layout(s) and, per ingesting part, the
 * staging chunks (file reads) and conversion segments.  n_parts is the number of ingesting devices/ranks
 * (1 for KK_MODE_SINGLE), chunk_bytes the staging slot size (0 = default 64 MiB).  JSON into `json`;
 * KK_ERANGE (and *required) when cap is too small.  CPU only; ctx may be NULL. */
int kk_plan_describe(kk_ctx* ctx, const char* path, const kk_load_opts* opts, int n_parts, uint64_t chunk_bytes,
                     char* json, size_t cap, size_t* required);

/* ---- Load ------------------------------------------------------------------------------------ */
int kk_load(kk_ctx* ctx, const char* path, int mode, int fanout, kk_model** out);
int kk_load_ex(kk_ctx* ctx, const char* path, const kk_load_opts* opts, kk_model** out);
/* LoRA adapters.  kk_load_adapter loads `path` with `opts` exactly as kk_load_ex would, then merges the PEFT LoRA adapter at
 * `adapter_path` into the pool(s) on the GPU.  kk_adapter_describe (CPU only, ctx may be NULL) validates the adapter against the checkpoint
 * as that load would see it and describes the merge as JSON: per target its pool name, dtype, shape, r, scaling and the adapter tensors
 * used, plus the targets skipped by the stage.  KK_ERANGE / *required as kk_plan_describe.
 *   input     adapter_path is a directory holding adapter_config.json and adapter_model.safetensors, or that safetensors file with the
 *             config beside it (PEFT's save_pretrained form).
 *   names     base_model.model.<M>.lora_A.weight [r, C] and base_model.model.<M>.lora_B.weight [R, r] target pool tensor <M>.weight [R, C],
 *             matched against the names the load plans over (HF names under KK_LOAD_HF_LAYOUT).  A target that exists in the checkpoint
 *             but lies outside the load's layer stage is skipped; one that does not exist is KK_ENOENT.  Nothing is dropped silently.
 *   scaling   s = (float)(lora_alpha / r), or (float)(lora_alpha / sqrt(r)) under use_rslora, computed in double and rounded once; r is
 *             each pair's own (A's rows), so rank_pattern needs nothing.
 *   merge     for element (i, j) of the full tensor (a SCATTER slice's slice_begin offsets i for dim 0 or j for dim 1), w the pool element
 *             after the ordinary load widened to fp32, A and B widened exactly from their file dtype:
 *               acc = 0.0f; for k = 0 .. r-1: acc = fmaf(B[i][k], A[k][j], acc)   (this order, no split-K; CUDA-core FFMA)
 *               out = fmaf(s, acc, w) rounded to nearest even into the pool dtype (bf16 / f16 overflow -> inf, f32 as is); any NaN -> 0x7FFF
 *                     (0x7FFFFFFF in an F32 pool); subnormals are kept
 *             Bytes outside the targets are untouched, and the pool layout (placements, offsets, sizes, dtypes) is that of the same load
 *             without the adapter.  The pool dtype follows the load: bf16, KK_LOAD_F16, KK_LOAD_KEEP_F32 and GGUF block types dequantised first.
 *   when      at the end of kk_load_adapter (one process: after the fan-out or RAW stage 2 on every pool) and, for a KK_LOAD_DEFER model, at the
 *             end of every kk_load_part (a repeated kk_load_part rewrites the base bytes and merges again: the result is identical).
 *   memory    A and B are uploaded as fp32 once per device that merges, in one buffer freed before the call returns; kk_stats shows its bytes.
 *   identity  the canonical adapter path is part of the model's identity: base + opts + adapter again is the same model (refcount + 1), the
 *             base alone and base + adapter are two models.  The manifest and kk_stats gain an "adapter" object.
 *   refusals  all raised before any device is touched.
 *             KK_EUNSUPPORTED: a non-empty alpha_pattern; use_dora / lora_magnitude_vector; fan_in_fan_out; lora_embedding_A/B;
 *                              modules_to_save tensors; bias tensors or bias other than "none"; adapter_model.bin; adapter dtypes other than
 *                              F32 / BF16 / F16; r outside 1..256; a target that is not 2-D or whose pool dtype is not bf16, f16 or F32 (FP8 kept
 *                              verbatim, integers, transposed GPT-2 weights); KK_FANOUT_NVLS; a part_count > 1 load whose pool receives peers'
 *                              stores (BROADCAST in any fan-out, SCATTER with KK_LOAD_SCATTER_EXCHANGE).  Multi-part SCATTER without the
 *                              exchange merges: a rank's pool is written by that rank only.
 *             KK_EFORMAT:      an unpaired lora_A / lora_B, mismatched shapes, a key that is not a LoRA key, a malformed config or a missing
 *                              or ill-typed config key (lora_alpha a finite number; use_rslora, use_dora, fan_in_fan_out booleans; bias a string).
 *             KK_ENOENT:       no adapter at adapter_path, no adapter_config.json, a target the checkpoint does not have.
 * kk_adapter_describe plans like kk_plan_describe with n_parts = part_count (1 when part_count <= 1). */
int kk_load_adapter(kk_ctx* ctx, const char* path, const kk_load_opts* opts, const char* adapter_path, kk_model** out);
int kk_adapter_describe(kk_ctx* ctx, const char* path, const kk_load_opts* opts, const char* adapter_path, char* json, size_t cap,
                        size_t* required);
/* kk_derive_adapter: the model kk_load_adapter(ctx, path, opts, adapter_path) would return, with path and opts those `base` was loaded with,
 * built from base's resident pool(s) instead of the checkpoint file.  Only the source of the base bytes differs:
 *   identity  the same registry key as that load: if the model is resident the call returns it (refcount + 1) and does no work, and a later
 *             kk_load_adapter with those arguments returns the derived model.  It holds no reference on base, which may be released at once.
 *   model     plan, placements, kk_model_tensor, kk_model_get_info, the manifest (the "adapter" object included), kk_export / kk_export_fd,
 *             the pool budget and kk_release are those of the kk_load_adapter model.  kk_load_part on a model derived from a KK_LOAD_DEFER
 *             base streams the file and merges again, with an identical result.
 *   bytes     on each local device every byte of the pool allocation outside the targets is base's byte (copied by the copy engines;
 *             nothing crosses NVLink), and every target is the kk_load_adapter merge of base's element, bit for bit.
 *   stats     kk_stats gains "derive": {"base_key", "t_copy", "t_merge" (CUDA events, slowest device), "t_host" (adapter read, widening and
 *             upload, seconds)}.
 *   refusals  all raised before any allocation, with the pool budget and the registry unchanged: every refusal of kk_load_adapter for base's
 *             options and plan; KK_ESTATE when base is not loaded (KK_LOAD_DEFER before kk_load_part, two-stage before kk_convert_local);
 *             KK_EINVAL when base itself carries an adapter (adapters do not stack); KK_ENOMEM past the pool budget.
 *   locks     base's data-moving calls (kk_load_part) wait while its pools are read. */
int kk_derive_adapter(kk_model* base, const char* adapter_path, kk_model** out);
/* Deferred / multi-process loading: after kk_load_ex(...KK_LOAD_DEFER...) and any kk_peer_attach calls,
 * move the data.  May be called again to re-load (pools are overwritten with identical bytes). */
int kk_load_part(kk_model* m);
/* Attach the pool of another process's model (same checkpoint/plan) as fan-out destination `rank`.
 * ipc_handle is the 64-byte handle that process got from kk_export.  rank must differ from part_index. */
int kk_peer_attach(kk_model* m, int rank, const void* ipc_handle_64B);
int kk_peer_detach_all(kk_model* m);
/* KK_FANOUT_RAW in multi-process operation: the fan-out destinations are the other ranks' raw images, exported and
 * attached like pools (which = KK_BUF_RAW).  After every rank's kk_load_part (stage 1) and a caller-side barrier,
 * kk_convert_local (stage 2) dequantises/casts the gathered bytes into the local pool; ms_total (may be NULL)
 * receives its CUDA-event time.  Single-process kk_load runs both stages itself. */
#define KK_BUF_POOL 0
#define KK_BUF_RAW 1
#define KK_BUF_POOL_PTR 2 /* kk_peer_attach_buffer only: `ipc_handle_64B` points at a `void*` holding a device pointer that is
                             already valid in THIS process (several ranks hosted by one process, e.g. the single-GPU tests) */
#define KK_BUF_SLICE 3     /* KK_FANOUT_PULL: the slice buffer (export: its IPC handle; attach: the peer's) */
#define KK_BUF_SLICE_PTR 4 /* same, by raw device pointer valid in this process: export writes a `void*` into the first 8 bytes of
                             ipc_handle_64B, attach reads one from it */
int kk_export_buffer(kk_model* m, int device, int which, void* ipc_handle_64B);
int kk_peer_attach_buffer(kk_model* m, int rank, int which, const void* ipc_handle_64B);
/* KK_FANOUT_PULL uses the same two-stage protocol: kk_load_part (stage 1: own part -> own pool + slice buffer), caller-side barrier,
 * kk_convert_local (stage 2: pull every attached peer's slice into the local pool). */
int kk_convert_local(kk_model* m, float* ms_total);

int kk_model_get_info(kk_model* m, kk_model_info* out);
int kk_placements(kk_model* m, const char* tensor, kk_placement* out, size_t cap, size_t* n);
/* Tensor metadata of a loaded model by position (0 <= i < n_tensors), same order as kk_index. */
int kk_model_tensor(kk_model* m, size_t i, kk_tensor_meta* out);

/* ---- Mount: export to an agent container ----------------------------------------------------- */
/* ipc_handle_64B receives the cudaIpcMemHandle_t of `device`'s pool; manifest_json receives the pool
 * manifest (name -> offset/shape/dtype).  If cap is too small returns KK_ERANGE and, when
 * required != NULL, the needed size.  Either output may be NULL to skip it. */
int kk_export(kk_model* m, int device, void* ipc_handle_64B, char* manifest_json, size_t cap);
int kk_export_size(kk_model* m, int device, size_t* required);
/* KK_CFG_VMM_POOLS only: a new file descriptor for `device`'s pool (the caller owns it: pass it over a Unix socket with SCM_RIGHTS, then close it) and
 * the mapped size.  KK_EUNSUPPORTED for cudaMalloc pools.  Consumer side, possibly another process that received the fd: kk_import_fd maps the
 * allocation on CUDA device `device` of THAT process — read-only when flags has KK_IMPORT_READONLY — and returns its address; kk_import_close
 * unmaps it.  Neither needs a kk_ctx. */
#define KK_IMPORT_READONLY 0x1u
typedef struct kk_import kk_import;
int kk_export_fd(kk_model* m, int device, int* fd_out, uint64_t* mapped_bytes);
int kk_import_fd(int fd, int device, uint64_t mapped_bytes, uint32_t flags, void** dev_ptr, kk_import** out);
int kk_import_close(kk_import* im);
/* Same-process consumers: raw device pointer of the pool. */
int kk_pool_ptr(kk_model* m, int device, void** dev_ptr, uint64_t* nbytes);

/* Stable identity of a CUDA device, for everything that leaves this process: CUDA ordinals follow CUDA_DEVICE_ORDER / CUDA_VISIBLE_DEVICES and mean
 * nothing in another process or container, and they are NOT the minor number of /dev/nvidia<N>.  pci_bus_id receives "dddd:bb:dd.f" (>= 16 bytes),
 * uuid receives "GPU-xxxxxxxx-xxxx-xxxx-xxxx-xxxxxxxxxxxx" (>= 41 bytes).  Either may be NULL.  The host side maps the bus id to the device node through
 * /proc/driver/nvidia/gpus/<bus id>/information ("Device Minor"), internal/ctr's WithGPUWeights exports the UUID to the container. */
int kk_device_identity(int device, char* pci_bus_id, size_t pci_cap, char* uuid, size_t uuid_cap);

/* ---- Session refcount ------------------------------------------------------------------------ */
int kk_acquire(kk_model* m);
int kk_release(kk_model* m); /* frees pools when the count reaches 0 */

/* ---- Observability / verification ------------------------------------------------------------ */
int kk_stats(kk_model* m, char* json, size_t cap);
/* Copy pool bytes back to the host (verification only; not on the hot path). */
int kk_read(kk_model* m, int device, uint64_t pool_offset, uint64_t nbytes, void* host_dst);
/* 64-bit order-sensitive checksum of a pool range computed on the device (see oracle for the definition):
 * sum over 8-byte little-endian words w_i (zero-padded tail) of mix(w_i + i*0x9E3779B97F4A7C15). */
int kk_checksum(kk_model* m, int device, uint64_t pool_offset, uint64_t nbytes, uint64_t* out);

/* ---- Kernel-stage measurement (inputs resident in HBM) --------------------------------------- */
/* Stage this model's (part of the) checkpoint bytes into a device-resident image (untimed), then
 * kk_convert_resident runs exactly the convert/fan-out launches of a load — one launch per shard — from
 * that image, timed with CUDA events on the launching stream.  ms_total receives the elapsed time of
 * all launches; ms_per_launch (cap entries, may be NULL) each launch's own duration; n_launches the count. */
int kk_stage_resident(kk_model* m);
int kk_convert_resident(kk_model* m, float* ms_total, float* ms_per_launch, size_t cap, size_t* n_launches);
int kk_unstage_resident(kk_model* m);

/* ---- Roofline probes (measurement only) ------------------------------------------------------- */
/* Time one launch of a probe kernel over a scratch buffer of `nbytes` (rounded down to 16) on `device`, after one untimed warm-up launch,
 * with CUDA events on the launching stream.  kind KK_PROBE_WRITE: store-only fill (the HBM-write roofline a conversion's output is
 * measured against, SURVEY.md §8(d)); KK_PROBE_COPY: plain ld.global / st.global copy of nbytes (reads nbytes, writes nbytes). */
#define KK_PROBE_WRITE 0
#define KK_PROBE_COPY 1
int kk_probe_hbm(kk_ctx* ctx, int device, int kind, uint64_t nbytes, float* ms);
/* NVLink probe for multi-process models: one copy-engine read of up to *nbytes from the buffer of rank `rank` that this model has attached
 * (which = KK_BUF_POOL, KK_BUF_RAW or KK_BUF_SLICE) into a local scratch, after one untimed pass.  *nbytes returns the bytes actually copied, *ms their
 * CUDA-event time.  Every rank probing its ring neighbour at the same moment measures the per-GPU NVLink ingress the fan-out is bounded by. */
int kk_probe_peer(kk_model* m, int rank, int which, uint64_t* nbytes, float* ms);

#ifdef __cplusplus
}
#endif
#endif /* KUKEON_GPULOAD_H */
