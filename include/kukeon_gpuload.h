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

typedef struct kk_ctx kk_ctx;     /* one per process (kukeond lifetime) */
typedef struct kk_model kk_model; /* refcounted; one per (checkpoint identity, mode, flags) */

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
  uint32_t dtype;             /* dtype in the pool (KK_BF16 for every float tensor by default) */
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
  uint32_t reserved[3];
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
