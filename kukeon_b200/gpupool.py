"""ctypes binding of libkukeon_gpuload.so — the Python twin of the Go package `internal/gpupool` that
kukeond would carry (a thin cgo wrapper; SURVEY.md §8(a9), INTEGRATION.md).

All logic lives behind the C ABI (include/kukeon_gpuload.h).  This module only marshals structs, maps
negative status codes onto exceptions the way the Go shim maps them onto `internal/errdefs` sentinels
(`fmt.Errorf("%w: %s", errdefs.ErrGPUPoolLoad, C.GoString(C.kk_last_error()))`, errdefs.go:23-), and
refuses to work without the native library: there is no CPU or pure-Python fallback.
"""
from __future__ import annotations

import ctypes as C
import json
import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

KK_MAX_DEVICES = 8
KK_MAX_DIMS = 8
KK_NAME_MAX = 256
KK_IPC_HANDLE_BYTES = 64
KK_POOL_ALIGN = 256

MODE_SINGLE, MODE_BROADCAST, MODE_SCATTER = 0, 1, 2
FANOUT_P2P, FANOUT_NVLS, FANOUT_NONE, FANOUT_RAW, FANOUT_PULL = 0, 1, 2, 3, 4
CFG_ZEROCOPY, CFG_NO_PEER_ACCESS, CFG_NO_NUMA_PIN, CFG_PEER_ALL, CFG_VMM_POOLS = 0x1, 0x2, 0x4, 0x8, 0x10
IMPORT_READONLY = 0x1
LOAD_GPT2_CONV1D_T, LOAD_KEEP_F32, LOAD_DEFER, LOAD_SCATTER_EXCHANGE, LOAD_F8_TO_BF16 = 0x1, 0x2, 0x4, 0x8, 0x10
LOAD_F16 = 0x80  # every float output as IEEE fp16 instead of bf16, same pool layout (kukeon_gpuload.h KK_LOAD_F16); 0x20 / 0x40 stay unused
LOAD_HF_LAYOUT = 0x100  # GGUF in Hugging Face layout: HF names, one tensor per expert, llama's Q/K rows un-permuted (KK_LOAD_HF_LAYOUT)
BUF_POOL, BUF_RAW, BUF_POOL_PTR, BUF_SLICE, BUF_SLICE_PTR = 0, 1, 2, 3, 4
PROBE_WRITE, PROBE_COPY = 0, 1

DTYPE_NAMES = {
    0: "BOOL", 1: "F4", 2: "F6_E2M3", 3: "F6_E3M2", 4: "U8", 5: "I8", 6: "F8_E5M2", 7: "F8_E4M3", 8: "F8_E8M0",
    9: "I16", 10: "U16", 11: "F16", 12: "BF16", 13: "I32", 14: "U32", 15: "F32", 16: "C64", 17: "F64", 18: "I64",
    19: "U64", 32: "Q4_0", 33: "Q4_1", 34: "Q5_0", 35: "Q5_1", 36: "Q8_0", 37: "Q2_K", 38: "Q3_K", 39: "Q4_K",
    40: "Q5_K", 41: "Q6_K", 42: "Q8_K", 43: "IQ4_NL", 44: "IQ4_XS", 45: "MXFP4",
    46: "IQ2_XXS", 47: "IQ2_XS", 48: "IQ2_S", 49: "IQ3_XXS", 50: "IQ3_S", 51: "IQ1_S", 52: "IQ1_M", 53: "TQ1_0", 54: "TQ2_0", 55: "NVFP4",
}


class GPUPoolError(RuntimeError):
    """Base of every error surfaced from the C ABI; `.code` is the negative kk_status."""
    code = 0

    def __init__(self, code: int, msg: str):
        super().__init__(f"{STATUS_NAMES.get(code, code)}: {msg}")
        self.code = code
        self.detail = msg


class ErrInvalid(GPUPoolError): pass          # KK_EINVAL
class ErrNotFound(GPUPoolError): pass         # KK_ENOENT
class ErrFormat(GPUPoolError): pass           # KK_EFORMAT
class ErrIO(GPUPoolError): pass               # KK_EIO
class ErrNoMemory(GPUPoolError): pass         # KK_ENOMEM
class ErrCUDA(GPUPoolError): pass             # KK_ECUDA
class ErrUnsupported(GPUPoolError): pass      # KK_EUNSUPPORTED
class ErrBusy(GPUPoolError): pass             # KK_EBUSY
class ErrRange(GPUPoolError): pass            # KK_ERANGE
class ErrState(GPUPoolError): pass            # KK_ESTATE


STATUS_NAMES = {0: "KK_OK", -1: "KK_EINVAL", -2: "KK_ENOENT", -3: "KK_EFORMAT", -4: "KK_EIO", -5: "KK_ENOMEM",
                -6: "KK_ECUDA", -7: "KK_EUNSUPPORTED", -8: "KK_EBUSY", -9: "KK_ERANGE", -10: "KK_ESTATE"}
_ERR = {-1: ErrInvalid, -2: ErrNotFound, -3: ErrFormat, -4: ErrIO, -5: ErrNoMemory, -6: ErrCUDA, -7: ErrUnsupported,
        -8: ErrBusy, -9: ErrRange, -10: ErrState}


class KKConfig(C.Structure):
    _fields_ = [("n_devices", C.c_int32), ("devices", C.c_int32 * KK_MAX_DEVICES), ("pool_bytes_per_device", C.c_uint64),
                ("n_staging_buffers", C.c_uint32), ("staging_buffer_bytes", C.c_uint64), ("n_reader_threads", C.c_uint32),
                ("flags", C.c_uint32)]


class KKTensorMeta(C.Structure):
    _fields_ = [("name", C.c_char * KK_NAME_MAX), ("dtype", C.c_uint32), ("n_dims", C.c_uint32),
                ("shape", C.c_uint64 * KK_MAX_DIMS), ("shard", C.c_uint32), ("reserved", C.c_uint32),
                ("file_offset", C.c_uint64), ("nbytes", C.c_uint64)]


class KKPlacement(C.Structure):
    _fields_ = [("device", C.c_int32), ("dtype", C.c_uint32), ("pool_offset", C.c_uint64), ("nbytes", C.c_uint64),
                ("n_dims", C.c_uint32), ("slice_dim", C.c_uint32), ("shape", C.c_uint64 * KK_MAX_DIMS),
                ("slice_begin", C.c_uint64)]


class KKLoadOpts(C.Structure):
    _fields_ = [("mode", C.c_int32), ("fanout", C.c_int32), ("flags", C.c_uint32), ("part_index", C.c_int32),
                ("part_count", C.c_int32), ("layer_begin", C.c_uint32), ("layer_end", C.c_uint32), ("reserved", C.c_uint32)]


class KKModelInfo(C.Structure):
    _fields_ = [("n_tensors", C.c_uint64), ("n_shards", C.c_uint64), ("file_bytes", C.c_uint64), ("pool_bytes", C.c_uint64),
                ("n_devices", C.c_int32), ("devices", C.c_int32 * KK_MAX_DEVICES), ("mode", C.c_int32), ("refcount", C.c_int32),
                ("loaded", C.c_int32), ("reserved", C.c_int32)]


LIB_NAME = "libkukeon_gpuload.so"
_lib = None

# every symbol include/kukeon_gpuload.h declares
ABI_SYMBOLS = [
    "kk_abi_version", "kk_last_error", "kk_status_name", "kk_open", "kk_close", "kk_index", "kk_free_index",
    "kk_index_shard", "kk_plan_describe", "kk_load", "kk_load_ex", "kk_load_part", "kk_peer_attach", "kk_peer_detach_all",
    "kk_export_buffer", "kk_peer_attach_buffer", "kk_convert_local",
    "kk_model_get_info", "kk_placements", "kk_model_tensor", "kk_export", "kk_export_size", "kk_pool_ptr",
    "kk_acquire", "kk_release", "kk_stats", "kk_read", "kk_checksum", "kk_stage_resident", "kk_convert_resident",
    "kk_unstage_resident", "kk_probe_hbm", "kk_probe_peer", "kk_device_identity",
    "kk_export_fd", "kk_import_fd", "kk_import_close", "kk_load_adapter", "kk_adapter_describe",
    "kk_derive_adapter",
]


def lib_path() -> str:
    """In-tree library next to this file; KUKEON_GPULOAD_LIB overrides it (experiments / packaged installs)."""
    return os.environ.get("KUKEON_GPULOAD_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), LIB_NAME)


def lib():
    """Load the native library or fail loudly — the product has no other implementation."""
    global _lib
    if _lib is not None:
        return _lib
    p = lib_path()
    if not os.path.exists(p):
        raise ImportError(f"{p} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          f"(or `make -C kukeon_b200/csrc`). kukeon_b200 has no CPU fallback.")
    L = C.CDLL(p)
    vp = C.c_void_p
    L.kk_abi_version.restype = C.c_int
    L.kk_last_error.restype = C.c_char_p
    L.kk_status_name.restype = C.c_char_p
    L.kk_status_name.argtypes = [C.c_int]
    L.kk_open.argtypes = [C.POINTER(KKConfig), C.POINTER(vp)]
    L.kk_close.argtypes = [vp]
    L.kk_probe_hbm.argtypes = [vp, C.c_int, C.c_int, C.c_uint64, C.POINTER(C.c_float)]
    L.kk_probe_peer.argtypes = [vp, C.c_int, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_float)]
    L.kk_device_identity.argtypes = [C.c_int, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]
    L.kk_export_fd.argtypes = [vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_uint64)]
    L.kk_import_fd.argtypes = [C.c_int, C.c_int, C.c_uint64, C.c_uint32, C.POINTER(vp), C.POINTER(vp)]
    L.kk_import_close.argtypes = [vp]
    L.kk_index.argtypes = [vp, C.c_char_p, C.POINTER(C.POINTER(KKTensorMeta)), C.POINTER(C.c_size_t)]
    L.kk_free_index.argtypes = [C.POINTER(KKTensorMeta)]
    L.kk_index_shard.argtypes = [vp, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.kk_plan_describe.argtypes = [vp, C.c_char_p, C.POINTER(KKLoadOpts), C.c_int, C.c_uint64, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.kk_load.argtypes = [vp, C.c_char_p, C.c_int, C.c_int, C.POINTER(vp)]
    L.kk_load_ex.argtypes = [vp, C.c_char_p, C.POINTER(KKLoadOpts), C.POINTER(vp)]
    L.kk_load_part.argtypes = [vp]
    L.kk_load_adapter.argtypes = [vp, C.c_char_p, C.POINTER(KKLoadOpts), C.c_char_p, C.POINTER(vp)]
    L.kk_adapter_describe.argtypes = [vp, C.c_char_p, C.POINTER(KKLoadOpts), C.c_char_p, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.kk_derive_adapter.argtypes = [vp, C.c_char_p, C.POINTER(vp)]
    L.kk_peer_attach.argtypes = [vp, C.c_int, C.c_void_p]
    L.kk_peer_detach_all.argtypes = [vp]
    L.kk_export_buffer.argtypes = [vp, C.c_int, C.c_int, C.c_void_p]
    L.kk_peer_attach_buffer.argtypes = [vp, C.c_int, C.c_int, C.c_void_p]
    L.kk_convert_local.argtypes = [vp, C.POINTER(C.c_float)]
    L.kk_model_get_info.argtypes = [vp, C.POINTER(KKModelInfo)]
    L.kk_placements.argtypes = [vp, C.c_char_p, C.POINTER(KKPlacement), C.c_size_t, C.POINTER(C.c_size_t)]
    L.kk_model_tensor.argtypes = [vp, C.c_size_t, C.POINTER(KKTensorMeta)]
    L.kk_export.argtypes = [vp, C.c_int, C.c_void_p, C.c_char_p, C.c_size_t]
    L.kk_export_size.argtypes = [vp, C.c_int, C.POINTER(C.c_size_t)]
    L.kk_pool_ptr.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(C.c_uint64)]
    L.kk_acquire.argtypes = [vp]
    L.kk_release.argtypes = [vp]
    L.kk_stats.argtypes = [vp, C.c_char_p, C.c_size_t]
    L.kk_read.argtypes = [vp, C.c_int, C.c_uint64, C.c_uint64, C.c_void_p]
    L.kk_checksum.argtypes = [vp, C.c_int, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64)]
    L.kk_stage_resident.argtypes = [vp]
    L.kk_convert_resident.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_size_t, C.POINTER(C.c_size_t)]
    L.kk_unstage_resident.argtypes = [vp]
    for s in ABI_SYMBOLS:
        if s not in ("kk_last_error", "kk_status_name"):
            getattr(L, s).restype = C.c_int
    if L.kk_abi_version() != 1:
        raise ImportError(f"{p}: ABI version {L.kk_abi_version()} != 1")
    _lib = L
    return L


class ImportedPool:
    """Consumer side of a VMM pool: the allocation behind `fd` mapped on CUDA device `device` of THIS process, read-only by default
    (stores through the mapping fault here and never reach the exporter's weights)."""

    def __init__(self, fd: int, device: int, mapped_bytes: int, readonly: bool = True):
        p, h = C.c_void_p(), C.c_void_p()
        _check(lib().kk_import_fd(fd, device, mapped_bytes, IMPORT_READONLY if readonly else 0, C.byref(p), C.byref(h)))
        self.ptr, self._h, self.nbytes = int(p.value or 0), h, mapped_bytes

    def close(self) -> None:
        if self._h:
            _check(lib().kk_import_close(self._h))
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def device_identity(ordinal: int) -> dict:
    """{"pci_bus_id": "0000:1b:00.0", "uuid": "GPU-..."} of CUDA device `ordinal` in this process (kk_device_identity)."""
    bus, uuid = C.create_string_buffer(32), C.create_string_buffer(64)
    _check(lib().kk_device_identity(ordinal, bus, len(bus), uuid, len(uuid)))
    return {"pci_bus_id": bus.value.decode(), "uuid": uuid.value.decode()}


def _check(rc: int) -> None:
    if rc != 0:
        msg = lib().kk_last_error().decode("utf-8", "replace")
        raise _ERR.get(rc, GPUPoolError)(rc, msg)


def _meta_to_dict(m: KKTensorMeta) -> dict:
    return dict(name=m.name.decode("utf-8"), dtype=DTYPE_NAMES.get(m.dtype, str(m.dtype)), shape=[int(m.shape[i]) for i in range(m.n_dims)],
                shard=int(m.shard), file_offset=int(m.file_offset), nbytes=int(m.nbytes))


def index(path: str) -> List[dict]:
    """kk_index: tensor records sorted by (shard, file_offset).  CPU only; needs no context."""
    L = lib()
    recs = C.POINTER(KKTensorMeta)()
    n = C.c_size_t()
    _check(L.kk_index(None, os.fsencode(path), C.byref(recs), C.byref(n)))
    try:
        return [_meta_to_dict(recs[i]) for i in range(n.value)]
    finally:
        L.kk_free_index(recs)


def index_shards(path: str) -> List[str]:
    L = lib()
    n = C.c_size_t()
    _check(L.kk_index_shard(None, os.fsencode(path), 0, None, 0, C.byref(n)))
    out = []
    buf = C.create_string_buffer(4096)
    for i in range(n.value):
        _check(L.kk_index_shard(None, os.fsencode(path), i, buf, len(buf), None))
        out.append(os.fsdecode(buf.value))
    return out


def _set_layers(o: KKLoadOpts, layers: Optional[Sequence[int]]) -> None:
    """layers=(begin, end): the pipeline stage [begin, end) (see kk_load_opts in kukeon_gpuload.h, which also validates the range);
    None: the whole checkpoint."""
    if layers is not None:
        b, e = (int(x) for x in layers)
        if not (0 <= b < 2**32 and 0 <= e < 2**32):
            raise ErrInvalid(-1, f"layer range [{b}, {e}) does not fit kk_load_opts' uint32 fields")
        o.layer_begin, o.layer_end = b, e


def plan_describe(path: str, mode: int = MODE_SINGLE, flags: int = 0, n_parts: int = 1, chunk_bytes: int = 0,
                  layers: Optional[Sequence[int]] = None) -> dict:
    """kk_plan_describe: pool layout + per-part chunk/segment lists, computed on the CPU.  layers=(begin, end) describes that
    pipeline stage only."""
    L = lib()
    o = KKLoadOpts()
    o.mode, o.flags = mode, flags
    _set_layers(o, layers)
    need = C.c_size_t()
    _check(L.kk_plan_describe(None, os.fsencode(path), C.byref(o), n_parts, chunk_bytes, None, 0, C.byref(need)))
    buf = C.create_string_buffer(need.value)
    _check(L.kk_plan_describe(None, os.fsencode(path), C.byref(o), n_parts, chunk_bytes, buf, need.value, None))
    return json.loads(buf.value.decode("utf-8"))


def adapter_describe(path: str, adapter: str, mode: int = MODE_SINGLE, fanout: int = FANOUT_P2P, flags: int = 0, part_index: int = 0,
                     part_count: int = 0, layers: Optional[Sequence[int]] = None) -> dict:
    """kk_adapter_describe: the LoRA merge a kk_load_adapter with these options would do (targets, ranks, scalings), or the error it
    would raise.  CPU only; needs no context."""
    L = lib()
    o = KKLoadOpts()
    o.mode, o.fanout, o.flags, o.part_index, o.part_count = mode, fanout, flags, part_index, part_count
    _set_layers(o, layers)
    need = C.c_size_t()
    _check(L.kk_adapter_describe(None, os.fsencode(path), C.byref(o), os.fsencode(adapter), None, 0, C.byref(need)))
    buf = C.create_string_buffer(need.value)
    _check(L.kk_adapter_describe(None, os.fsencode(path), C.byref(o), os.fsencode(adapter), buf, need.value, None))
    return json.loads(buf.value.decode("utf-8"))


@dataclass
class Placement:
    device: int
    dtype: str
    pool_offset: int
    nbytes: int
    shape: List[int]
    slice_dim: Optional[int]
    slice_begin: int


class Model:
    """A resident checkpoint (kk_model*).  One reference is held by the object until release()."""

    def __init__(self, pool: "Pool", handle: int):
        self._pool = pool
        self._h = C.c_void_p(handle)
        self._released = False

    # -- info ---------------------------------------------------------------------------------
    def info(self) -> dict:
        mi = KKModelInfo()
        _check(lib().kk_model_get_info(self._h, C.byref(mi)))
        return dict(n_tensors=int(mi.n_tensors), n_shards=int(mi.n_shards), file_bytes=int(mi.file_bytes), pool_bytes=int(mi.pool_bytes),
                    devices=[int(mi.devices[i]) for i in range(mi.n_devices)], mode=int(mi.mode), refcount=int(mi.refcount),
                    loaded=bool(mi.loaded))

    def tensors(self) -> List[dict]:
        n = self.info()["n_tensors"]
        out = []
        m = KKTensorMeta()
        for i in range(n):
            _check(lib().kk_model_tensor(self._h, i, C.byref(m)))
            out.append(_meta_to_dict(m))
        return out

    def placements(self, tensor: str) -> List[Placement]:
        arr = (KKPlacement * KK_MAX_DEVICES)()
        n = C.c_size_t()
        _check(lib().kk_placements(self._h, tensor.encode("utf-8"), arr, KK_MAX_DEVICES, C.byref(n)))
        out = []
        for i in range(n.value):
            p = arr[i]
            out.append(Placement(int(p.device), DTYPE_NAMES.get(p.dtype, str(p.dtype)), int(p.pool_offset), int(p.nbytes),
                                 [int(p.shape[d]) for d in range(p.n_dims)], None if p.slice_dim == 0xFFFFFFFF else int(p.slice_dim),
                                 int(p.slice_begin)))
        return out

    def stats(self) -> dict:
        buf = C.create_string_buffer(1 << 16)
        _check(lib().kk_stats(self._h, buf, len(buf)))
        return json.loads(buf.value.decode("utf-8"))

    # -- Mount --------------------------------------------------------------------------------
    def export(self, device: int) -> tuple[bytes, dict]:
        """(64-byte CUDA IPC handle, manifest dict) for `device`'s pool."""
        need = C.c_size_t()
        _check(lib().kk_export_size(self._h, device, C.byref(need)))
        man = C.create_string_buffer(need.value)
        h = C.create_string_buffer(KK_IPC_HANDLE_BYTES)
        _check(lib().kk_export(self._h, device, h, man, need.value))
        return h.raw, json.loads(man.value.decode("utf-8"))

    def manifest(self, device: int) -> dict:
        need = C.c_size_t()
        _check(lib().kk_export_size(self._h, device, C.byref(need)))
        man = C.create_string_buffer(need.value)
        _check(lib().kk_export(self._h, device, None, man, need.value))
        return json.loads(man.value.decode("utf-8"))

    def export_fd(self, device: int) -> tuple[int, int]:
        """(file descriptor, mapped bytes) of `device`'s pool — KK_CFG_VMM_POOLS contexts only.  The caller owns the fd: send it to the consumer
        over a Unix socket (socket.send_fds) and close it."""
        fd, n = C.c_int(-1), C.c_uint64()
        _check(lib().kk_export_fd(self._h, device, C.byref(fd), C.byref(n)))
        return int(fd.value), int(n.value)

    def pool_ptr(self, device: int) -> tuple[int, int]:
        p = C.c_void_p()
        n = C.c_uint64()
        _check(lib().kk_pool_ptr(self._h, device, C.byref(p), C.byref(n)))
        return int(p.value or 0), int(n.value)

    # -- multi-process ------------------------------------------------------------------------
    def peer_attach(self, rank: int, ipc_handle: bytes) -> None:
        assert len(ipc_handle) == KK_IPC_HANDLE_BYTES
        _check(lib().kk_peer_attach(self._h, rank, C.c_char_p(ipc_handle)))

    def export_buffer(self, device: int, which: int) -> bytes:
        """IPC handle of the pool (BUF_POOL), of the raw image of a KK_FANOUT_RAW model (BUF_RAW) or of the slice buffer of a
        KK_FANOUT_PULL model (BUF_SLICE; BUF_SLICE_PTR: its raw device pointer in the first 8 bytes, for ranks sharing a process)."""
        h = C.create_string_buffer(KK_IPC_HANDLE_BYTES)
        _check(lib().kk_export_buffer(self._h, device, which, h))
        return h.raw

    def peer_attach_buffer(self, rank: int, which: int, ipc_handle: bytes) -> None:
        assert len(ipc_handle) == KK_IPC_HANDLE_BYTES
        _check(lib().kk_peer_attach_buffer(self._h, rank, which, C.c_char_p(ipc_handle)))

    def peer_attach_local_pointer(self, rank: int, dev_ptr: int) -> None:
        """Several ranks hosted by one process (tests): attach another model's pool by raw device pointer."""
        p = C.c_void_p(dev_ptr)
        _check(lib().kk_peer_attach_buffer(self._h, rank, BUF_POOL_PTR, C.byref(p)))

    def convert_local(self) -> float:
        """Stage 2 of a multi-process KK_FANOUT_RAW load (dequantise the gathered bytes) or of a KK_FANOUT_PULL load (pull the peers'
        slices over NVLink); returns its CUDA-event milliseconds."""
        ms = C.c_float()
        _check(lib().kk_convert_local(self._h, C.byref(ms)))
        return float(ms.value)

    def probe_peer(self, rank: int, which: int = BUF_POOL, nbytes: int = 1 << 30) -> float:
        """GB/s of one copy-engine read of up to `nbytes` from the attached buffer of rank `rank` (NVLink ingress probe)."""
        n = C.c_uint64(nbytes)
        ms = C.c_float()
        _check(lib().kk_probe_peer(self._h, rank, which, C.byref(n), C.byref(ms)))
        return n.value / (ms.value / 1e3) / 1e9 if ms.value > 0 else 0.0

    def peer_detach_all(self) -> None:
        _check(lib().kk_peer_detach_all(self._h))

    def load_part(self) -> None:
        _check(lib().kk_load_part(self._h))

    def derive(self, adapter: str) -> "Model":
        """kk_derive_adapter: the model Pool.load(<this model's path and options>, adapter=adapter) returns, its pools built from this
        model's resident pools on the GPU instead of from the checkpoint file.  A model of its own; this one may be released at once."""
        h = C.c_void_p()
        _check(lib().kk_derive_adapter(self._h, os.fsencode(adapter), C.byref(h)))
        return Model(self._pool, h.value)

    # -- verification / measurement -----------------------------------------------------------
    def read(self, device: int, offset: int, nbytes: int):
        import numpy as np
        out = np.empty(nbytes, np.uint8)
        if nbytes:
            _check(lib().kk_read(self._h, device, offset, nbytes, out.ctypes.data_as(C.c_void_p)))
        return out

    def checksum(self, device: int, offset: int, nbytes: int) -> int:
        v = C.c_uint64()
        _check(lib().kk_checksum(self._h, device, offset, nbytes, C.byref(v)))
        return int(v.value)

    def stage_resident(self) -> None:
        _check(lib().kk_stage_resident(self._h))

    def unstage_resident(self) -> None:
        _check(lib().kk_unstage_resident(self._h))

    def convert_resident(self) -> tuple[float, List[float]]:
        """Run the convert/fan-out launches from the resident image; (total ms, per-launch ms)."""
        tot = C.c_float()
        per = (C.c_float * 256)()
        n = C.c_size_t()
        _check(lib().kk_convert_resident(self._h, C.byref(tot), per, 256, C.byref(n)))
        return float(tot.value), [float(per[i]) for i in range(min(n.value, 256))]

    # -- refcount -----------------------------------------------------------------------------
    def acquire(self) -> None:
        _check(lib().kk_acquire(self._h))

    def release(self) -> None:
        _check(lib().kk_release(self._h))

    @property
    def handle(self) -> int:
        return int(self._h.value or 0)


class Pool:
    """kk_ctx*: the daemon-lifetime GPU pool manager (Go: `gpupool.Open(cfg)` in daemon.NewServer,
    internal/daemon/server.go:87; closed from Server.Stop, server.go:242)."""

    def __init__(self, devices: Sequence[int] = (0,), pool_bytes_per_device: int = 0, n_staging_buffers: int = 0,
                 staging_buffer_bytes: int = 0, n_reader_threads: int = 0, flags: int = 0):
        cfg = KKConfig()
        cfg.n_devices = len(devices)
        for i, d in enumerate(devices):
            cfg.devices[i] = d
        cfg.pool_bytes_per_device = pool_bytes_per_device
        cfg.n_staging_buffers = n_staging_buffers
        cfg.staging_buffer_bytes = staging_buffer_bytes
        cfg.n_reader_threads = n_reader_threads
        cfg.flags = flags
        h = C.c_void_p()
        _check(lib().kk_open(C.byref(cfg), C.byref(h)))
        self._h = h
        self.devices = list(devices)

    def load(self, path: str, mode: int = MODE_SINGLE, fanout: int = FANOUT_P2P, flags: int = 0, part_index: int = 0,
             part_count: int = 0, layers: Optional[Sequence[int]] = None, adapter: Optional[str] = None) -> Model:
        """kk_load_ex.  layers=(begin, end) loads the pipeline stage [begin, end) only, as a model of its own.  adapter: a PEFT LoRA
        adapter (directory or adapter_model.safetensors) merged into the pool(s) after the load (kk_load_adapter), a model of its own."""
        o = KKLoadOpts()
        o.mode, o.fanout, o.flags, o.part_index, o.part_count = mode, fanout, flags, part_index, part_count
        _set_layers(o, layers)
        h = C.c_void_p()
        if adapter is None:
            _check(lib().kk_load_ex(self._h, os.fsencode(path), C.byref(o), C.byref(h)))
        else:
            _check(lib().kk_load_adapter(self._h, os.fsencode(path), C.byref(o), os.fsencode(adapter), C.byref(h)))
        return Model(self, h.value)

    def probe_hbm(self, device: int, kind: int = 0, nbytes: int = 4 << 30) -> float:
        """GB/s of one probe launch over `nbytes` of scratch HBM: kind 0 (PROBE_WRITE) store-only — bytes written / time;
        kind 1 (PROBE_COPY) ld/st copy — bytes read + written / time."""
        ms = C.c_float()
        _check(lib().kk_probe_hbm(self._h, device, kind, nbytes, C.byref(ms)))
        moved = nbytes * (2 if kind == PROBE_COPY else 1)
        return moved / (ms.value / 1e3) / 1e9 if ms.value > 0 else 0.0

    def close(self) -> None:
        if self._h:
            _check(lib().kk_close(self._h))
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()
