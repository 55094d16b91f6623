// NOT COMPILED HERE (no Go toolchain) — reviewed source; see host/go/README.md.

//go:build cgo && linux

// Package gpupool wraps libkukeon_gpuload.so: one Pool per kukeond process (its lifetime is the daemon's, internal/daemon/server.go:87,242),
// refcounted resident Models shared by the cells that mount them.
package gpupool

/*
#cgo CFLAGS:  -I${SRCDIR}/../../third_party/kukeon_gpuload/include
#cgo LDFLAGS: -lkukeon_gpuload
#include <stdlib.h>
#include "kukeon_gpuload.h"
*/
import "C"

import (
	"fmt"
	"runtime"
	"unsafe"

	"github.com/eminwux/kukeon/internal/errdefs"
)

type Mode int

const (
	ModeSingle    Mode = C.KK_MODE_SINGLE
	ModeBroadcast Mode = C.KK_MODE_BROADCAST
	ModeScatter   Mode = C.KK_MODE_SCATTER
)

// Load flags (kk_load_opts.flags); the models[].options of a manifest map onto these.
const (
	FlagGPT2Conv1DTranspose uint32 = C.KK_LOAD_GPT2_CONV1D_T
	FlagKeepF32             uint32 = C.KK_LOAD_KEEP_F32
	FlagF8ToBF16            uint32 = C.KK_LOAD_F8_TO_BF16
	// FlagF16 stores every float output as IEEE fp16 instead of bf16 (F16 tensors verbatim, BF16 / F32 / GGUF blocks rounded once);
	// the pool layout is that of the same load without it.  An f16 and a bf16 load of one file are two models.
	FlagF16 uint32 = C.KK_LOAD_F16
	// FlagHFLayout loads a GGUF checkpoint in Hugging Face layout: HF tensor names, one tensor per expert and llama's Q/K rows
	// un-permuted.  GGUF only (llama, qwen2, qwen3).
	FlagHFLayout uint32 = C.KK_LOAD_HF_LAYOUT
)

type Config struct {
	Devices            []int
	PoolBytesPerDevice uint64
	StagingBuffers     uint32
	StagingBufferBytes uint64
	ReaderThreads      uint32
	// VMMPools allocates pools with the driver's virtual-memory API (KK_CFG_VMM_POOLS): they are exported as POSIX file descriptors that agent
	// containers map READ-ONLY (Model.ExportFD + the staged pool.sock) instead of as cudaIpcMemHandles, which map read-write in every opener.
	// Set it whenever the cells that mount a model do not trust each other.
	VMMPools bool
}

type Pool struct{ h *C.kk_ctx }
type Model struct{ h *C.kk_model }

// call runs one library entry point and maps a negative kk_status onto an errdefs sentinel, the way internal/ctr wraps containerd errors
// (internal/ctr/container.go:561,586).  kk_last_error is THREAD-local and the Go scheduler may move a goroutine to another OS thread
// between two cgo calls, so the failing call and the read of its message are bracketed by runtime.LockOSThread (round-1 review: without
// it the text could belong to another goroutine's failure).
func call(f func() C.int) error {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	return wrap(f())
}

// wrap must run on the OS thread that made the failing call: only call() uses it.
func wrap(rc C.int) error {
	if rc == C.KK_OK {
		return nil
	}
	msg := C.GoString(C.kk_last_error())
	switch rc {
	case C.KK_ENOENT:
		return fmt.Errorf("%w: %s", errdefs.ErrGPUPoolModelNotFound, msg)
	case C.KK_EFORMAT:
		return fmt.Errorf("%w: %s", errdefs.ErrGPUPoolBadCheckpoint, msg)
	case C.KK_ENOMEM:
		return fmt.Errorf("%w: %s", errdefs.ErrGPUPoolNoMemory, msg)
	case C.KK_EBUSY:
		return fmt.Errorf("%w: %s", errdefs.ErrGPUPoolBusy, msg)
	case C.KK_EUNSUPPORTED:
		return fmt.Errorf("%w: %s", errdefs.ErrGPUPoolUnsupported, msg)
	default:
		return fmt.Errorf("%w: %s", errdefs.ErrGPUPoolLoad, msg)
	}
}

func Open(cfg Config) (*Pool, error) {
	if len(cfg.Devices) == 0 || len(cfg.Devices) > C.KK_MAX_DEVICES {
		return nil, fmt.Errorf("%w: %d devices", errdefs.ErrGPUPoolUnsupported, len(cfg.Devices))
	}
	var c C.kk_config
	c.n_devices = C.int32_t(len(cfg.Devices))
	for i, d := range cfg.Devices {
		c.devices[i] = C.int32_t(d)
	}
	c.pool_bytes_per_device = C.uint64_t(cfg.PoolBytesPerDevice)
	c.n_staging_buffers = C.uint32_t(cfg.StagingBuffers)
	c.staging_buffer_bytes = C.uint64_t(cfg.StagingBufferBytes)
	c.n_reader_threads = C.uint32_t(cfg.ReaderThreads)
	if cfg.VMMPools {
		c.flags |= C.KK_CFG_VMM_POOLS
	}
	p := &Pool{}
	if err := call(func() C.int { return C.kk_open(&c, &p.h) }); err != nil {
		return nil, err
	}
	return p, nil
}

func (p *Pool) Close() error { return call(func() C.int { return C.kk_close(p.h) }) }

// TensorMeta is one record of the tensor index (kk_tensor_meta).
type TensorMeta struct {
	Name       string
	Dtype      uint32
	Shape      []uint64
	Shard      uint32
	FileOffset uint64
	NBytes     uint64
}

// Index is modelhub.Pull's worker: CPU only, no device is touched (the Pool may be nil).
func Index(path string) ([]TensorMeta, error) {
	cs := C.CString(path)
	defer C.free(unsafe.Pointer(cs))
	var recs *C.kk_tensor_meta
	var n C.size_t
	if err := call(func() C.int { return C.kk_index(nil, cs, &recs, &n) }); err != nil {
		return nil, err
	}
	defer C.kk_free_index(recs)
	out := make([]TensorMeta, int(n))
	for i, r := range unsafe.Slice(recs, int(n)) {
		shape := make([]uint64, int(r.n_dims))
		for d := range shape {
			shape[d] = uint64(r.shape[d])
		}
		out[i] = TensorMeta{Name: C.GoString(&r.name[0]), Dtype: uint32(r.dtype), Shape: shape, Shard: uint32(r.shard),
			FileOffset: uint64(r.file_offset), NBytes: uint64(r.nbytes)}
	}
	return out, nil
}

// Layers selects a pipeline stage: layers [Begin, End) of the checkpoint (kk_load_opts.layer_begin / layer_end).  The zero value is
// the whole checkpoint.  The library checks the range against the checkpoint and documents which outer tensors each stage keeps.
type Layers struct {
	Begin, End uint32
}

// Plan is the dry run behind `kuke model plan` (kk_plan_describe): JSON, CPU only.
func Plan(path string, mode Mode, flags uint32, gpus int, layers Layers) ([]byte, error) {
	cs := C.CString(path)
	defer C.free(unsafe.Pointer(cs))
	var o C.kk_load_opts
	o.mode = C.int32_t(mode)
	o.flags = C.uint32_t(flags)
	o.layer_begin = C.uint32_t(layers.Begin)
	o.layer_end = C.uint32_t(layers.End)
	var need C.size_t
	if err := call(func() C.int { return C.kk_plan_describe(nil, cs, &o, C.int(gpus), 0, nil, 0, &need) }); err != nil {
		return nil, err
	}
	buf := make([]byte, need)
	if err := call(func() C.int { return C.kk_plan_describe(nil, cs, &o, C.int(gpus), 0, (*C.char)(unsafe.Pointer(&buf[0])), need, nil) }); err != nil {
		return nil, err
	}
	return buf[:need-1], nil
}

// Load makes the checkpoint resident (or returns the already-resident copy with its refcount bumped): N concurrent StartCell
// calls for the same model share one load.  A pipeline stage (layers not zero) is a model of its own.  adapter, when not empty, is a
// PEFT LoRA adapter merged into the pool(s) after the load (kk_load_adapter); base + adapter is a model of its own.
func (p *Pool) Load(path string, mode Mode, flags uint32, layers Layers, adapter string) (*Model, error) {
	cs := C.CString(path)
	defer C.free(unsafe.Pointer(cs))
	var o C.kk_load_opts
	o.mode = C.int32_t(mode)
	o.fanout = C.KK_FANOUT_P2P
	o.flags = C.uint32_t(flags)
	o.layer_begin = C.uint32_t(layers.Begin)
	o.layer_end = C.uint32_t(layers.End)
	m := &Model{}
	if adapter == "" {
		if err := call(func() C.int { return C.kk_load_ex(p.h, cs, &o, &m.h) }); err != nil {
			return nil, err
		}
		return m, nil
	}
	ca := C.CString(adapter)
	defer C.free(unsafe.Pointer(ca))
	if err := call(func() C.int { return C.kk_load_adapter(p.h, cs, &o, ca, &m.h) }); err != nil {
		return nil, err
	}
	return m, nil
}

// AdapterDescribe validates a LoRA adapter against the checkpoint as Load would see it and returns the merge it would do as JSON
// (kk_adapter_describe; CPU only).
func AdapterDescribe(path string, mode Mode, flags uint32, layers Layers, adapter string) ([]byte, error) {
	cs, ca := C.CString(path), C.CString(adapter)
	defer C.free(unsafe.Pointer(cs))
	defer C.free(unsafe.Pointer(ca))
	var o C.kk_load_opts
	o.mode = C.int32_t(mode)
	o.flags = C.uint32_t(flags)
	o.layer_begin = C.uint32_t(layers.Begin)
	o.layer_end = C.uint32_t(layers.End)
	var need C.size_t
	if err := call(func() C.int { return C.kk_adapter_describe(nil, cs, &o, ca, nil, 0, &need) }); err != nil {
		return nil, err
	}
	buf := make([]byte, need)
	if err := call(func() C.int { return C.kk_adapter_describe(nil, cs, &o, ca, (*C.char)(unsafe.Pointer(&buf[0])), need, nil) }); err != nil {
		return nil, err
	}
	return buf[:need-1], nil
}

// ExportFD returns a new file descriptor for the VMM pool of `device` and its mapped size (KK_CFG_VMM_POOLS contexts only).  The caller sends it to
// the agent over the staged Unix socket (SCM_RIGHTS) and closes it; the agent maps it with kk_import_fd(..., KK_IMPORT_READONLY).
func (m *Model) ExportFD(device int) (int, uint64, error) {
	var fd C.int
	var size C.uint64_t
	if err := call(func() C.int { return C.kk_export_fd(m.h, C.int(device), &fd, &size) }); err != nil {
		return -1, 0, err
	}
	return int(fd), uint64(size), nil
}

// DeviceIdentity is what leaves the process instead of a CUDA ordinal: the PCI bus id (key of /proc/driver/nvidia/gpus/<id>/information, where
// the /dev/nvidia<minor> number is read) and the GPU UUID (how the agent picks the device inside its container).
func DeviceIdentity(ordinal int) (pciBusID, uuid string, err error) {
	bus := make([]byte, 32)
	id := make([]byte, 64)
	if err = call(func() C.int {
		return C.kk_device_identity(C.int(ordinal), (*C.char)(unsafe.Pointer(&bus[0])), C.size_t(len(bus)), (*C.char)(unsafe.Pointer(&id[0])), C.size_t(len(id)))
	}); err != nil {
		return "", "", err
	}
	return C.GoString((*C.char)(unsafe.Pointer(&bus[0]))), C.GoString((*C.char)(unsafe.Pointer(&id[0]))), nil
}

// Derive returns the model Load(<m's path, mode, flags and layers>, adapter) returns, built from m's resident pools on the GPU instead of
// from the checkpoint file (kk_derive_adapter).  It is a model of its own and holds no reference on m.
func (m *Model) Derive(adapter string) (*Model, error) {
	ca := C.CString(adapter)
	defer C.free(unsafe.Pointer(ca))
	d := &Model{}
	if err := call(func() C.int { return C.kk_derive_adapter(m.h, ca, &d.h) }); err != nil {
		return nil, err
	}
	return d, nil
}

func (m *Model) Acquire() error { return call(func() C.int { return C.kk_acquire(m.h) }) }
func (m *Model) Release() error { return call(func() C.int { return C.kk_release(m.h) }) }

// Export returns the 64-byte CUDA IPC handle and the pool manifest JSON for one device (what Mount stages for the container).
func (m *Model) Export(device int) ([]byte, []byte, error) {
	var need C.size_t
	if err := call(func() C.int { return C.kk_export_size(m.h, C.int(device), &need) }); err != nil {
		return nil, nil, err
	}
	handle := make([]byte, C.KK_IPC_HANDLE_BYTES)
	manifest := make([]byte, need)
	if err := call(func() C.int { return C.kk_export(m.h, C.int(device), unsafe.Pointer(&handle[0]), (*C.char)(unsafe.Pointer(&manifest[0])), need) }); err != nil {
		return nil, nil, err
	}
	return handle, manifest[:need-1], nil
}
