// NOT COMPILED HERE (no Go toolchain) — reviewed source; see host/go/README.md.
//
// Additions to internal/errdefs/errdefs.go, next to the volume block (errdefs.go:131-144).

package errdefs

import "errors"

// GPU pool (libkukeon_gpuload) errors: one sentinel per kk_status class a caller can act on.
var (
	ErrGPUPoolModelNotFound = errors.New("model checkpoint not found")
	ErrGPUPoolBadCheckpoint = errors.New("model checkpoint is malformed")
	ErrGPUPoolNoMemory      = errors.New("gpu pool is out of memory or over its budget")
	ErrGPUPoolBusy          = errors.New("gpu pool object is still referenced")
	ErrGPUPoolUnsupported   = errors.New("not supported by the gpu pool on this machine")
	ErrGPUPoolLoad          = errors.New("gpu pool load failed")
)

// models[] validation errors (internal/controller/validate_models.go).
var (
	ErrModelNameRequired         = errors.New("model name is required")
	ErrModelNameDuplicate        = errors.New("model name is declared more than once in the container")
	ErrModelNameInvalid          = errors.New("model name must be one path component of letters, digits, '.', '_' or '-' (it becomes a directory and an env-name suffix)")
	ErrModelSourceRequired       = errors.New("model source is required")
	ErrModelSourceNotAbsolute    = errors.New("model source must be an absolute host path")
	ErrModelSourceNotFound       = errors.New("model source does not exist on the host")
	ErrModelTargetNotAbsolute    = errors.New("model target must be an absolute container path")
	ErrModelModeUnknown          = errors.New("model mode is not recognized; expected \"\", \"single\", \"broadcast\", or \"scatter\"")
	ErrModelDevicesInvalid       = errors.New("model devices must be distinct non-negative CUDA ordinals")
	ErrModelLayersInvalid        = errors.New("model layers must be [begin, end): two non-negative integers with begin < end")
	ErrModelOptionUnknown        = errors.New("model option is not recognized")
	ErrModelRegistryNotSupported = errors.New("registry references are not supported; use an absolute host path as source")
	ErrModelAdapterNotAbsolute   = errors.New("model adapter must be an absolute host path")
	ErrModelAdapterNotFound      = errors.New("model adapter does not exist on the host")
	ErrModelAdapterRegistryNotSupported = errors.New("adapter registry references are not supported; use an absolute host path as adapter")
)
