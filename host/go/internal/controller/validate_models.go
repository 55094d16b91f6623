// NOT COMPILED HERE (no Go toolchain) — reviewed source; see host/go/README.md.
//
// validateModels is the sibling of validateVolumes (create_container.go:284-380): same order of checks, same error style.  It needs
//   pkg/api/model/v1beta1:  ContainerSpec.Models []ModelMount `json:"models,omitempty" yaml:"models,omitempty"`   (next to Volumes, container.go:206)
//   internal/modelhub:      the version-less twin of ModelMount (conversion in internal/apischeme like VolumeMount)
// Tested twin: kukeon_b200/schema.py (tests/test_schema_cli.py carries the table of rejections this must reproduce).

package controller

import (
	"regexp"
	"fmt"
	"math"
	"os"
	"path/filepath"
	"strings"

	"github.com/eminwux/kukeon/internal/errdefs"
	"github.com/eminwux/kukeon/internal/gpupool"
	intmodel "github.com/eminwux/kukeon/internal/modelhub"
)

const (
	defaultModelTarget = "/run/kukeon/gpupool"
	maxModelDevices    = 8 // KK_MAX_DEVICES
)

var modelModes = map[string]gpupool.Mode{
	"": gpupool.ModeSingle, "single": gpupool.ModeSingle, "broadcast": gpupool.ModeBroadcast, "scatter": gpupool.ModeScatter,
}

var modelOptionFlags = map[string]uint32{
	"gpt2Conv1dTranspose": gpupool.FlagGPT2Conv1DTranspose,
	"keepF32":             gpupool.FlagKeepF32,
	"f8ToBf16":            gpupool.FlagF8ToBF16,
	"f16":                 gpupool.FlagF16,
	"hfLayout":            gpupool.FlagHFLayout,
}

// validateModels normalises and checks the models[] of one container.
//   - name: required, unique within the container (it becomes a directory and an env-name suffix).
//   - source: required, absolute host path that exists; "org/name" or "scheme://..." look like registry references and are rejected with
//     ErrModelRegistryNotSupported, pointing at the deferred feature the way ErrVolumeNamedNotSupported does.
//   - target: absolute container path; empty means /run/kukeon/gpupool.
//   - mode: "", single, broadcast, scatter (case-insensitive).
//   - devices: distinct non-negative ordinals, at most 8; empty means every device of the daemon's pool.
//   - layers: absent, or [begin, end) with 0 <= begin < end: the pipeline stage of the checkpoint this container mounts.
//   - options: gpt2Conv1dTranspose, keepF32, f8ToBf16, f16 (every float tensor as fp16 instead of bf16, for fp16 engines and fp16
//     checkpoints; a model apart from the bf16 load of the same source).
var modelNameRE = regexp.MustCompile(`^[A-Za-z0-9][A-Za-z0-9._-]*$`)

func validateModels(in []intmodel.ModelMount) ([]intmodel.ModelMount, error) {
	if len(in) == 0 {
		return nil, nil
	}
	out := make([]intmodel.ModelMount, len(in))
	seen := make(map[string]struct{}, len(in))
	for i, m := range in {
		name := strings.TrimSpace(m.Name)
		if name == "" {
			return nil, fmt.Errorf("%w (model[%d])", errdefs.ErrModelNameRequired, i)
		}
		// The name is joined into <cell dir>/gpupool/<name> on the host and into the mount target inside the container: a "/", ".." or NUL
		// in it would let a manifest write outside the cell directory.  One path component of [A-Za-z0-9._-], not starting with '.'.
		if !modelNameRE.MatchString(name) {
			return nil, fmt.Errorf("%w (model[%d] name %q)", errdefs.ErrModelNameInvalid, i, name)
		}
		if _, dup := seen[name]; dup {
			return nil, fmt.Errorf("%w (model[%d] name %q)", errdefs.ErrModelNameDuplicate, i, name)
		}
		seen[name] = struct{}{}

		src := strings.TrimSpace(m.Source)
		if src == "" {
			return nil, fmt.Errorf("%w (model[%d])", errdefs.ErrModelSourceRequired, i)
		}
		if !filepath.IsAbs(src) {
			if strings.Contains(src, "://") || (strings.ContainsRune(src, os.PathSeparator) && !strings.HasPrefix(src, ".")) {
				return nil, fmt.Errorf("%w (model[%d] source %q)", errdefs.ErrModelRegistryNotSupported, i, src)
			}
			return nil, fmt.Errorf("%w (model[%d] source %q)", errdefs.ErrModelSourceNotAbsolute, i, src)
		}
		if _, statErr := os.Stat(src); statErr != nil {
			if os.IsNotExist(statErr) {
				return nil, fmt.Errorf("%w (model[%d] source %q)", errdefs.ErrModelSourceNotFound, i, src)
			}
			return nil, fmt.Errorf("failed to stat model[%d] source %q: %w", i, src, statErr)
		}

		// adapter: absent, or a PEFT LoRA adapter on the host merged into the pool on load (kk_load_adapter), validated like source
		adapter := strings.TrimSpace(m.Adapter)
		if m.Adapter != "" {
			if !filepath.IsAbs(adapter) {
				if strings.Contains(adapter, "://") || (strings.ContainsRune(adapter, os.PathSeparator) && !strings.HasPrefix(adapter, ".")) {
					return nil, fmt.Errorf("%w (model[%d] adapter %q)", errdefs.ErrModelAdapterRegistryNotSupported, i, adapter)
				}
				return nil, fmt.Errorf("%w (model[%d] adapter %q)", errdefs.ErrModelAdapterNotAbsolute, i, adapter)
			}
			if _, statErr := os.Stat(adapter); statErr != nil {
				if os.IsNotExist(statErr) {
					return nil, fmt.Errorf("%w (model[%d] adapter %q)", errdefs.ErrModelAdapterNotFound, i, adapter)
				}
				return nil, fmt.Errorf("failed to stat model[%d] adapter %q: %w", i, adapter, statErr)
			}
		}

		target := strings.TrimSpace(m.Target)
		if target == "" {
			target = defaultModelTarget
		}
		if !filepath.IsAbs(target) {
			return nil, fmt.Errorf("%w (model[%d] target %q)", errdefs.ErrModelTargetNotAbsolute, i, target)
		}

		mode := strings.ToLower(strings.TrimSpace(m.Mode))
		if _, ok := modelModes[mode]; !ok {
			return nil, fmt.Errorf("%w (model[%d] mode %q)", errdefs.ErrModelModeUnknown, i, mode)
		}

		if len(m.Devices) > maxModelDevices {
			return nil, fmt.Errorf("%w (model[%d] devices %v)", errdefs.ErrModelDevicesInvalid, i, m.Devices)
		}
		devSeen := make(map[int]struct{}, len(m.Devices))
		for _, d := range m.Devices {
			if _, dup := devSeen[d]; d < 0 || dup {
				return nil, fmt.Errorf("%w (model[%d] devices %v)", errdefs.ErrModelDevicesInvalid, i, m.Devices)
			}
			devSeen[d] = struct{}{}
		}

		if m.Layers != nil && (len(m.Layers) != 2 || m.Layers[0] < 0 || m.Layers[0] >= m.Layers[1] || int64(m.Layers[1]) > math.MaxUint32) {
			return nil, fmt.Errorf("%w (model[%d] layers %v)", errdefs.ErrModelLayersInvalid, i, m.Layers)
		}

		for k := range m.Options {
			if _, ok := modelOptionFlags[k]; !ok {
				return nil, fmt.Errorf("%w (model[%d] option %q)", errdefs.ErrModelOptionUnknown, i, k)
			}
		}

		out[i] = intmodel.ModelMount{Name: name, Source: src, Target: target, Mode: mode, Devices: append([]int(nil), m.Devices...), Options: m.Options,
			Layers: append([]int(nil), m.Layers...), Adapter: adapter}
	}
	return out, nil
}

// modelLoadLayers turns the validated layers into the stage the load selects (the zero value: the whole checkpoint).
func modelLoadLayers(m intmodel.ModelMount) gpupool.Layers {
	if len(m.Layers) != 2 {
		return gpupool.Layers{}
	}
	return gpupool.Layers{Begin: uint32(m.Layers[0]), End: uint32(m.Layers[1])}
}

// modelLoadFlags folds the validated options into kk_load_opts.flags.
func modelLoadFlags(m intmodel.ModelMount) uint32 {
	var f uint32
	for k, on := range m.Options {
		if on {
			f |= modelOptionFlags[k]
		}
	}
	return f
}
