// NOT COMPILED HERE (no Go toolchain) — reviewed source; see host/go/README.md.

// Package model hosts the `kuke model` parent command.  `pull` and `plan` belong to the daemon-independent, in-process category
// `kuke image *` defines (cmd/kuke/image/image.go): they read checkpoint files and call the CPU-only entry points of
// libkukeon_gpuload (kk_index, kk_plan_describe) — no GPU, no kukeond.  The verbs that act on resident pools (`load`, `get`, `rm`) are
// daemon RPCs, because a pool lives exactly as long as kukeond does (internal/daemon/server.go:87,242); they are not in this package.
package model

import (
	"encoding/json"

	"github.com/eminwux/kukeon/internal/gpupool"
	"github.com/spf13/cobra"
)

// MockIndexerKey injects a fake Indexer via context for tests (the MockControllerKey pattern of cmd/kuke/image/image.go).
type MockIndexerKey struct{}

// Indexer is the narrow surface the subcommands use; satisfied by the cgo package and by per-test fakes.
type Indexer interface {
	Index(path string) ([]gpupool.TensorMeta, error)
	Plan(path string, mode gpupool.Mode, flags uint32, gpus int, layers gpupool.Layers) ([]byte, error)
}

type cgoIndexer struct{}

func (cgoIndexer) Index(path string) ([]gpupool.TensorMeta, error) { return gpupool.Index(path) }
func (cgoIndexer) Plan(path string, mode gpupool.Mode, flags uint32, gpus int, layers gpupool.Layers) ([]byte, error) {
	return gpupool.Plan(path, mode, flags, gpus, layers)
}

func resolveIndexer(cmd *cobra.Command) Indexer {
	if m, ok := cmd.Context().Value(MockIndexerKey{}).(Indexer); ok {
		return m
	}
	return cgoIndexer{}
}

// NewModelCmd builds `kuke model`.
func NewModelCmd() *cobra.Command {
	cmd := &cobra.Command{
		Use:           "model",
		Short:         "Inspect model checkpoints for GPU-resident loading",
		SilenceUsage:  true,
		SilenceErrors: false,
	}
	cmd.AddCommand(NewPullCmd(), NewPlanCmd())
	return cmd
}

// planSummary is what `kuke model plan` prints unless --full is given.
type planSummary struct {
	Path              string   `json:"path"              yaml:"path"`
	Mode              string   `json:"mode"              yaml:"mode"`
	GPUs              int      `json:"gpus"              yaml:"gpus"`
	FileBytes         uint64   `json:"fileBytes"         yaml:"fileBytes"`
	PoolBytesPerGPU   []uint64 `json:"poolBytesPerGpu"   yaml:"poolBytesPerGpu"`
	IngestBytesPerGPU []uint64 `json:"ingestBytesPerGpu" yaml:"ingestBytesPerGpu"`
	Tensors           int      `json:"tensors"           yaml:"tensors"`
	Layers            []uint32 `json:"layers,omitempty"  yaml:"layers,omitempty"`
	NLayers           uint64   `json:"nLayers,omitempty" yaml:"nLayers,omitempty"`
}

// planDoc mirrors the fields of kk_plan_describe's JSON the summary needs.
type planDoc struct {
	FileBytes uint64   `json:"file_bytes"`
	Layers    []uint32 `json:"layers"`
	NLayers   uint64   `json:"n_layers"`
	Layouts   []struct {
		PoolBytes uint64            `json:"pool_bytes"`
		Tensors   []json.RawMessage `json:"tensors"`
	} `json:"layouts"`
	Parts []struct {
		SrcBytes uint64 `json:"src_bytes"`
	} `json:"parts"`
}
