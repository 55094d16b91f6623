// NOT COMPILED HERE (no Go toolchain) — reviewed source; see host/go/README.md.

package model

import (
	"encoding/json"
	"fmt"
	"strconv"
	"strings"

	getshared "github.com/eminwux/kukeon/cmd/kuke/get/shared"
	"github.com/eminwux/kukeon/internal/gpupool"
	"github.com/spf13/cobra"
)

// NewPlanCmd builds `kuke model plan <path>`: the dry run of a load — pool layout and bytes per GPU — before any device is touched, so a
// cell manifest can be sized against the daemon's pool budget.
func NewPlanCmd() *cobra.Command {
	cmd := &cobra.Command{
		Use:           "plan <path>",
		Short:         "Dry-run a model load: bytes each GPU ingests and holds",
		Args:          cobra.ExactArgs(1),
		SilenceUsage:  true,
		SilenceErrors: false,
		RunE: func(cmd *cobra.Command, args []string) error {
			outputFormat, err := getshared.ParseOutputFormat(cmd)
			if err != nil {
				return err
			}
			modeName, _ := cmd.Flags().GetString("mode")
			gpus, _ := cmd.Flags().GetInt("gpus")
			full, _ := cmd.Flags().GetBool("full")
			modes := map[string]gpupool.Mode{"single": gpupool.ModeSingle, "broadcast": gpupool.ModeBroadcast, "scatter": gpupool.ModeScatter}
			mode, ok := modes[strings.ToLower(strings.TrimSpace(modeName))]
			if !ok {
				return fmt.Errorf("invalid mode: %s (supported: single, broadcast, scatter)", modeName)
			}
			if mode == gpupool.ModeSingle {
				gpus = 1
			}
			var layers gpupool.Layers
			if s, _ := cmd.Flags().GetString("layers"); s != "" {
				b, e, found := strings.Cut(s, ":")
				lb, berr := strconv.ParseUint(b, 10, 32)
				le, eerr := strconv.ParseUint(e, 10, 32)
				if !found || berr != nil || eerr != nil || lb >= le {
					return fmt.Errorf("invalid layer range: %s (expected B:E with integers 0 <= B < E)", s)
				}
				layers = gpupool.Layers{Begin: uint32(lb), End: uint32(le)}
			}
			raw, err := resolveIndexer(cmd).Plan(strings.TrimSpace(args[0]), mode, 0, gpus, layers)
			if err != nil {
				return err
			}
			if full && outputFormat != getshared.OutputFormatTable {
				var doc interface{}
				if uerr := json.Unmarshal(raw, &doc); uerr != nil {
					return uerr
				}
				if outputFormat == getshared.OutputFormatJSON {
					return getshared.PrintJSON(doc)
				}
				return getshared.PrintYAML(doc)
			}
			var doc planDoc
			if uerr := json.Unmarshal(raw, &doc); uerr != nil {
				return uerr
			}
			sum := planSummary{Path: args[0], Mode: strings.ToLower(modeName), GPUs: gpus, FileBytes: doc.FileBytes, Layers: doc.Layers, NLayers: doc.NLayers}
			if len(doc.Layouts) > 0 {
				sum.Tensors = len(doc.Layouts[0].Tensors)
			}
			for g := 0; g < gpus; g++ {
				layout := 0
				if mode == gpupool.ModeScatter {
					layout = g
				}
				sum.PoolBytesPerGPU = append(sum.PoolBytesPerGPU, doc.Layouts[layout].PoolBytes)
				sum.IngestBytesPerGPU = append(sum.IngestBytesPerGPU, doc.Parts[g].SrcBytes)
			}
			switch outputFormat {
			case getshared.OutputFormatJSON:
				return getshared.PrintJSON(sum)
			case getshared.OutputFormatYAML:
				return getshared.PrintYAML(sum)
			default:
				rows := make([][]string, 0, gpus)
				for g := 0; g < gpus; g++ {
					rows = append(rows, []string{strconv.Itoa(g), formatSize(int64(sum.IngestBytesPerGPU[g])), formatSize(int64(sum.PoolBytesPerGPU[g]))})
				}
				getshared.PrintTable(cmd, []string{"GPU", "INGESTS", "POOL"}, rows)
				stage := ""
				if len(sum.Layers) == 2 {
					stage = fmt.Sprintf(", layers %d-%d of %d", sum.Layers[0], sum.Layers[1]-1, sum.NLayers)
				}
				cmd.Printf("%d tensors, %s in the files, mode %s%s\n", sum.Tensors, formatSize(int64(sum.FileBytes)), sum.Mode, stage)
				return nil
			}
		},
	}
	cmd.Flags().String("mode", "single", "Load mode: single, broadcast, scatter")
	cmd.Flags().Int("gpus", 1, "Number of GPUs the load is planned for")
	cmd.Flags().String("layers", "", "Pipeline stage B:E: plan only layers [B, E) of the checkpoint")
	cmd.Flags().Bool("full", false, "yaml/json: print the whole plan (chunks, reads, segments) instead of the summary")
	cmd.Flags().StringP("output", "o", "", "Output format (yaml, json, table). Default: table")
	return cmd
}
