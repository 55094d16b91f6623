// PEFT LoRA adapters (kk_load_adapter, kk_adapter_describe): parse adapter_config.json + adapter_model.safetensors and match the pairs
// against the plan of a load.  Host only, no CUDA: kk_adapter_describe runs exactly this, so the CPU tier sees what a load merges.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "kk_plan.hpp"

namespace kk {

// One lora_A / lora_B pair and the pool tensor it targets.
struct LoraPair {
  std::string module;  // <M>: the keys are base_model.model.<M>.lora_{A,B}.weight, the target <M>.weight
  uint32_t tensor = 0; // index of the target in the plan's index
  TensorRec a, b;      // in the adapter file: A [r, C], B [R, r]
  uint32_t r = 0;
  float s = 0.f;       // lora_alpha / r (lora_alpha / sqrt(r) under use_rslora), in double, rounded once
};

struct Adapter {
  std::string path;   // the adapter as given, made absolute (part of the model's identity)
  std::string file;   // adapter_model.safetensors
  double alpha = 0;
  bool rslora = false;
  std::vector<LoraPair> pairs;        // targets the load holds, in index order
  std::vector<std::string> skipped;   // targets in the checkpoint but outside the load's layer stage
};

// The refusals that follow from the load options alone (KK_EUNSUPPORTED): KK_FANOUT_NVLS, and a part_count > 1 load whose pool receives
// peers' stores (BROADCAST, or SCATTER with KK_LOAD_SCATTER_EXCHANGE).
void check_adapter_opts(const kk_load_opts& opts);

// Parse the adapter at `adapter_path` (its directory, or its adapter_model.safetensors with the config beside it) and match it against P,
// the plan of checkpoint `ckpt_path` loaded with `flags` (the rules and every refusal: kk_load_adapter in kukeon_gpuload.h).  Throws kk::Error.
Adapter match_adapter(const std::string& adapter_path, const std::string& ckpt_path, uint32_t flags, const Plan& P);

// kk_adapter_describe's JSON.
std::string adapter_to_json(const Adapter& A, const Plan& P);

// KK_LORA_BF16 / KK_LORA_F16 / KK_LORA_F32 for a pool dtype (one of KK_BF16, KK_F16, KK_F32).
uint32_t lora_out_of(uint32_t pool_dtype);

// Every A and B of A.pairs read from the adapter file and widened to fp32 (exact), back to back; a_off[i] / b_off[i] index them.
std::vector<float> read_adapter_f32(const Adapter& A, std::vector<uint64_t>& a_off, std::vector<uint64_t>& b_off);

}  // namespace kk
