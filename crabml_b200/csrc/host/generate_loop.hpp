// generate_loop.hpp -- the decode loop behind ccr_runner_generate_greedy_ex (llama2_runner.cpp) and ccr_runner_generate_ex
// (llama2_sampler.cpp), parameterised by the sampler of one step.
#pragma once
#include <functional>

#include "../../../include/crabml_runner.h"
#include "cuda_tensor.hpp"

// samples generated token `index` from `logits` into device slot 0 and history[index]
using ccr_step_sampler = std::function<void(const crabml::CudaTensor& logits, int64_t index)>;

int ccr_runner_fail(ccr_runner* r, int code, const char* msg);      // records msg as the last error, returns code
int ccr_runner_generate_loop(ccr_runner* r, const int64_t* prompt, int32_t n_prompt, int32_t steps, int64_t eos_token, int64_t* out_tokens,
                             int32_t* n_out, float* logits_out, const ccr_step_sampler& pick);
