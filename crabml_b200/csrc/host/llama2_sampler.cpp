// llama2_sampler.cpp -- generation with Llama2Sampler (crabml-llama2/src/sampler.rs:27-107): the greedy decode loop with the
// temperature / top-p sampler of the device (cc_sample_to_slot) in place of the argmax.
#include "generate_loop.hpp"

using crabml::CudaTensor;

extern "C" CC_API int ccr_runner_generate_ex(ccr_runner* r, const int64_t* prompt, int32_t n_prompt, int32_t steps, int64_t eos_token,
                                             float temperature, float topp, uint64_t seed, int64_t* out_tokens, int32_t* n_out, float* logits_out) {
    if (!r) return CC_ERR_ARG;
    // checked before the prompt runs: a rejected setting must not leave the KV cache grown
    if (!(temperature >= 0.0f) || topp != topp) {
        if (n_out) *n_out = 0;
        return ccr_runner_fail(r, CC_ERR_TENSOR, "generate: temperature must be a number >= 0 and topp must not be NaN");
    }
    if (temperature == 0.0f)                      // sampler.rs:28-30: the greedy loop, op for op
        return ccr_runner_generate_loop(r, prompt, n_prompt, steps, eos_token, out_tokens, n_out, logits_out,
                                        [](const CudaTensor& lg, int64_t i) { lg.argmax_to_slot(0, i); });
    // coin index = generated-token index: one seed reproduces one run in every execution mode (and on every rank of a sharded run,
    // whose gathered logits are identical)
    return ccr_runner_generate_loop(r, prompt, n_prompt, steps, eos_token, out_tokens, n_out, logits_out,
                                    [=](const CudaTensor& lg, int64_t i) { lg.sample_to_slot(temperature, topp, seed, i, 0, i); });
}
