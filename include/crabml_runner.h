/*
 * crabml_runner.h -- C entry points of the C++ host driver that replays crabml-llama2's Llama2Runner
 * (crabml-llama2/src/llama2.rs:45-281,527-638) over the C ABI of crabml_cuda.h.
 *
 * The reference's runner is Rust and generic over `T: Tensor`; with a Rust toolchain it is used unchanged
 * (INTEGRATION.md).  This image has no Rust, so the same op sequence is replayed from C++
 * (crabml_b200/csrc/host/llama2_runner.cpp) for the end-to-end tests and bench.py.  Not part of the
 * drop-in boundary.
 */
#ifndef CRABML_RUNNER_H
#define CRABML_RUNNER_H

#include "crabml_cuda.h"

#ifdef __cplusplus
extern "C" {
#endif

/* LlamaConfig, crabml-llama2/src/model.rs:30-53 (llama architecture subset) */
typedef struct ccr_llama_config {
    int32_t n_heads, n_kv_heads, n_layers, embedding_dim, hidden_dim, seq_len, vocab_size;
    int32_t rope_dim;          /* <= 0: use head_dim (llama2.rs:218) */
    float rms_norm_eps;
    int32_t use_f16_kv_cache;  /* llama2.rs:51-55 */
    /* sharded decode (not in the reference: SURVEY 8e).  shard_world <= 1: single device.  Otherwise the weights passed to
     * ccr_runner_create are THIS rank's shards (crabml_b200/sharding.py) and hidden_local is its share of hidden_dim. */
    int32_t shard_rank, shard_world, hidden_local;
    /* ModelArchitecture (model.rs:21-27): which forward replays -- 0 llama (llama2.rs:213-281), 1 qwen2 (:283-352: q/k/v bias adds, Neox
     * RoPE), 2 gemma (:455-524: embedding scaled by sqrt(dim), Neox RoPE, GeLU ffn, tied classifier) */
    int32_t arch;
} ccr_llama_config;
#define CCR_ARCH_LLAMA 0
#define CCR_ARCH_QWEN2 1
#define CCR_ARCH_GEMMA 2

/* LlamaWeights<T>, model.rs:55-84; arrays have n_layers entries; output_weight may be NULL (llama2.rs:201-206) */
typedef struct ccr_llama_weights {
    cc_buf* token_embed;
    cc_buf* const* wq; cc_buf* const* wk; cc_buf* const* wv; cc_buf* const* wo;
    cc_buf* const* ffn_gate; cc_buf* const* ffn_down; cc_buf* const* ffn_up;
    cc_buf* const* rms_att; cc_buf* const* rms_ffn;
    cc_buf* rms_final;
    cc_buf* output_weight;
    cc_buf* const* bq; cc_buf* const* bk; cc_buf* const* bv;      /* qwen2 only (model.rs bq/bk/bv), else NULL */
} ccr_llama_weights;

typedef struct ccr_runner ccr_runner;

CC_API int ccr_runner_create(cc_device* dev, const ccr_llama_config* conf, const ccr_llama_weights* w,
                             int32_t kv_seq_len, ccr_runner** out);
CC_API void ccr_runner_destroy(ccr_runner* r);
CC_API const char* ccr_runner_last_error(ccr_runner* r);
/* Llama2Runner::forward (llama2.rs:184-211): n_tokens tokens at position pos; logits of the last token are
 * exported to logits_out (vocab_size floats) unless it is NULL (then nothing is copied to the host). */
CC_API int ccr_runner_forward(ccr_runner* r, const int64_t* tokens, int32_t n_tokens, int64_t pos, float* logits_out);
CC_API int64_t ccr_runner_kv_cache_len(ccr_runner* r);                /* llama2.rs:107-109 */
/* greedy decode loop (prefill + generate with temperature 0: llama2.rs:111-172, sampler.rs:109-116):
 * feeds `prompt`, then generates up to `steps` tokens into out_tokens; returns the count via *n_out. */
CC_API int ccr_runner_generate_greedy(ccr_runner* r, const int64_t* prompt, int32_t n_prompt, int32_t steps,
                                      int64_t eos_token, int64_t* out_tokens, int32_t* n_out);

/* the same loop with the logits of every generated position exported asynchronously (logits_out: steps x vocab floats, may be
 * NULL).  Sampling runs on the device (cc_argmax_to_slot) and the sampled id feeds the next step from a device slot: with
 * eos_token < 0 no step waits for the host. */
CC_API int ccr_runner_generate_greedy_ex(ccr_runner* r, const int64_t* prompt, int32_t n_prompt, int32_t steps,
                                         int64_t eos_token, int64_t* out_tokens, int32_t* n_out, float* logits_out);

/* the same loop with Llama2Sampler (sampler.rs:27-107: temperature, top-p) in place of the argmax, on the device
 * (cc_sample_to_slot); the coin of generated token i is coin_index i of `seed`.  temperature == 0 is
 * ccr_runner_generate_greedy_ex, bit for bit.  A NaN or negative temperature or a NaN topp is CC_ERR_TENSOR. */
CC_API int ccr_runner_generate_ex(ccr_runner* r, const int64_t* prompt, int32_t n_prompt, int32_t steps, int64_t eos_token,
                                  float temperature, float topp, uint64_t seed, int64_t* out_tokens, int32_t* n_out, float* logits_out);

#ifdef __cplusplus
}
#endif
#endif
