// llama2_runner.cpp -- replay of crabml-llama2's Llama2Runner<T> with T = CudaTensor.
// The op ORDER is the reference's, verbatim (llama2.rs:184-281 forward/forward_llama, :527-603 attention,
// :605-638 ffn); this file contains no arithmetic of its own.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../../include/crabml_runner.h"
#include "cuda_tensor.hpp"
#include "generate_loop.hpp"

using crabml::CudaTensor;
using crabml::TensorStrider;

struct ccr_runner {
    cc_device* dev = nullptr;
    ccr_llama_config conf{};
    CudaTensor token_embed, rms_final, output_weight;
    std::vector<CudaTensor> wq, wk, wv, wo, ffn_gate, ffn_down, ffn_up, rms_att, rms_ffn, bq, bk, bv;
    std::vector<CudaTensor> key_cache, value_cache;       // (layer) x [n_kv_heads, seq, head_dim]
    std::vector<float> logits;
    float* pinned_logits = nullptr;       // staging ring of the asynchronous logits export (generate_greedy_ex), grown on demand
    size_t pinned_floats = 0;
    std::string last_error;
    ~ccr_runner() { if (pinned_logits) cc_host_free(dev, pinned_logits); }

    // Sharded decode (SURVEY 8e).  shard_world > 1: this process holds heads [rank*H/N, (rank+1)*H/N) of wq/wk/wv (rows), the
    // matching COLUMNS of wo, hidden_local rows of gate/up and columns of down, vocab/N rows of the classifier; the replay is
    // the reference's op order with one all_reduce_sum after wo and after ffn_down and one all_gather of the logits.
    int world() const { return conf.shard_world > 1 ? conf.shard_world : 1; }
    int local_heads() const { return conf.n_heads / world(); }
    int local_kv_heads() const { return conf.n_kv_heads / world(); }
    int head_size() const { return conf.embedding_dim / conf.n_heads; }
    int64_t kv_cache_len() const { return key_cache[0].shape()[1]; }

    CudaTensor forward_llama(const std::vector<int64_t>& tokens, int64_t pos, int slot = -1);
    CudaTensor forward_arch(const std::vector<int64_t>& tokens, int64_t pos, int slot = -1);
    CudaTensor forward_qwen2(const std::vector<int64_t>& tokens, int64_t pos, int slot);
    CudaTensor forward_gemma(const std::vector<int64_t>& tokens, int64_t pos, int slot);
    CudaTensor logits_tensor(CudaTensor x, int64_t n_batch);
    void decode_step(const int64_t* token, int64_t pos, int64_t hist_index, float* logits_async, const ccr_step_sampler& pick);
    CudaTensor forward_multi_query_attention(CudaTensor q, CudaTensor k, CudaTensor v, int l, int64_t n_batch);
    CudaTensor forward_ffn(CudaTensor x, int l, bool gelu = false);
    void forward(const std::vector<int64_t>& tokens, int64_t pos, float* logits_out);
};

// llama2.rs:195-208: last row -> classifier (-> gather of the vocab/N slices on the sharded path)
CudaTensor ccr_runner::logits_tensor(CudaTensor x, int64_t n_batch) {
    CudaTensor x_final = CudaTensor::alloc({conf.embedding_dim}, CC_F32, dev);
    x_final.copy_rows_from(x, {n_batch - 1});
    const CudaTensor& ow = output_weight.valid() ? output_weight : token_embed;
    CudaTensor lg = ow.matmul_vec(x_final);
    if (world() > 1) {                                   // row-split classifier: gather the vocab/N slices
        CudaTensor full = CudaTensor::alloc({conf.vocab_size}, CC_F32, dev);
        full.all_gather_from(lg);
        lg = std::move(full);
    }
    return lg;
}

// llama2.rs:184-211
void ccr_runner::forward(const std::vector<int64_t>& tokens, int64_t pos, float* logits_out) {
    CudaTensor lg = logits_tensor(forward_arch(tokens, pos), (int64_t)tokens.size());
    if (logits_out) lg.export_to(logits_out, (size_t)conf.vocab_size);
    else CudaTensor::check(dev, cc_device_flush(dev));     // lazy mode: submit this token's work without a host sync
}

// One decode step whose sampled token never visits the host: forward (token from the host, or -- token == nullptr -- from device slot 0),
// the sampler (greedy: argmax, sampler.rs:109-116) into slot 0 and the device-side history; optionally the logits are exported WITHOUT waiting.
void ccr_runner::decode_step(const int64_t* token, int64_t pos, int64_t hist_index, float* logits_async, const ccr_step_sampler& pick) {
    CudaTensor x = token ? forward_arch({*token}, pos) : forward_arch({0}, pos, 0);
    CudaTensor lg = logits_tensor(std::move(x), 1);
    pick(lg, hist_index);
    if (logits_async) lg.export_async(logits_async, (size_t)conf.vocab_size);     // flushes (asynchronously) as well
    else CudaTensor::check(dev, cc_device_flush(dev));
}

// llama2.rs:213-281
CudaTensor ccr_runner::forward_llama(const std::vector<int64_t>& tokens, int64_t pos, int slot) {
    const int64_t embed_dim = conf.embedding_dim, n_heads = local_heads(), n_kv_heads = local_kv_heads();
    const int64_t head_dim = head_size();
    const int64_t rope_dim = conf.rope_dim > 0 ? conf.rope_dim : head_dim;
    const int64_t n_batch = (int64_t)tokens.size();

    CudaTensor x = CudaTensor::alloc({n_batch, embed_dim}, CC_F32, dev);
    if (slot >= 0) x.copy_rows_from_slot(token_embed, slot);      // the id sampled on the device by the previous step
    else x.copy_rows_from(token_embed, tokens);

    for (int l = 0; l < conf.n_layers; l++) {
        CudaTensor x_attn_orig = x.dup();
        x = std::move(x).rms_norm_inplace(conf.rms_norm_eps);
        x = std::move(x).mul_inplace(rms_att[l]);
        x = std::move(x).with_name("attn_rmsnorm:" + std::to_string(l) + ":" + std::to_string(pos));
        x = std::move(x).with_name("x_debug:" + std::to_string(l) + ":" + std::to_string(pos));

        CudaTensor q = wq[l].matmul_vec(x);
        CudaTensor k = wk[l].matmul_vec(x);
        CudaTensor v = wv[l].matmul_vec(x);

        q = std::move(q).reshape({n_batch, n_heads, head_dim});
        k = std::move(k).reshape({n_batch, n_kv_heads, head_dim});
        q = std::move(q).rope_inplace(CC_ROPE_LLAMA, pos, rope_dim);
        k = std::move(k).rope_inplace(CC_ROPE_LLAMA, pos, rope_dim);

        x = forward_multi_query_attention(std::move(q), std::move(k), std::move(v), l, n_batch);
        if (world() > 1) x = std::move(x).all_reduce_sum_inplace();      // column-split wo: sum the [dim] partials
        x = std::move(x).with_name("attn_out:" + std::to_string(l) + ":" + std::to_string(pos));
        x = std::move(x).add_inplace(x_attn_orig);
        x = forward_ffn(std::move(x), l);
        x = std::move(x).with_name("ffn_out:" + std::to_string(l) + ":" + std::to_string(pos));
    }
    x = std::move(x).rms_norm_inplace(conf.rms_norm_eps);
    x = std::move(x).mul_inplace(rms_final);
    return std::move(x).with_name("final_rmsnorm:" + std::to_string(pos));
}

// llama2.rs:186-192: dispatch on the model architecture
CudaTensor ccr_runner::forward_arch(const std::vector<int64_t>& tokens, int64_t pos, int slot) {
    switch (conf.arch) {
    case CCR_ARCH_QWEN2: return forward_qwen2(tokens, pos, slot);
    case CCR_ARCH_GEMMA: return forward_gemma(tokens, pos, slot);
    default: return forward_llama(tokens, pos, slot);
    }
}

// llama2.rs:283-352
CudaTensor ccr_runner::forward_qwen2(const std::vector<int64_t>& tokens, int64_t pos, int slot) {
    const int64_t embed_dim = conf.embedding_dim, n_heads = local_heads(), n_kv_heads = local_kv_heads();
    const int64_t head_dim = head_size();
    const int64_t rope_dim = conf.rope_dim > 0 ? conf.rope_dim : head_dim;
    const int64_t n_batch = (int64_t)tokens.size();

    CudaTensor x = CudaTensor::alloc({n_batch, embed_dim}, CC_F32, dev);
    if (slot >= 0) x.copy_rows_from_slot(token_embed, slot);
    else x.copy_rows_from(token_embed, tokens);

    for (int l = 0; l < conf.n_layers; l++) {
        CudaTensor x_attn_orig = x.dup();
        x = std::move(x).rms_norm_inplace(conf.rms_norm_eps);
        x = std::move(x).mul_inplace(rms_att[l]);
        x = std::move(x).with_name("attn_rmsnorm:" + std::to_string(l) + ":" + std::to_string(pos));

        CudaTensor q = wq[l].matmul_vec(x);
        CudaTensor k = wk[l].matmul_vec(x);
        CudaTensor v = wv[l].matmul_vec(x);
        q = std::move(q).add_inplace(bq[l]);
        k = std::move(k).add_inplace(bk[l]);
        v = std::move(v).add_inplace(bv[l]);

        q = std::move(q).reshape({n_batch, n_heads, head_dim});
        k = std::move(k).reshape({n_batch, n_kv_heads, head_dim});
        q = std::move(q).rope_inplace(CC_ROPE_NEOX, pos, rope_dim);
        k = std::move(k).rope_inplace(CC_ROPE_NEOX, pos, rope_dim);

        x = forward_multi_query_attention(std::move(q), std::move(k), std::move(v), l, n_batch);
        x = std::move(x).with_name("attn_out:" + std::to_string(l) + ":" + std::to_string(pos));
        x = std::move(x).add_inplace(x_attn_orig);
        x = forward_ffn(std::move(x), l, false);
        x = std::move(x).with_name("ffn_out:" + std::to_string(l) + ":" + std::to_string(pos));
    }
    x = std::move(x).rms_norm_inplace(conf.rms_norm_eps);
    x = std::move(x).mul_inplace(rms_final);
    return std::move(x).with_name("final_rmsnorm:" + std::to_string(pos));
}

// llama2.rs:455-524
CudaTensor ccr_runner::forward_gemma(const std::vector<int64_t>& tokens, int64_t pos, int slot) {
    const int64_t embed_dim = conf.embedding_dim, n_heads = local_heads(), n_kv_heads = local_kv_heads();
    const int64_t head_dim = head_size();
    const int64_t rope_dim = conf.rope_dim > 0 ? conf.rope_dim : head_dim;
    const int64_t n_batch = (int64_t)tokens.size();

    CudaTensor x = CudaTensor::alloc({n_batch, embed_dim}, CC_F32, dev);
    if (slot >= 0) x.copy_rows_from_slot(token_embed, slot);
    else x.copy_rows_from(token_embed, tokens);
    // GEMMA: the embedding is scaled by sqrt(embed_dim)
    x = std::move(x).scale_inplace(std::sqrt((float)embed_dim));
    x = std::move(x).with_name("scaled_embed");

    for (int l = 0; l < conf.n_layers; l++) {
        CudaTensor x_attn_orig = x.dup();
        x = std::move(x).rms_norm_inplace(conf.rms_norm_eps);
        x = std::move(x).mul_inplace(rms_att[l]);
        x = std::move(x).with_name("attn_rmsnorm:" + std::to_string(l) + ":" + std::to_string(pos));

        CudaTensor q = wq[l].matmul_vec(x);
        CudaTensor k = wk[l].matmul_vec(x);
        CudaTensor v = wv[l].matmul_vec(x);

        q = std::move(q).reshape({n_heads, head_dim});
        k = std::move(k).reshape({n_kv_heads, head_dim});
        q = std::move(q).rope_inplace(CC_ROPE_NEOX, pos, rope_dim);
        k = std::move(k).rope_inplace(CC_ROPE_NEOX, pos, rope_dim);

        x = forward_multi_query_attention(std::move(q), std::move(k), std::move(v), l, n_batch);
        x = std::move(x).add_inplace(x_attn_orig);
        x = forward_ffn(std::move(x), l, true);
        x = std::move(x).with_name("ffn_out:" + std::to_string(l) + ":" + std::to_string(pos));
    }
    x = std::move(x).rms_norm_inplace(conf.rms_norm_eps);
    x = std::move(x).mul_inplace(rms_final);
    return std::move(x).with_name("final_rmsnorm:" + std::to_string(pos));
}

// llama2.rs:527-603
CudaTensor ccr_runner::forward_multi_query_attention(CudaTensor q, CudaTensor k, CudaTensor v, int l, int64_t n_batch) {
    const int64_t n_heads = local_heads(), n_kv_heads = local_kv_heads(), head_dim = head_size(), embed_dim = n_heads * head_dim;
    {
        CudaTensor kt = std::move(k).reshape({n_batch, n_kv_heads, head_dim}).transpose({1, 0, 2});
        CudaTensor vt = std::move(v).reshape({n_batch, n_kv_heads, head_dim}).transpose({1, 0, 2});
        key_cache[l].concatenate(kt, 1);
        value_cache[l].concatenate(vt, 1);
    }
    q = std::move(q).reshape({n_batch, n_heads, head_dim}).transpose({1, 0, 2}).contiguous().scale_inplace(1.0f / std::sqrt((float)head_dim));

    CudaTensor k_cache = std::move(key_cache[l]);
    TensorStrider k_strider_orig = k_cache.strider();
    k_cache = std::move(k_cache).transpose({0, 2, 1});
    CudaTensor attn = q.batch_matmul(k_cache);
    attn = std::move(attn).softmax_inplace(2);
    key_cache[l] = std::move(k_cache).with_strider(k_strider_orig);

    CudaTensor v_cache = std::move(value_cache[l]);
    TensorStrider v_strider_orig = v_cache.strider();
    CudaTensor x_with_attn = attn.batch_matmul(v_cache);
    if (n_batch == 1) x_with_attn = std::move(x_with_attn).reshape({n_batch, embed_dim});
    else x_with_attn = std::move(x_with_attn).transpose({1, 0, 2}).contiguous().reshape({n_batch, embed_dim});
    value_cache[l] = std::move(v_cache).with_strider(v_strider_orig);
    return wo[l].matmul_vec(x_with_attn);
}

// llama2.rs:605-638
CudaTensor ccr_runner::forward_ffn(CudaTensor x, int l, bool gelu) {
    CudaTensor x_orig_ffn = x.dup();
    x = std::move(x).rms_norm_inplace(1e-5f);              // literal in the reference (quirk B5)
    x = std::move(x).mul_inplace(rms_ffn[l]);
    CudaTensor h1 = ffn_gate[l].matmul_vec(x);
    CudaTensor h2 = ffn_up[l].matmul_vec(x);
    h1 = gelu ? std::move(h1).gelu_inplace() : std::move(h1).silu_inplace();      // Activation::{SiLU, GeLU} (llama2.rs:624-628)
    h1 = std::move(h1).mul_inplace(h2);
    x = ffn_down[l].matmul_vec(h1);
    if (world() > 1) x = std::move(x).all_reduce_sum_inplace();          // column-split ffn_down
    x = std::move(x).add_inplace(x_orig_ffn);
    return x;
}

static int64_t sample_argmax(const std::vector<float>& logits) {       // sampler.rs:109-116: max_by keeps the LAST maximum
    int64_t best = 0;
    for (int64_t i = 1; i < (int64_t)logits.size(); i++)
        if (!(logits[i] < logits[best])) best = i;
    return best;
}

template <class F>
static int guarded(ccr_runner* r, F&& f) {
    try {
        f();
        return CC_OK;
    } catch (const crabml::TensorError& e) {
        if (r) r->last_error = e.what();
        return CC_ERR_TENSOR;
    } catch (const std::exception& e) {
        if (r) r->last_error = e.what();
        return CC_ERR_ARG;
    }
}

extern "C" CC_API int ccr_runner_create(cc_device* dev, const ccr_llama_config* conf, const ccr_llama_weights* w,
                                        int32_t kv_seq_len, ccr_runner** out) {
    if (!dev || !conf || !w || !out) return CC_ERR_ARG;
    ccr_runner* r = new ccr_runner();
    r->dev = dev;
    r->conf = *conf;
    int rc = guarded(r, [&] {
        const int N = r->world();
        const int64_t dim = conf->embedding_dim, hd = dim / conf->n_heads;
        const int64_t q_dim = hd * r->local_heads(), kv_dim = hd * r->local_kv_heads();
        const int64_t hidden = N > 1 ? conf->hidden_local : conf->hidden_dim, vocab_rows = conf->vocab_size / N;
        if (conf->arch < CCR_ARCH_LLAMA || conf->arch > CCR_ARCH_GEMMA) throw crabml::TensorError("unknown architecture id");
        if (N > 1 && conf->arch != CCR_ARCH_LLAMA) throw crabml::TensorError("sharding: only the llama forward is sharded");
        if (N > 1) {
            if (conf->n_heads % N || conf->n_kv_heads % N || conf->vocab_size % N) throw crabml::TensorError("sharding: heads / kv heads / vocab must divide by the world size");
            // the F32-cache attention of the reference pairs query head h with kv head h % n_kv (batch_matmul.rs:47-71, quirk B13):
            // contiguous head ranges keep that mapping local only without grouping
            if (conf->n_heads != conf->n_kv_heads && !conf->use_f16_kv_cache) throw crabml::TensorError("sharding: grouped-query models need the f16 kv cache (contiguous kv groups)");
            if (!w->output_weight) throw crabml::TensorError("sharding: tied classifier is not supported (pass a row shard as output_weight)");
            if (hidden <= 0) throw crabml::TensorError("sharding: hidden_local missing");
        }
        r->token_embed = CudaTensor::wrap(dev, w->token_embed, {conf->vocab_size, dim});
        r->rms_final = CudaTensor::wrap(dev, w->rms_final, {dim});
        if (w->output_weight) r->output_weight = CudaTensor::wrap(dev, w->output_weight, {vocab_rows, dim});
        for (int l = 0; l < conf->n_layers; l++) {
            r->wq.push_back(CudaTensor::wrap(dev, w->wq[l], {q_dim, dim}));
            r->wk.push_back(CudaTensor::wrap(dev, w->wk[l], {kv_dim, dim}));
            r->wv.push_back(CudaTensor::wrap(dev, w->wv[l], {kv_dim, dim}));
            r->wo.push_back(CudaTensor::wrap(dev, w->wo[l], {dim, q_dim}));
            r->ffn_gate.push_back(CudaTensor::wrap(dev, w->ffn_gate[l], {hidden, dim}));
            r->ffn_down.push_back(CudaTensor::wrap(dev, w->ffn_down[l], {dim, hidden}));
            r->ffn_up.push_back(CudaTensor::wrap(dev, w->ffn_up[l], {hidden, dim}));
            if (conf->arch == CCR_ARCH_QWEN2) {
                if (!w->bq || !w->bk || !w->bv) throw crabml::TensorError("qwen2: the q/k/v biases are missing");
                r->bq.push_back(CudaTensor::wrap(dev, w->bq[l], {q_dim}));
                r->bk.push_back(CudaTensor::wrap(dev, w->bk[l], {kv_dim}));
                r->bv.push_back(CudaTensor::wrap(dev, w->bv[l], {kv_dim}));
            }
            r->rms_att.push_back(CudaTensor::wrap(dev, w->rms_att[l], {dim}));
            r->rms_ffn.push_back(CudaTensor::wrap(dev, w->rms_ffn[l], {dim}));
            // llama2.rs:65-86: pre-allocated [n_kv_heads, seq_len, head_dim], resized to length 0
            int kvt = conf->use_f16_kv_cache ? CC_F16 : CC_F32;
            r->key_cache.push_back(CudaTensor::alloc({r->local_kv_heads(), kv_seq_len, hd}, kvt, dev).resize(1, 0));
            r->value_cache.push_back(CudaTensor::alloc({r->local_kv_heads(), kv_seq_len, hd}, kvt, dev).resize(1, 0));
        }
        r->logits.assign((size_t)conf->vocab_size, 0.0f);
    });
    if (rc != CC_OK) { delete r; return rc; }
    *out = r;
    return CC_OK;
}

extern "C" CC_API void ccr_runner_destroy(ccr_runner* r) { delete r; }
int ccr_runner_fail(ccr_runner* r, int code, const char* msg) { r->last_error = msg; return code; }
extern "C" CC_API const char* ccr_runner_last_error(ccr_runner* r) { return r ? r->last_error.c_str() : ""; }
extern "C" CC_API int64_t ccr_runner_kv_cache_len(ccr_runner* r) { return r ? r->kv_cache_len() : -1; }

extern "C" CC_API int ccr_runner_forward(ccr_runner* r, const int64_t* tokens, int32_t n_tokens, int64_t pos, float* logits_out) {
    if (!r || !tokens || n_tokens < 1) return CC_ERR_ARG;
    return guarded(r, [&] { r->forward(std::vector<int64_t>(tokens, tokens + n_tokens), pos, logits_out); });
}

// Greedy decode loop (prefill + generate with temperature 0: llama2.rs:111-172, sampler.rs:109-116).  Sampling runs on the device
// and the sampled id feeds the next step from a device slot, so no step waits for the host:
//   eos_token < 0  : all steps are submitted back to back, the ids come back in one copy at the end
//   eos_token >= 0 : the id of every step is read back (8 bytes) before the next step is submitted, to stop at EOS exactly like
//                    the reference (the KV cache must not grow past it)
// logits_out (optional, steps x vocab floats): the logits of every generated position, exported asynchronously through a pinned
// staging ring -- what a host-side sampler would consume.
extern "C" CC_API int ccr_runner_generate_greedy_ex(ccr_runner* r, const int64_t* prompt, int32_t n_prompt, int32_t steps,
                                                    int64_t eos_token, int64_t* out_tokens, int32_t* n_out, float* logits_out) {
    return ccr_runner_generate_loop(r, prompt, n_prompt, steps, eos_token, out_tokens, n_out, logits_out,
                                    [](const CudaTensor& lg, int64_t i) { lg.argmax_to_slot(0, i); });
}
// the loop of both generate entry points (generate_loop.hpp); `pick` samples generated token i into slot 0 and history[i]
int ccr_runner_generate_loop(ccr_runner* r, const int64_t* prompt, int32_t n_prompt, int32_t steps, int64_t eos_token, int64_t* out_tokens,
                             int32_t* n_out, float* logits_out, const ccr_step_sampler& pick) {
    if (!r || !prompt || n_prompt < 1 || !out_tokens || !n_out || steps < 1) return CC_ERR_ARG;
    *n_out = 0;
    float* pinned = nullptr;
    return guarded(r, [&] {
        const size_t vocab = (size_t)r->conf.vocab_size;
        int64_t pos = r->kv_cache_len();
        // how many tokens may be generated: the first comes from the prompt pass, the rest are bounded by the context (llama2.rs:141-147)
        const int64_t max_seq = r->conf.seq_len - (pos + n_prompt) - 1;
        const int64_t total = 1 + std::max<int64_t>(0, std::min<int64_t>(max_seq, (int64_t)steps - 1));
        if (logits_out) {
            if (r->pinned_floats < (size_t)total * vocab) {
                if (r->pinned_logits) { CudaTensor::check(r->dev, cc_device_synchronize(r->dev)); cc_host_free(r->dev, r->pinned_logits); r->pinned_logits = nullptr; r->pinned_floats = 0; }
                CudaTensor::check(r->dev, cc_host_alloc(r->dev, (size_t)total * vocab * 4, (void**)&r->pinned_logits));
                r->pinned_floats = (size_t)total * vocab;
            }
            pinned = r->pinned_logits;
        }
        for (int i = 0; i + 1 < n_prompt; i++) r->forward({prompt[i]}, pos++, nullptr);
        r->decode_step(&prompt[n_prompt - 1], pos++, 0, pinned, pick);
        int64_t done = 1;
        if (eos_token < 0) {
            for (; done < total; done++) r->decode_step(nullptr, pos++, done, pinned ? pinned + (size_t)done * vocab : nullptr, pick);
            CudaTensor::check(r->dev, cc_read_history(r->dev, 0, done, out_tokens));
        } else {
            CudaTensor::check(r->dev, cc_read_history(r->dev, 0, 1, out_tokens));
            for (; done < total; done++) {
                r->decode_step(nullptr, pos++, done, pinned ? pinned + (size_t)done * vocab : nullptr, pick);
                CudaTensor::check(r->dev, cc_read_history(r->dev, done, 1, out_tokens + done));
                if (out_tokens[done] == eos_token) break;          // the reference returns before yielding EOS (llama2.rs:160-163)
            }
        }
        *n_out = (int32_t)done;
        if (logits_out) { CudaTensor::check(r->dev, cc_device_synchronize(r->dev)); std::memcpy(logits_out, pinned, (size_t)done * vocab * 4); }
    });
}

extern "C" CC_API int ccr_runner_generate_greedy(ccr_runner* r, const int64_t* prompt, int32_t n_prompt, int32_t steps,
                                                 int64_t eos_token, int64_t* out_tokens, int32_t* n_out) {
    return ccr_runner_generate_greedy_ex(r, prompt, n_prompt, steps, eos_token, out_tokens, n_out, nullptr);
}
