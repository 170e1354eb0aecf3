// op_record.cuh -- one trait op after capi.cu has checked its arguments: eager mode runs it at once (cc_run_op), lazy mode queues it
// (lazy.cu), and runs it through the same cc_run_op when no fused step takes it.
#pragma once
#include <string.h>

#include "sample_dev.cuh"

// What the scalar slots of each kind hold (a slot not listed is 0 / empty).  `a` is self / lhs / dst, `b` rhs / src, and DUP, CONTIGUOUS,
// MATVEC and BMM write the result they allocate, `out`.
//   COPY_ROWS    rows: the row indices; or i2 = slot + 1: the one row index is in device slot `slot` (cc_copy_rows_from_slot)
//   RMS_NORM     f: eps
//   MUL, ADD     i0, i1: elements of a and of b that chunks_exact(4) keeps (arithmetic.rs:5-68)
//   SCALE        f: the factor
//   ROPE         f: mode, i0: position, i1: batches, i2: batch stride, rows[0]: rope dims
//   CONCAT       i0: axis
//   ALLREDUCE, ALLGATHER   i0: elements (per rank)
//   ARGMAX       i0: slot, i1: history index
//   SAMPLE       f: temperature, i0: slot, i1: history index, i2: coin index, rows[0]: seed, rows[1]: the bits of topp (cc_sample_dyn)
enum LKind { L_COPY_ROWS, L_DUP, L_RMS_NORM, L_MUL, L_ADD, L_SCALE, L_MATVEC, L_ROPE, L_CONCAT, L_CONTIGUOUS, L_BMM, L_SOFTMAX, L_SILU, L_GELU, L_ALLREDUCE, L_ALLGATHER, L_ARGMAX, L_SAMPLE };

struct LOp {
    int kind;
    cc_view a{}, b{};
    cc_buf* out = nullptr;
    float f = 0.0f;
    int64_t i0 = 0, i1 = 0, i2 = 0;
    std::vector<int64_t> rows;
    bool done = false;       // lazy.cu: taken by a step of the plan being built
};

// ---- strider helpers (tensor/strider.rs) ------------------------------------------------------------------
inline int64_t view_len(const cc_view* v) {
    int64_t n = 1;
    for (int i = 0; i < v->ndim; i++) n *= v->shape[i];
    return n;
}
inline bool view_contiguous(const cc_view* v) {                      // strider.rs:182-206
    if (v->ndim == 0) return true;
    if (v->strides[v->ndim - 1] != 1) return false;
    int64_t last = 1;
    for (int i = v->ndim - 1; i >= 0; i--) {
        if (last != v->strides[i]) return false;
        last *= v->shape[i];
    }
    return true;
}

// the sampler's per-call values of a SAMPLE op
inline SampleDyn cc_sample_dyn(const LOp& op) {
    SampleDyn s;
    s.seed = (unsigned long long)op.rows[0]; s.coin_index = op.i2; s.hist_index = op.i1; s.temperature = op.f;
    const uint32_t pb = (uint32_t)op.rows[1];
    memcpy(&s.topp, &pb, 4);
    return s;
}

int cc_run_op(cc_device* dev, const LOp& op);       // capi.cu
int cc_lazy_record(cc_device* dev, LOp op);         // lazy.cu
