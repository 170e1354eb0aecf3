// matvec_stream.cu -- the streaming matvec for the decode hot path (b = 1).
//
// History:
//   r01a  matvec.cu (warp per row, 4 loads in flight, activation staged before the first weight load, 1.33 waves):
//         latency bound.
//   r01b  first persistent version with a per-group register ring and the Q8_0 quantisation of x fused into every
//         CTA's prologue: 171 instructions per 1 KB group and 2.3 M redundant prologue instructions -> issue bound
//         (low IPC with few warps per scheduler).  Lesson: this kernel must be ~20 instructions per
//         group, and x is quantised ONCE (quantize.cu / the producer's epilogue), not once per SM.
//   this  persistent grid (2 CTAs x 8 warps per SM), rows dealt round-robin to warps; the weight stream of a warp is
//         cut into SEGMENTS of 4 groups (4 x 32 blocks = 4096 weights = 4 KB of Q8_0) that are double-buffered in
//         registers across row boundaries: the loads of segment u+1 are issued before segment u is consumed
//         (8 KB in flight per warp, 128 KB per SM).  All shared-memory and global offsets inside a segment are
//         lane-relative immediates.  The first segment is requested BEFORE the activation is staged.
//   * the quantised activation (Q8_0 blocks as SoA: qs | f32 scale | block sums) is copied global -> shared once per CTA;
//   * up to 3 matrices that share the activation (wq,wk,wv / gate,up) run as one launch;
//   * epilogues: store | + one f32 vector per matrix: the residual (llama2.rs:266,636) or qwen2's q/k/v biases
//     (llama2.rs:315-317) | silu(gate) * up (llama2.rs:620-630).
// Q8_0 device layout: inside each group of 32 blocks the 16-byte first halves of all blocks precede the second
// halves, so lane l reads block 32g+l with two fully coalesced LDG.128 (512 B per warp request).
#include "common.cuh"

#define MS_THREADS 256
#define MS_WARPS 8
#define MS_CTAS_PER_SM 2
#define MS_SEG 4                      // groups per segment

__device__ __forceinline__ int dp16(const int4& w, const int4& a) {
    return __dp4a(w.x, a.x, __dp4a(w.y, a.y, __dp4a(w.z, a.z, __dp4a(w.w, a.w, 0))));
}

template <int TYPE> struct Seg;
template <> struct Seg<CC_Q8_0> { int4 a[MS_SEG], b[MS_SEG]; uint16_t s[MS_SEG]; };
template <> struct Seg<CC_Q4_0> { int4 a[MS_SEG]; uint16_t s[MS_SEG]; };

// pointers of one row, already offset to this lane
struct RowPtr { const uint8_t* q; const uint16_t* d; };

template <int TYPE>
__device__ __forceinline__ RowPtr row_ptr(const StreamMats& M, int mat, int r, int nb, int lane) {
    RowPtr p;
    constexpr int BB = TYPE == CC_Q8_0 ? 32 : 16;
    // ternaries instead of M.qs[mat]: a dynamically indexed kernel-parameter array would be copied to local memory
    const uint8_t* q0 = mat == 0 ? M.qs[0] : mat == 1 ? M.qs[1] : M.qs[2];
    const uint16_t* d0 = mat == 0 ? M.d[0] : mat == 1 ? M.d[1] : M.d[2];
    p.q = q0 + (size_t)r * nb * BB + lane * 16;
    p.d = d0 + (size_t)r * CC_D_STRIDE(nb) + lane;
    return p;
}

// issue the loads of segment `seg` of a row (groups 4*seg .. 4*seg+3); lanes past the row end get zeros
template <int TYPE>
__device__ __forceinline__ void seg_load(Seg<TYPE>& S, const RowPtr& p, int seg, int nb, int GR, int last_half_off, int lane, bool valid) {
    constexpr int GB = TYPE == CC_Q8_0 ? 1024 : 512;           // bytes per full group
    const uint8_t* q = p.q + (size_t)seg * (MS_SEG * GB);
    const uint16_t* d = p.d + seg * (MS_SEG * 32);
#pragma unroll
    for (int g = 0; g < MS_SEG; g++) {
        const int gi = seg * MS_SEG + g;
        const bool on = valid && (gi * 32 + lane < nb);
        if constexpr (TYPE == CC_Q8_0) {
            const int hoff = gi == GR - 1 ? last_half_off : 512;
            if (on) { S.a[g] = ld_stream_16(q + g * GB); S.b[g] = ld_stream_16(q + g * GB + hoff); S.s[g] = d[g * 32]; }
            else { S.a[g] = make_int4(0, 0, 0, 0); S.b[g] = S.a[g]; S.s[g] = 0; }
        } else {
            if (on) { S.a[g] = ld_stream_16(q + g * GB); S.s[g] = d[g * 32]; }
            else { S.a[g] = make_int4(0, 0, 0, 0); S.s[g] = 0; }
        }
    }
}

// shared memory (padded with zeros to GR*32 blocks): quants | f32 scales | (Q4_0) i32 block sums; all lane-relative
template <int TYPE>
__device__ __forceinline__ float seg_dot(const Seg<TYPE>& S, int seg, const int4* aq_l, const float* ad_l, const int* as_l) {
    float acc = 0.0f;
    const int4* aq = aq_l + seg * (MS_SEG * 64);
    const float* ad = ad_l + seg * (MS_SEG * 32);
#pragma unroll
    for (int g = 0; g < MS_SEG; g++) {
        if constexpr (TYPE == CC_Q8_0) {
            int sumi = dp16(S.a[g], aq[g * 64]) + dp16(S.b[g], aq[g * 64 + 1]);
            acc += (float)sumi * h2f_bits(S.s[g]) * ad[g * 32];                       // buf_q8_0.rs:283 per-block term
        } else {
            const int4 w = S.a[g];
            int4 lo = make_int4(w.x & 0x0F0F0F0F, w.y & 0x0F0F0F0F, w.z & 0x0F0F0F0F, w.w & 0x0F0F0F0F);
            int4 hi = make_int4((w.x >> 4) & 0x0F0F0F0F, (w.y >> 4) & 0x0F0F0F0F, (w.z >> 4) & 0x0F0F0F0F, (w.w >> 4) & 0x0F0F0F0F);
            int sumi = dp16(lo, aq[g * 64]) + dp16(hi, aq[g * 64 + 1]) - 8 * as_l[(seg * MS_SEG + g) * 32];   // buf_q4_0.rs:244-249
            acc += (float)sumi * h2f_bits(S.s[g]) * ad[g * 32];
        }
    }
    return acc;
}

template <int TYPE>
__global__ void __launch_bounds__(MS_THREADS, MS_CTAS_PER_SM) matvec_stream_kernel(StreamArgs A, const uint16_t* __restrict__ exp_lut) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int k = A.k, nb = k >> 5, GR = (nb + 31) >> 5, NSEG = (GR + MS_SEG - 1) / MS_SEG;
    const int nbp = NSEG * MS_SEG * 32;                           // padded block count
    int8_t* s_q = (int8_t*)smem;
    float* s_d = (float*)(smem + (size_t)nbp * 32);
    int* s_s = (int*)(smem + (size_t)nbp * 32 + (size_t)nbp * 4);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gw = blockIdx.x * MS_WARPS + warp, TW = gridDim.x * MS_WARPS;
    const StreamMats& M = A.mats;
    const bool pair = A.epilogue == 2;
    // virtual row list of this warp: plain -> rows gw, gw+TW, ... over the concatenated matrices;
    // pair -> (mat0 row r, mat1 row r) for r = gw, gw+TW, ...
    const int m_cat = pair ? M.m[0] : M.m[0] + (M.n > 1 ? M.m[1] : 0) + (M.n > 2 ? M.m[2] : 0);
    const int n_rows = gw < m_cat ? (m_cat - gw + TW - 1) / TW : 0;
    const int n_vrows = pair ? 2 * n_rows : n_rows;
    const int U = n_vrows * NSEG;                                  // segments this warp will stream
    const int last_half_off = 16 * (nb - 32 * (GR - 1));

    auto vrow_ptr = [&](int i) -> RowPtr {                         // i-th virtual row of this warp
        int mat = 0, r;
        if (pair) { mat = i & 1; r = gw + (i >> 1) * TW; }
        else {
            r = gw + i * TW;
            if (M.n > 1 && r >= M.m[0]) { r -= M.m[0]; mat = 1; if (M.n > 2 && r >= M.m[1]) { r -= M.m[1]; mat = 2; } }
        }
        return row_ptr<TYPE>(M, mat, r, nb, lane);
    };

    // ---- 1. request the first segment of the weight stream before anything else -------------------------
    Seg<TYPE> buf0, buf1;
    int l_i = 0, l_seg = 0;                                        // load cursor: virtual row index, segment
    RowPtr l_ptr = vrow_ptr(0);
    seg_load<TYPE>(buf0, l_ptr, 0, nb, GR, last_half_off, lane, U > 0);
    auto advance_load = [&]() { if (++l_seg == NSEG) { l_seg = 0; l_ptr = vrow_ptr(++l_i); } };
    advance_load();
    // programmatic dependent launch: let the next kernel be scheduled (it will prefetch ITS weights), then wait for
    // the producer of our activation; everything above only touched immutable weights
    asm volatile("griddepcontrol.launch_dependents;");
    asm volatile("griddepcontrol.wait;" ::: "memory");

    // ---- 2. stage the quantised activation (global scratch -> shared), zero the padding ---------------------
    {
        const uint8_t* act = (const uint8_t*)A.act;
        const int4* gq = (const int4*)act;
        int4* sq4 = (int4*)s_q;
        for (int i = threadIdx.x; i < nbp * 2; i += MS_THREADS) sq4[i] = i < nb * 2 ? gq[i] : make_int4(0, 0, 0, 0);
        const float* gd = (const float*)(act + ((k + 15) & ~15));
        const int* gs = (const int*)(act + ((k + 15) & ~15) + ((nb * 4 + 15) & ~15));
        for (int i = threadIdx.x; i < nbp; i += MS_THREADS) {
            s_d[i] = i < nb ? gd[i] : 0.0f;
            if constexpr (TYPE == CC_Q4_0) s_s[i] = i < nb ? gs[i] : 0;
        }
    }
    __syncthreads();
    const int4* aq_l = (const int4*)s_q + 2 * lane;
    const float* ad_l = s_d + lane;
    const int* as_l = s_s + lane;

    // ---- 3. stream -----------------------------------------------------------------------------------------------
    float acc = 0.0f, first = 0.0f;
    int c_i = 0, c_seg = 0;                                        // consume cursor
    auto finish_segment = [&]() {
        if (++c_seg < NSEG) return;
        c_seg = 0;
        float r = warp_sum(acc);
        acc = 0.0f;
        const int i = c_i++;
        if (pair) {
            if ((i & 1) == 0) { first = r; return; }
            if (lane == 0) {                                       // silu.rs:6-13 then mul (llama2.rs:625-630)
                float g = first;
                float nexp = h2f_bits(exp_lut[f2h_bits(-g)]);
                M.out[0][gw + (i >> 1) * TW] = (g / (1.0f + nexp)) * r;
            }
            return;
        }
        if (lane == 0) {
            int mat = 0, rr = gw + i * TW;
            if (M.n > 1 && rr >= M.m[0]) { rr -= M.m[0]; mat = 1; if (M.n > 2 && rr >= M.m[1]) { rr -= M.m[1]; mat = 2; } }
            if (A.epilogue == 1) r = r + (mat == 0 ? A.residual[0] : mat == 1 ? A.residual[1] : A.residual[2])[rr];
            float* o = mat == 0 ? M.out[0] : mat == 1 ? M.out[1] : M.out[2];
            o[rr] = r;
        }
    };
    for (int u = 0; u < U; u += 2) {
        seg_load<TYPE>(buf1, l_ptr, l_seg, nb, GR, last_half_off, lane, u + 1 < U);
        advance_load();
        acc += seg_dot<TYPE>(buf0, c_seg, aq_l, ad_l, as_l);
        finish_segment();
        if (u + 1 >= U) break;
        seg_load<TYPE>(buf0, l_ptr, l_seg, nb, GR, last_half_off, lane, u + 2 < U);
        advance_load();
        acc += seg_dot<TYPE>(buf1, c_seg, aq_l, ad_l, as_l);
        finish_segment();
    }
}

static size_t stream_smem_bytes(int type, int k) {
    size_t nb = k / 32, GR = (nb + 31) / 32, NSEG = (GR + MS_SEG - 1) / MS_SEG, nbp = NSEG * MS_SEG * 32;
    return nbp * 32 + nbp * 4 + (type == CC_Q4_0 ? nbp * 4 : 0);
}

bool cc_stream_supported(int type, int64_t k) { return (type == CC_Q8_0 || type == CC_Q4_0) && k % 32 == 0 && k <= 32768; }

int cc_launch_matvec_stream(cc_device* dev, int type, const StreamArgs& A) {
    size_t smem = stream_smem_bytes(type, A.k);
    int grid = dev->sm_count * MS_CTAS_PER_SM;
    int64_t m_cat = A.epilogue == 2 ? A.mats.m[0] : (int64_t)A.mats.m[0] + (A.mats.n > 1 ? A.mats.m[1] : 0) + (A.mats.n > 2 ? A.mats.m[2] : 0);
    int64_t need = (m_cat + MS_WARPS - 1) / MS_WARPS;
    if (need < grid) grid = (int)(need > 0 ? need : 1);
    auto kernel = type == CC_Q8_0 ? matvec_stream_kernel<CC_Q8_0> : matvec_stream_kernel<CC_Q4_0>;
    if (smem > 48 * 1024) CC_CUDA(dev, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaError_t e = launch_pdl(kernel, dim3(grid), dim3(MS_THREADS), smem, dev->stream, dev->pdl, A, (const uint16_t*)dev->exp_lut);
    if (e != cudaSuccess) return cc_fail(dev, CC_ERR_CUDA, "matvec_stream launch: %s", cudaGetErrorString(e));
    dev->launches++;
    return CC_OK;
}

// plain matmul_vec (eager trait call): activation already quantised into `act` by quantize.cu
int cc_launch_matvec_stream_plain(cc_device* dev, const cc_buf* w, const void* act, float* out, int64_t m, int64_t k) {
    StreamArgs A = {};
    A.mats.n = 1;
    A.mats.qs[0] = w->plane[0];
    A.mats.d[0] = (const uint16_t*)w->plane[1];
    A.mats.out[0] = out;
    A.mats.m[0] = (int)m;
    A.act = act;
    A.k = (int)k;
    return cc_launch_matvec_stream(dev, w->dtype, A);
}
