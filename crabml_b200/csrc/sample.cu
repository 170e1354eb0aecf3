// sample.cu -- temperature + top-p sampling into a token slot (cc_sample_to_slot): the one-CTA kernel of eager mode and of the
// CUDA-graph mode.  The routine itself is sample_dev.cuh, shared with the megakernel's MK_SAMPLE phase.
#include "sample_dev.cuh"

__global__ void __launch_bounds__(SMP_THREADS) sample_kernel(const float* x, int n, const SampleDyn args, const SampleDyn* args_dev, bool exact,
                                                             const SampleScratch S, long long* slot, long long* hist, const uint16_t* __restrict__ lut) {
    __shared__ __align__(16) uint8_t sm[SMP_SMEM_BYTES];
    const SampleDyn a = args_dev ? *args_dev : args;
    const long long id = cc_sample_block(x, n, a, exact, S, sm, lut);
    if (threadIdx.x == 0) {
        *slot = id;
        if (hist && a.hist_index >= 0 && a.hist_index < CC_HISTORY_CAP) hist[a.hist_index] = id;
    }
}

// grown only; a larger row replaces the buffer after the stream has drained (the lazy modes hash the pointer into their graph key)
int cc_ensure_sample_scratch(cc_device* dev, int64_t n) {
    const size_t need = cc_sample_scratch_bytes(n);
    if (need <= dev->sample_scratch_bytes) return CC_OK;
    if (dev->sample_scratch) {
        CC_CUDA(dev, cudaStreamSynchronize(dev->stream));
        CC_CUDA(dev, cudaFree(dev->sample_scratch));
        dev->sample_scratch = nullptr; dev->sample_scratch_bytes = 0;
    }
    size_t cap = (size_t)1 << 20;
    while (cap < need) cap <<= 1;
    CC_CUDA(dev, cudaMalloc(&dev->sample_scratch, cap));
    dev->sample_scratch_bytes = cap;
    return CC_OK;
}

// args: the values of this call (eager mode); args_dev: the same in device memory (the lazy modes' dyn block), used when non-null
int cc_launch_sample(cc_device* dev, const float* x, int64_t n, const SampleDyn* args, const SampleDyn* args_dev, int64_t* slot, int64_t* hist) {
    const SampleDyn a = args ? *args : SampleDyn{};
    sample_kernel<<<1, SMP_THREADS, 0, dev->stream>>>(x, (int)n, a, args_dev, dev->exact, cc_sample_scratch(dev->sample_scratch, n), (long long*)slot,
                                                       (long long*)hist, dev->exp_lut);
    CC_LAUNCH_CHECK(dev);
    return CC_OK;
}
