// Addition to the mock C ABI (mock_abi.cpp) for the host-logic test of the sampled generate loop (tests/test_host_sampler_trace.py):
// cc_sample_to_slot records its call through the mock's tap entry, which appends "tap <name>" to the same trace.
#include <cstdio>
#include <string>

#include "../../include/crabml_cuda.h"

extern "C" CC_API int cc_sample_to_slot(cc_device* dev, const cc_view* x, float temperature, float topp, uint64_t seed, int64_t coin_index,
                                        int32_t slot, int64_t hist_index) {
    char b[256];
    snprintf(b, sizeof b, "sample_to_slot n=%lld slot=%d hist=%lld T=%.9g topp=%.9g seed=%llu coin=%lld", (long long)x->shape[0], (int)slot,
             (long long)hist_index, (double)temperature, (double)topp, (unsigned long long)seed, (long long)coin_index);
    return cc_debug_tensor_tap(dev, b, x);
}
