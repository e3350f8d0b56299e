// Host dispatch of the wgmma statistics pre-pass (kernel: cca_tc_stats.cuh) and its fp32 / bf16 instantiations.
#include "cca_tc_stats.cuh"

namespace cca {
using namespace tc;

// parts: [nparts][B*H*W] fp32.  Also clears zero_bytes bytes at zero_ptr and n_counters words at counters (both may be 0).
cudaError_t tc_stats(const void *q, const void *k, float *parts, void *zero_ptr, long zero_bytes, unsigned int *counters,
                     int n_counters, Dims d, int dtype, cudaStream_t st, const char **why)
{
    const int lk = tc::lk_for(tc::max_tile(tc::make_space(d.B, d.H, d.W)));
    if (dtype == CCA_F16)
        return lk == 80 ? launch_stats<80, __half>(q, k, parts, zero_ptr, zero_bytes, counters, n_counters, d, st, why)
                        : launch_stats<112, __half>(q, k, parts, zero_ptr, zero_bytes, counters, n_counters, d, st, why);
    if (dtype == CCA_BF16)
        return lk == 80 ? launch_stats<80, __nv_bfloat16>(q, k, parts, zero_ptr, zero_bytes, counters, n_counters, d, st, why)
                        : launch_stats<112, __nv_bfloat16>(q, k, parts, zero_ptr, zero_bytes, counters, n_counters, d, st, why);
    return lk == 80 ? launch_stats<80, float>(q, k, parts, zero_ptr, zero_bytes, counters, n_counters, d, st, why)
                    : launch_stats<112, float>(q, k, parts, zero_ptr, zero_bytes, counters, n_counters, d, st, why);
}

}  // namespace cca
