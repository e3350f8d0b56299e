// Host dispatch of the wgmma statistics pre-pass (kernel: cca_tc_stats.cuh) and its fp32 / bf16 instantiations.
#include "cca_tc_stats.cuh"

namespace cca {
using namespace tc;

cudaError_t tc_stats(const void *q, const void *k, float *parts, unsigned int *counters, int n_counters, Dims d, int dtype,
                     cudaStream_t st, const char **why)
{
    const StatsArgs a{q, k, parts, counters, n_counters, d, st, why};
    return with_elem_tile(dtype, d, [&](auto e, auto lk) { return launch_stats<lk(), decltype(e)>(a); });
}

}  // namespace cca
