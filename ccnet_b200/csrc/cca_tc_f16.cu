// f16 instantiations of the three wgmma kernels (statistics, forward values, backward) for LK = 80 and 112.  The dispatch is
// in cca_tc_stats.cu, cca_tc_fwd.cu and cca_tc_bwd.cu; keeping these in their own translation unit compiles them in parallel
// with the fp32 / bf16 ones.
#include "cca_tc_bwd.cuh"
#include "cca_tc_fwd.cuh"
#include "cca_tc_stats.cuh"

namespace cca {
namespace tc {

template cudaError_t launch_stats<80, __half>(const StatsArgs &);
template cudaError_t launch_stats<112, __half>(const StatsArgs &);
template cudaError_t launch_fwd<80, __half>(const FwdArgs &);
template cudaError_t launch_fwd<112, __half>(const FwdArgs &);
template cudaError_t launch_bwd<80, __half>(const BwdArgs &);
template cudaError_t launch_bwd<112, __half>(const BwdArgs &);

}  // namespace tc
}  // namespace cca
