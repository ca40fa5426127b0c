// One kernel variant per object file: the Makefile compiles this unit once per entry of its VARIANTS list with
// -DRN_BN=<N tile> -DRN_CL=<cluster> -DRN_MS=<M sub-tiles> -DRN_SPLIT=<0|1> -DRN_HALF=<0|1>,
// so `make -j` spreads the (slow) ptxas runs over all cores.  rn_igemm.cu dispatches to them.
#include "rn_igemm_kernel.cuh"

namespace rn {
template cudaError_t launch_ms<RN_BN, RN_CL, RN_MS, (RN_SPLIT != 0), (RN_HALF != 0)>(const IgemmParams&, int, size_t,
                                                                                    cudaStream_t);
}  // namespace rn
