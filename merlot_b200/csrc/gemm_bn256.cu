// K1 kernel instances for the 256-column tile (see gemm_kernel.cuh)
#include "gemm_kernel.cuh"

namespace mb {
template int launch_gemm_bn<256>(bool, bool, int, const CUtensorMap&, const CUtensorMap&, const CUtensorMap&, const CUtensorMap&,
                                  const GemmDev&, int, cudaStream_t);
}
