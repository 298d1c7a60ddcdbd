// lld_kernel_f32.cu -- the lld_kernel instances for inputs pre-converted to mono float samples (LldParams::pcmF32).  They are
// compiled apart from the int16 instances in kernels.cu so that the two halves of the family build in parallel.
#include "lld_kernel.cuh"

namespace osm {

template cudaError_t launch_lld_kernel<true>(const LldParams &, int, int, cudaStream_t, LldLaunchInfo *, bool);

}  // namespace osm
