// tmac_gemv_experts.cu -- the gemv3_kernel instantiations of the routed-expert launches (tmac_kernels.cuh, IN = kInExperts /
// kInExpertsGlu): each slot picks its tensor from the router's ids on the device, 3 bit widths x 6 fp groupings x 2 register bounds
// x 2 kinds.  In their own translation unit so that they compile in parallel with tmac_b200.cu.
#include "tmac_kernels.cuh"

namespace tmac_b200 {

template gemv3_fn pick_gemv3_in<kInExperts>(int, bool, int, int, int);
template gemv3_fn pick_gemv3_in<kInExpertsGlu>(int, bool, int, int, int);

}  // namespace tmac_b200
