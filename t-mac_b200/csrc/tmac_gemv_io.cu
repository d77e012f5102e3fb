// tmac_gemv_io.cu -- the gemv3_kernel instantiations that build the LUT from activation rows (tmac_kernels.cuh): the plain row with
// an optional residual (kInRow: 3 bit widths x (6 fp + 3 integer-path groupings) x 2 register bounds), and the fp-path GEMV behind
// an RMSNorm, SwiGLU, SwiGLU-then-RMSNorm or squared-ReLU-then-RMSNorm input, and the RMSNorm input with a bias on the outputs
// (kInNorm, kInGlu, kInGluNorm, kInRelu2Norm, kInNormBias: 3 bit widths x 6 fp groupings x 2 register bounds each).  In their own
// translation unit so that they compile in parallel with tmac_b200.cu.
#include "tmac_kernels.cuh"

namespace tmac_b200 {

template gemv3_fn pick_gemv3_in<kInRow>(int, bool, int, int, int);
template gemv3_fn pick_gemv3_in<kInNorm>(int, bool, int, int, int);
template gemv3_fn pick_gemv3_in<kInGlu>(int, bool, int, int, int);
template gemv3_fn pick_gemv3_in<kInGluNorm>(int, bool, int, int, int);
template gemv3_fn pick_gemv3_in<kInRelu2Norm>(int, bool, int, int, int);
template gemv3_fn pick_gemv3_in<kInNormBias>(int, bool, int, int, int);

}  // namespace tmac_b200
