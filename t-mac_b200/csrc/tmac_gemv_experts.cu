// tmac_gemv_experts.cu -- the gemv3_kernel instantiations of the routed-expert launches (tmac_kernels.cuh, IO = kIoExperts /
// kIoExpertsGlu): each slot picks its tensor from the router's ids on the device, 3 bit widths x 6 fp groupings x 2 register bounds
// x 2 kinds.  In their own translation unit so that they compile in parallel with tmac_b200.cu.
#include "tmac_kernels.cuh"
#include "tmac_layout.h"

namespace tmac_b200 {

namespace {
template <int MINB, int IO> gemv3_fn pick_experts(int pb, int qch, int agq) {
    return with_pb<gemv3_fn>(pb, [&](auto PB) {
        return FpGroupings::find<gemv3_fn>(qch, agq, [&](auto QCH, auto AGQ) -> gemv3_fn {
            return gemv3_kernel<PB, true, QCH, AGQ, MINB, true, IO>;
        });
    });
}
template <int MINB> gemv3_fn pick_experts_kind(int pb, int qch, int agq, int io) {
    switch (io) {
        case kIoExperts: return pick_experts<MINB, kIoExperts>(pb, qch, agq);
        case kIoExpertsGlu: return pick_experts<MINB, kIoExpertsGlu>(pb, qch, agq);
        default: return nullptr;
    }
}
}  // namespace

gemv3_fn pick_gemv3_experts(int pb, int qch, int agq, int minb, int io) {
    return minb == 3 ? pick_experts_kind<3>(pb, qch, agq, io) : pick_experts_kind<4>(pb, qch, agq, io);
}

}  // namespace tmac_b200
