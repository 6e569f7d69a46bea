// wunet_tc_pp.cu — the ping-pong form of the weight-resident decoder blocks (wunet_tc_pp.cuh) for bf16 and fp16 with float I/O,
// for sm_90a; the host launches it for the last decoder block (pp::selected). A unit of its own so that the kernels of
// wunet_tc.cu and wunet_tc_f16.cu keep their machine code; the host code of wunet_tc.cu reaches these kernels through the
// functions below.
#include "wunet_common.cuh"
#include "wunet_wgmma.cuh"
#include "wunet_tc_common.cuh"

#define WUNET_TC_CONV_ONLY 1

namespace wunet {
namespace pp {

namespace bf16 {
using TcElem = TcBf16;
#include "wunet_tc_kernels.cuh"
#include "wunet_tc_pp.cuh"
}  // namespace bf16

namespace f16 {
#define WUNET_TC_FP16 1
using TcElem = TcF16;
#include "wunet_tc_kernels.cuh"
#include "wunet_tc_pp.cuh"
#undef WUNET_TC_FP16
}  // namespace f16

ConvKernel conv_kernel(bool fp16, bool mg)
{
    if (fp16) return mg ? f16::conv_tc_pp_kernel<1> : f16::conv_tc_pp_kernel<0>;
    return mg ? bf16::conv_tc_pp_kernel<1> : bf16::conv_tc_pp_kernel<0>;
}

void set_smem_attributes()
{
    for (bool fp16 : {false, true})
        for (bool mg : {false, true}) cudaFuncSetAttribute(conv_kernel(fp16, mg), cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
}

bool selected(const TcParams &p, bool upcat, bool small, int io)
{
    return io == IO_F32 && p.split == 0 && upcat && !small && p.resident && p.nsplit == 1 && !p.packed && p.hd == 0 && p.MT == 1 &&
           p.Nh <= bf16::kPpAccCols && p.head;
}

}  // namespace pp
}  // namespace wunet
