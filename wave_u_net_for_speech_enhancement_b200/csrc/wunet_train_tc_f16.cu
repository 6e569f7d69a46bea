// wunet_train_tc_f16.cu — tensor-core convolutions of the training step with fp16 operands and per-block dz scaling
// (Model(train_precision="fp16_scaled"), DESIGN.md §5.4): the instances of the kernels in wunet_train_tc_kernels.cuh at the F16
// operand type. A unit of its own, so that the bf16 / tf32 unit keeps its kernels. Reached through train_tc_pack,
// launch_train_conv_tc and launch_train_wgrad_tc (wunet_train_tc.cu) with TRAIN_FP16_SCALED.
#include "wunet_train_tc_kernels.cuh"

namespace wunet {

int train_tc_pack_f16(const float *w, void *wf, void *wb, int Cout, int Cin, int K, cudaStream_t st)
{
    return pack<F16>(w, wf, wb, Cout, Cin, K, st);
}

int launch_train_conv_tc_f16(const ConvArgs &a, int ksize, int mode, cudaStream_t st)
{
    return launch_conv_op<F16>(a, ksize, mode, st);
}

int launch_train_wgrad_tc_f16(const ConvArgs &a, const float *dz, float *dw, int ksize, int mode, cudaStream_t st, bool slices)
{
    return launch_wgrad_op<F16>(a, dz, dw, ksize, mode, st, slices);
}

}  // namespace wunet
