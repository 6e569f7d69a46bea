// wunet_tc_io.cuh — the tensor-core inference kernels that read the network input or write its output, with a 16-bit I/O element
// type (a half model's forward). Included by wunet_tc_io_f16.cu (WUNET_TC_IO = __half, namespace io_f16) and wunet_tc_io_bf16.cu
// (__nv_bfloat16, io_bf16), which define WUNET_TC_IO and WUNET_TC_IO_NS first.
//
// wunet_tc_kernels.cuh is compiled here with WUNET_TC_IO_ONLY, once per activation element type (bf16, fp16), so these units
// hold only the 16-bit I/O forms the planner launches, and the float forms in wunet_tc.cu / wunet_tc_f16.cu / wunet_tc_wide.cu
// stay the kernels they were:
//   * block 0: enc0_kernel (bf16, split precision, fp16 rows), enc0_wide_kernel (wide plans: bf16, split precision, fp16), and
//     x_to_bf16_kernel (the opt-in group-of-8 block 0, bf16 only). The persistent enc0_kernel_v2 streams float samples with 4-byte
//     cp.async, which cannot widen 16-bit ones: a 16-bit input runs enc0_kernel, whose output is the same.
//   * the last block, whose fused head reads x and writes y: the large flavour of the decoder form (plain, merged tail chunk)
//     for bf16 and fp16, and the split-precision one. The planner gives the last block neither the small flavour (only a tuning
//     override does) nor the row-pair form.
#include "wunet_common.cuh"
#include "wunet_wgmma.cuh"
#include "wunet_tc_common.cuh"

#define WUNET_TC_IO_ONLY 1

namespace wunet {
namespace WUNET_TC_IO_NS {

namespace bf16 {
using TcElem = TcBf16;
#include "wunet_tc_kernels.cuh"
#include "wunet_tc_wide.cuh"
}  // namespace bf16

namespace f16 {
#define WUNET_TC_FP16 1
using TcElem = TcF16;
#include "wunet_tc_kernels.cuh"
#include "wunet_tc_wide.cuh"
#undef WUNET_TC_FP16
}  // namespace f16

using IoT = WUNET_TC_IO;

::wunet::f16::ConvKernel head_kernel(int mode, bool mg)
{
    if (mode == 2)
        return mg ? f16::conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 1>
                  : f16::conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 0>;
    if (mode == 1) return bf16::conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 0, 1>;
    return mg ? bf16::conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 1>
              : bf16::conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 0>;
}

void set_smem_attributes(int enc0_wide_max)
{
    for (int mode : {0, 1, 2})
        for (bool mg : {false, true}) cudaFuncSetAttribute(head_kernel(mode, mg), cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
    cudaFuncSetAttribute(bf16::enc0_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
    cudaFuncSetAttribute(f16::enc0_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
    cudaFuncSetAttribute(bf16::enc0_wide_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, enc0_wide_max);
    cudaFuncSetAttribute(bf16::enc0_wide_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, enc0_wide_max);
    cudaFuncSetAttribute(f16::enc0_wide_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, enc0_wide_max);
}

cudaError_t launch_enc0(const cudaLaunchConfig_t &cfg, int mode, const void *x, const float *w, const float *scale, const float *shift,
                        void *out, int B, int T, int C, void *even_out)
{
    const IoT *xi = static_cast<const IoT *>(x);
    if (mode == 2)
        return cudaLaunchKernelEx(&cfg, f16::enc0_kernel, xi, w, scale, shift, static_cast<__half *>(out), B, T, C, 0,
                                  static_cast<__half *>(even_out));
    return cudaLaunchKernelEx(&cfg, bf16::enc0_kernel, xi, w, scale, shift, static_cast<__nv_bfloat16 *>(out), B, T, C, mode == 1 ? 1 : 0,
                              static_cast<__nv_bfloat16 *>(even_out));
}

cudaError_t launch_enc0_wide(const cudaLaunchConfig_t &cfg, int mode, const void *x, const float *w, const float *scale,
                             const float *shift, void *out, int B, int T, int C)
{
    const IoT *xi = static_cast<const IoT *>(x);
    if (mode == 2)
        return cudaLaunchKernelEx(&cfg, f16::enc0_wide_kernel<2>, xi, w, scale, shift, static_cast<__half *>(out), B, T, C, 0);
    if (mode == 1)
        return cudaLaunchKernelEx(&cfg, bf16::enc0_wide_kernel<4>, xi, w, scale, shift, static_cast<__nv_bfloat16 *>(out), B, T, C, 1);
    return cudaLaunchKernelEx(&cfg, bf16::enc0_wide_kernel<2>, xi, w, scale, shift, static_cast<__nv_bfloat16 *>(out), B, T, C, 0);
}

cudaError_t launch_x_to_bf16(const void *x, __nv_bfloat16 *xb, long long n4, cudaStream_t stream)
{
    bf16::x_to_bf16_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(static_cast<const IoT *>(x), xb, n4);
    return cudaGetLastError();
}

}  // namespace WUNET_TC_IO_NS
}  // namespace wunet
