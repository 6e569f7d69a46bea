// wunet_tc_f16.cu — fp16 kernels of the tensor-core inference path (WUNET_PREC_FP16) for sm_90a.
//
// The same kernel bodies as the bf16 path (wunet_tc_kernels.cuh), compiled with fp16 elements: activations are channels-last
// fp16, weights fp16 (round to nearest even from the fp32 parameters, saturating), products accumulate in fp32 on
// wgmma.m64nNk16.f32.f16.f16, and the folded BatchNorm and LeakyReLU run in fp32 in the epilogue. Only the forms the bf16 plan
// launches have fp16 twins: no split-precision kernels and no tensor-core block 0. The host code (planner, state, launches) is
// the bf16 path's, in wunet_tc.cu; it reaches these kernels through the functions below.
#define WUNET_TC_FP16 1
#include "wunet_common.cuh"
#include "wunet_wgmma.cuh"
#include "wunet_tc_common.cuh"

namespace wunet {
namespace f16 {

using TcElem = TcF16;
#include "wunet_tc_kernels.cuh"

void set_smem_attributes()
{
    const ConvKernel conv[] = {
        conv_tc_kernel<15, false, kEpiWarpsLarge, 0, 0>, conv_tc_kernel<15, false, kEpiWarpsSmall, 0, 0>,
        conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 0>, conv_tc_kernel<5, true, kEpiWarpsSmall, kProducerWarpsSmall, 0>,
        conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 1>, conv_tc_kernel<5, true, kEpiWarpsSmall, kProducerWarpsSmall, 1>,
        conv_tc_kernel<9, false, kEpiWarpsLarge, 0, 0>, conv_tc_kernel<9, false, kEpiWarpsSmall, 0, 0>};
    for (ConvKernel k : conv) cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
    cudaFuncSetAttribute(gemm_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
    cudaFuncSetAttribute(enc0_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
    cudaFuncSetAttribute(enc0_kernel_v2, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
}

ConvKernel conv_kernel(int ks, bool small, bool mg)
{
    if (ks == 9) return small ? conv_tc_kernel<9, false, kEpiWarpsSmall, 0, 0> : conv_tc_kernel<9, false, kEpiWarpsLarge, 0, 0>;
    if (ks == 15) return small ? conv_tc_kernel<15, false, kEpiWarpsSmall, 0, 0> : conv_tc_kernel<15, false, kEpiWarpsLarge, 0, 0>;
    if (mg)
        return small ? conv_tc_kernel<5, true, kEpiWarpsSmall, kProducerWarpsSmall, 1>
                     : conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 1>;
    return small ? conv_tc_kernel<5, true, kEpiWarpsSmall, kProducerWarpsSmall, 0>
                 : conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 0>;
}

GemmKernel gemm_kernel() { return gemm_tc_kernel; }

cudaError_t launch_enc0(const cudaLaunchConfig_t &cfg, bool persistent, const float *x, const float *w, const float *scale,
                        const float *shift, void *out, int B, int T, int C, void *even_out)
{
    return cudaLaunchKernelEx(&cfg, persistent ? enc0_kernel_v2 : enc0_kernel, x, w, scale, shift, static_cast<__half *>(out), B, T,
                              C, 0, static_cast<__half *>(even_out));
}

cudaError_t pack(const float *w, const float *scale, const float *shift, void *wp, float2 *ss, int Cout, int Cin0, int Cin1, int K,
                 int Npad, int Ktot, cudaStream_t stream)
{
    const size_t nel = (size_t)K * Npad * Ktot;
    pack_tc_kernel<<<(unsigned)((nel + 255) / 256), 256, 0, stream>>>(w, scale, shift, static_cast<__half *>(wp), ss, Cout, Cin0, Cin1,
                                                                      K, Npad, Ktot);
    return cudaGetLastError();
}

cudaError_t pack_merged(const float *w, void *wp, int Cout, int Cin0, int Cin1, int K, int Npad, int Ktot, int s, int u,
                        cudaStream_t stream)
{
    const size_t nm = (size_t)K * Npad * 64;
    pack_tc_merged_kernel<<<(unsigned)((nm + 255) / 256), 256, 0, stream>>>(w, static_cast<__half *>(wp), Cout, Cin0, Cin1, K, Npad,
                                                                            Ktot, s, u);
    return cudaGetLastError();
}

cudaError_t expand_gemm_weights(const float *w, void *wx, size_t n, int Cout, int Cin0, int Cin1, int K, int L, int dec, int npos0,
                                int cpp0, int npos1, int cpp1, float up_scale, cudaStream_t stream)
{
    expand_gemm_weights_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(w, static_cast<__half *>(wx), Cout, Cin0, Cin1, K, L,
                                                                                 dec, npos0, cpp0, npos1, cpp1, up_scale);
    return cudaGetLastError();
}

cudaError_t nlc_to_ncl(const void *src, float *dst, int B, int L, int C, cudaStream_t stream)
{
    const long long nel = (long long)B * C * L;
    nlc_f16_to_ncl_f32_kernel<<<(unsigned)((nel + 255) / 256), 256, 0, stream>>>(static_cast<const __half *>(src), dst, B, L, C);
    return cudaGetLastError();
}

}  // namespace f16
}  // namespace wunet
