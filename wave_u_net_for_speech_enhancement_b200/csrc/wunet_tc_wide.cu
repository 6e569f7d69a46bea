// wunet_tc_wide.cu — kernels that only the wide channel plans (channels_interval 40 .. 64, a multiple of 8) of the tensor-core
// inference path launch, for sm_90a. Every other block of a wide plan runs the forms of wunet_tc.cu / wunet_tc_f16.cu.
//
//   * enc0_wide_kernel: block 0 with a tile that shrinks with C, so that its staged rows fit in shared memory at any supported
//     width (enc0_kernel's 1024-row tile needs 160 KiB at C = 40 in split precision). bf16, fp16 and split precision.
//   * conv_tc_kernel<..., SP = 2>: the split-precision (fp32_tc) conv form whose chunk_map lists chunks rather than K-loop
//     positions (chunk_info), for blocks with more than 48 positions: the middle decoders of 12 layers at ci >= 48. With
//     pack_tc_split_wide_kernel for its weights.
// The unit includes wunet_tc_kernels.cuh with WUNET_TC_CONV_ONLY, once per element type (namespaces wide::bf16, wide::f16),
// and instantiates only the forms above; the host code (wunet_tc.cu) reaches them through the functions at the end.
#include "wunet_common.cuh"
#include "wunet_wgmma.cuh"
#include "wunet_tc_common.cuh"

#include <algorithm>

#define WUNET_TC_CONV_ONLY 1

namespace wunet {
namespace wide {

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

namespace {
// channel slices of enc0_wide_kernel: a tile of 1024 / S rows of RC <= 128 channels stages at most 64 KiB
int enc0_slices(int split) { return split ? 4 : 2; }
size_t enc0_smem(int C, int split)
{
    const int tile = 1024 / enc0_slices(split), RC = split ? 2 * C : C;
    return (size_t)(15 * C + 2 * C + 4 + tile + 16) * sizeof(float) + (size_t)tile * RC * 2 + 16;
}
}  // namespace

void set_smem_attributes()
{
    const int enc0_max = (int)std::max(enc0_smem(64, 0), enc0_smem(64, 1));
    cudaFuncSetAttribute(bf16::conv_tc_kernel<15, false, kEpiWarpsLarge, 0, 0, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
    cudaFuncSetAttribute(bf16::conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 0, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         kSmemLimit);
    cudaFuncSetAttribute(bf16::enc0_wide_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, enc0_max);
    cudaFuncSetAttribute(bf16::enc0_wide_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, enc0_max);
    cudaFuncSetAttribute(f16::enc0_wide_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, enc0_max);
    io_f16::set_smem_attributes(enc0_max);               // and the 16-bit I/O forms of every unit (wunet_tc_io.cuh)
    io_bf16::set_smem_attributes(enc0_max);
}

cudaError_t launch_enc0(cudaLaunchConfig_t cfg, int mode, const void *x_io, const float *w, const float *scale, const float *shift, void *out,
                        int B, int T, int C, int io)
{
    const int split = mode == 1 ? 1 : 0;
    const int tile = 1024 / enc0_slices(split);
    cfg.gridDim = dim3((unsigned)((T + tile - 1) / tile), (unsigned)B, 1);
    cfg.blockDim = dim3(256);
    cfg.dynamicSmemBytes = enc0_smem(C, split);
    if (io == IO_F16) return io_f16::launch_enc0_wide(cfg, mode, x_io, w, scale, shift, out, B, T, C);
    if (io == IO_BF16) return io_bf16::launch_enc0_wide(cfg, mode, x_io, w, scale, shift, out, B, T, C);
    const float *x = static_cast<const float *>(x_io);
    if (mode == 2)
        return cudaLaunchKernelEx(&cfg, f16::enc0_wide_kernel<2>, x, w, scale, shift, static_cast<__half *>(out), B, T, C, 0);
    if (split)
        return cudaLaunchKernelEx(&cfg, bf16::enc0_wide_kernel<4>, x, w, scale, shift, static_cast<__nv_bfloat16 *>(out), B, T, C, 1);
    return cudaLaunchKernelEx(&cfg, bf16::enc0_wide_kernel<2>, x, w, scale, shift, static_cast<__nv_bfloat16 *>(out), B, T, C, 0);
}

ConvKernel conv_split_kernel(bool upcat)
{
    return upcat ? bf16::conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 0, 2>
                 : bf16::conv_tc_kernel<15, false, kEpiWarpsLarge, 0, 0, 2>;
}

cudaError_t pack_split(const float *w, void *wp, int Cout, int Cin, int K, int Npad, const SplitTable &tab, cudaStream_t stream)
{
    const size_t ns = (size_t)K * Npad * tab.n * 64;
    bf16::pack_tc_split_wide_kernel<<<(unsigned)((ns + 255) / 256), 256, 0, stream>>>(w, static_cast<__nv_bfloat16 *>(wp), Cout, Cin, K,
                                                                                      Npad, tab);
    return cudaGetLastError();
}

}  // namespace wide
}  // namespace wunet
