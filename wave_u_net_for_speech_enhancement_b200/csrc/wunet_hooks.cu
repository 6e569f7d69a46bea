// wunet_hooks.cu — device work behind the block forward hooks of the Python module (include/wunet_b200.h:
// wunet_forward_export, wunet_train_backward_inject): a stored block output converted to [B][C][L] in a 16-bit I/O type, and
// the addition of a hook's upstream gradient into a block's activation gradient. A unit of its own, so that no kernel of the
// forward or training units changes.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include "wunet_common.cuh"

namespace wunet {

namespace {

// element (b, c, l) of a stored block output, widened exactly to fp32 (LEVEL_*: wunet_common.cuh). The split form's value is
// hi + lo in fp32, as read_level computes it.
template <int KIND>
__device__ __forceinline__ float level_value(const void *src, int b, int c, int l, int L, int C)
{
    const size_t row = (size_t)b * L + l;
    if (KIND == LEVEL_BF16) return __bfloat162float(static_cast<const __nv_bfloat16 *>(src)[row * C + c]);
    if (KIND == LEVEL_F16) return __half2float(static_cast<const __half *>(src)[row * C + c]);
    if (KIND == LEVEL_SPLIT) {
        const __nv_bfloat16 *r = static_cast<const __nv_bfloat16 *>(src) + row * (2 * C);
        return __bfloat162float(r[c]) + __bfloat162float(r[C + c]);
    }
    return static_cast<const float *>(src)[((size_t)b * C + c) * L + l];      // LEVEL_F32_NCL
}

// dst [B][C][L] = the level, rounded once to OUT (nearest even)
template <int KIND, typename OUT>
__global__ void level_export_kernel(const void *__restrict__ src, OUT *__restrict__ dst, int B, int L, int C)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * C * L) return;
    const int l = (int)(i % L);
    const int c = (int)((i / L) % C);
    const int b = (int)(i / ((long long)L * C));
    io_st(dst + i, level_value<KIND>(src, b, c, l, L, C));
}

template <typename OUT>
void launch_export(const void *src, int kind, OUT *dst, int B, int L, int C, unsigned grid, cudaStream_t st)
{
    if (kind == LEVEL_BF16) level_export_kernel<LEVEL_BF16, OUT><<<grid, 256, 0, st>>>(src, dst, B, L, C);
    else if (kind == LEVEL_F16) level_export_kernel<LEVEL_F16, OUT><<<grid, 256, 0, st>>>(src, dst, B, L, C);
    else if (kind == LEVEL_SPLIT) level_export_kernel<LEVEL_SPLIT, OUT><<<grid, 256, 0, st>>>(src, dst, B, L, C);
    else level_export_kernel<LEVEL_F32_NCL, OUT><<<grid, 256, 0, st>>>(src, dst, B, L, C);
}

// ga[i] += g[i]: one add per element, so the sum does not depend on the launch
__global__ void grad_inject_kernel(float *__restrict__ ga, const float *__restrict__ g, long long n)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) ga[i] += g[i];
}

}  // namespace

int launch_level_export_io(const void *src, int kind, void *dst, int io, int B, int L, int C, cudaStream_t st)
{
    const long long n = (long long)B * C * L;
    const unsigned grid = (unsigned)((n + 255) / 256);
    if (io == IO_F16) launch_export(src, kind, static_cast<__half *>(dst), B, L, C, grid, st);
    else if (io == IO_BF16) launch_export(src, kind, static_cast<__nv_bfloat16 *>(dst), B, L, C, grid, st);
    else return -1;
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_grad_inject(float *ga, const float *g, long long n, cudaStream_t st)
{
    grad_inject_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ga, g, n);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace wunet
