// wunet_train.cu — training step of the Wave-U-Net (SURVEY.md §8f row N1): forward with BatchNorm1d in training mode and the
// backward pass, fp32, NCL layout, CUDA cores (one formula per kernel, in the order autograd would replay them); checked
// against float64 golden steps (tests/test_train_gpu.py). The three convolution-shaped passes carry ~99 % of the work:
//   forward conv and input gradient  -> the tuned fp32 kernels of wunet_fp32.cu (sliding-window / implicit GEMM) with a linear
//                                       epilogue; the input gradient is the same convolution with the weights transposed and
//                                       flipped, read from dz (train_pack_kernel writes both packings every step);
//   weight gradient                  -> train_wgrad_kernel below (register-tiled reduction over (batch, position) tiles staged in
//                                       shared memory, split over the batch, combined with atomicAdd).
// TRAIN_DETERMINISTIC replaces the two float-atomic combines (weight gradients, head gradients) with partial sums stored to a
// scratch region after the workspace layout and summed in an order fixed by the shapes (train_slice_sum_kernel,
// train_head_sum_kernel); every other reduction of the step already has a fixed order.
// The naive one-thread-per-output kernels they replace are kept as WUNET_TRAIN_NAIVE=1 (cross-check, tests).
// TRAIN_BF16 / TRAIN_TF32 / TRAIN_FP16_SCALED (Model(train_precision="bf16" / "tf32" / "fp16_scaled")): the forward conv,
// input gradient and weight gradient of every block but the first (Cin = 1) run on the tensor-core kernels of
// wunet_train_tc_kernels.cuh at that operand precision instead; everything else is the same fp32 code. TRAIN_FP16_SCALED adds
// one reduction per block: the BatchNorm backward that writes dz also finds max |dz| (train_bn_bwd_apply_amax_kernel), from
// which the two passes that read dz take its power-of-two scale on the device (no host sync; max is order-independent).
// TRAIN_FROZEN_BN (eval-mode BatchNorm: running statistics, never updated) and TRAIN_NO_PARAM_GRADS (input gradient only) only
// change the BatchNorm arithmetic and which reductions run; the convolution-shaped passes are the same kernels. The same holds
// per block (bn_frozen) and per parameter (null gradient slots), with an early stop below the lowest block that needs a
// gradient (fine-tuning with frozen layers; DESIGN §5.4). The input
// gradient dx is train_input_grad_kernel below (head's raw-input channel + block 0's transposed conv).
// BnSync (nn.SyncBatchNorm over data-parallel ranks): the batch-statistics reductions are split at the cross-rank sums
// (train_bn_sync_* kernels, a host hook between them); without it the step issues exactly the launches it always did.
//
// Reference: trainer/trainer.py:34-38 (forward, loss.backward()), model/unet_basic.py:77-100 with the BatchNorm1d of
// :12, :25, :55 in .train() mode (batch statistics; running statistics updated with momentum 0.1 and the unbiased variance).
// The parameters are read in the reference's own layouts straight from the torch tensors (they change every step: there
// is nothing to pack), gradients are written in the same layouts.
#include "wunet_train.cuh"
#include "wunet_common.cuh"

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <vector>

namespace wunet {

namespace {

thread_local char g_train_err[512] = "";
int train_fail(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_train_err, sizeof(g_train_err), fmt, ap);
    va_end(ap);
    return -1;
}

// ---------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------
// z[b][co][l] = bias[co] + sum_ci sum_k in(b, ci, l + k - pad) * w[co][ci][k]        (Conv1d, model/unet_basic.py:10,23,53)
// `in` is the block input the reference builds between two convolutions (decimate / interpolate + cat), fetched on the fly.
template <int KS, int MODE>
__global__ void __launch_bounds__(128) train_conv_fwd_kernel(const ConvArgs a, const float *__restrict__ w,
                                                             const float *__restrict__ bias, float *__restrict__ z)
{
    constexpr int PAD = (KS - 1) / 2, CO = 8;
    const int l = blockIdx.x * 128 + threadIdx.x;
    const int co0 = blockIdx.y * CO;
    const int b = blockIdx.z;
    float acc[CO];
#pragma unroll
    for (int j = 0; j < CO; ++j) acc[j] = 0.f;
    for (int ci = 0; ci < a.Cin; ++ci) {
        float xin[KS];
#pragma unroll
        for (int k = 0; k < KS; ++k) xin[k] = fetch_src<MODE>(a, b, ci, l + k - PAD);
#pragma unroll
        for (int j = 0; j < CO; ++j) {
            if (co0 + j < a.Cout) {
                const float *wr = w + ((size_t)(co0 + j) * a.Cin + ci) * KS;
#pragma unroll
                for (int k = 0; k < KS; ++k) acc[j] = fmaf(xin[k], __ldg(wr + k), acc[j]);
            }
        }
    }
    if (l < a.L) {
#pragma unroll
        for (int j = 0; j < CO; ++j)
            if (co0 + j < a.Cout) z[((size_t)b * a.Cout + co0 + j) * a.L + l] = acc[j] + __ldg(bias + co0 + j);
    }
}

__device__ __forceinline__ double block_sum(double v, double *sh)
{
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    double t = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += sh[i];
    return t;
}

// BatchNorm1d training statistics of channel c = blockIdx.x over (B, L): two passes in double; the running statistics of
// the module are updated in place: rm = (1-m) rm + m mean, rv = (1-m) rv + m var * n/(n-1)   (torch.nn.BatchNorm1d)
__global__ void __launch_bounds__(256) train_bn_stats_kernel(const float *__restrict__ z, int B, int C, int L, float momentum,
                                                             float *__restrict__ mean, float *__restrict__ invstd,
                                                             float *__restrict__ running_mean, float *__restrict__ running_var)
{
    __shared__ double sh[8];
    const int c = blockIdx.x;
    const long long n = (long long)B * L;
    double s = 0.0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const int b = (int)(i / L), l = (int)(i - (long long)b * L);
        s += (double)z[((size_t)b * C + c) * L + l];
    }
    const double mu = block_sum(s, sh) / (double)n;
    double q = 0.0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const int b = (int)(i / L), l = (int)(i - (long long)b * L);
        const double d = (double)z[((size_t)b * C + c) * L + l] - mu;
        q += d * d;
    }
    const double var = block_sum(q, sh) / (double)n;          // biased: what normalises the batch
    if (threadIdx.x == 0) {
        mean[c] = (float)mu;
        invstd[c] = (float)(1.0 / sqrt(var + (double)kBnEps));
        const double unbiased = var * ((double)n / (double)(n > 1 ? n - 1 : 1));
        running_mean[c] = (float)((1.0 - momentum) * (double)running_mean[c] + momentum * mu);
        running_var[c] = (float)((1.0 - momentum) * (double)running_var[c] + momentum * unbiased);
    }
}

// The same statistics synchronised over data-parallel ranks (nn.SyncBatchNorm; BnSync), split where the cross-rank sums go.
// Each pass has train_bn_stats_kernel's loop and block_sum order, so a pass-through hook reproduces it bit for bit.
// pass 1: buf[c] = local sum z, buf[C] = local B L                                  -> hook(buf, C + 1)
__global__ void __launch_bounds__(256) train_bn_sync_sum_kernel(const float *__restrict__ z, int B, int C, int L,
                                                                double *__restrict__ buf)
{
    __shared__ double sh[8];
    const int c = blockIdx.x;
    const long long n = (long long)B * L;
    double s = 0.0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const int b = (int)(i / L), l = (int)(i - (long long)b * L);
        s += (double)z[((size_t)b * C + c) * L + l];
    }
    const double t = block_sum(s, sh);
    if (threadIdx.x == 0) {
        buf[c] = t;
        if (c == 0) buf[C] = (double)n;
    }
}

// pass 2: buf[C + 1 + c] = local sum (z - mean)^2 about the global mean buf[c] / buf[C]        -> hook(buf + C + 1, C)
__global__ void __launch_bounds__(256) train_bn_sync_centred_kernel(const float *__restrict__ z, int B, int C, int L,
                                                                    double *__restrict__ buf)
{
    __shared__ double sh[8];
    const int c = blockIdx.x;
    const long long n = (long long)B * L;
    const double mu = buf[c] / buf[C];
    double q = 0.0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const int b = (int)(i / L), l = (int)(i - (long long)b * L);
        const double d = (double)z[((size_t)b * C + c) * L + l] - mu;
        q += d * d;
    }
    const double t = block_sum(q, sh);
    if (threadIdx.x == 0) buf[C + 1 + c] = t;
}

// mean, invstd and the running statistics from the global sums, rounded as train_bn_stats_kernel rounds them
__global__ void train_bn_sync_finalize_kernel(const double *__restrict__ buf, int C, float momentum, float *__restrict__ mean,
                                              float *__restrict__ invstd, float *__restrict__ running_mean,
                                              float *__restrict__ running_var)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const double nd = buf[C];
    const long long n = (long long)nd;
    const double mu = buf[c] / nd;
    const double var = buf[C + 1 + c] / nd;
    mean[c] = (float)mu;
    invstd[c] = (float)(1.0 / sqrt(var + (double)kBnEps));
    const double unbiased = var * ((double)n / (double)(n > 1 ? n - 1 : 1));
    running_mean[c] = (float)((1.0 - momentum) * (double)running_mean[c] + momentum * mu);
    running_var[c] = (float)((1.0 - momentum) * (double)running_var[c] + momentum * unbiased);
}

// eval-mode BatchNorm (TRAIN_FROZEN_BN, model/unet_basic.py in .eval()): normalise by the running statistics, rounding invstd
// as the batch-statistics path does; the running buffers are only read
__global__ void train_bn_frozen_stats_kernel(const float *__restrict__ running_mean, const float *__restrict__ running_var,
                                             float *__restrict__ mean, float *__restrict__ invstd, int C)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    mean[c] = running_mean[c];
    invstd[c] = (float)(1.0 / sqrt((double)running_var[c] + (double)kBnEps));
}

// a = LeakyReLU(gamma * (z - mean) * invstd + beta)
__global__ void train_bn_act_kernel(const float *__restrict__ z, const float *__restrict__ mean, const float *__restrict__ invstd,
                                    const float *__restrict__ gamma, const float *__restrict__ beta, float *__restrict__ act,
                                    int B, int C, int L)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * C * L) return;
    const int c = (int)((i / L) % C);
    const float y = fmaf(gamma[c], (z[i] - mean[c]) * invstd[c], beta[c]);
    act[i] = y >= 0.f ? y : kLreluSlope * y;
}

// ---------------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------------
// head: y = tanh(sum_c Wo[c] cat[c] + bo), cat = [a_last (C channels) | x]   (model/unet_basic.py:98-99)
//   dpre = dy (1 - y^2);  dWo[c] = sum dpre cat[c];  dbo = sum dpre;  d a_last[c] = Wo[c] dpre
// g_wo == nullptr (TRAIN_NO_PARAM_GRADS): d a_last only. The warp sums of dWo and dbo are combined with atomicAdd or, with
// PARTIALS (deterministic mode), summed in warp order per CTA in double and stored to part[blockIdx.x][C + 2] (dWo, dbo) for
// train_head_sum_kernel.
template <bool PARTIALS>
__global__ void __launch_bounds__(256) train_head_bwd_kernel(const float *__restrict__ dy, const float *__restrict__ y,
                                                             const float *__restrict__ a_last, const float *__restrict__ x,
                                                             const float *__restrict__ wo, float *__restrict__ ga_last,
                                                             float *__restrict__ g_wo, float *__restrict__ g_bo,
                                                             double *__restrict__ part, int B, int C, int T)
{
    __shared__ double sh[8];
    // warp sum of v -> g[c] (atomically) or -> part (CTA sum in warp order); every thread of the CTA calls it
    auto combine = [&](float v, float *g, int c) {
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (!PARTIALS) {
            if ((threadIdx.x & 31) == 0) atomicAdd(g, v);
            return;
        }
        if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = (double)v;
        __syncthreads();
        if (threadIdx.x == 0) {
            double s = 0.0;
            for (int w = 0; w < 8; ++w) s += sh[w];
            part[(size_t)blockIdx.x * (C + 2) + c] = s;
        }
        __syncthreads();
    };
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;      // over [B][T]
    const bool ok = i < (long long)B * T;
    const int b = ok ? (int)(i / T) : 0, l = ok ? (int)(i - (long long)b * T) : 0;
    const float yv = ok ? y[i] : 0.f;
    const float dpre = ok ? dy[i] * (1.f - yv * yv) : 0.f;
    if (!g_wo) {
        if (ok)
            for (int c = 0; c < C; ++c) ga_last[((size_t)b * C + c) * T + l] = wo[c] * dpre;
        return;
    }
    for (int c = 0; c <= C; ++c) {
        float v;
        if (c < C) {
            const size_t idx = ((size_t)b * C + c) * T + l;
            v = ok ? dpre * a_last[idx] : 0.f;
            if (ok) ga_last[idx] = wo[c] * dpre;
        } else {
            v = ok ? dpre * x[i] : 0.f;
        }
        combine(v, g_wo + c, c);
    }
    combine(dpre, g_bo, C + 1);
}

// deterministic head gradients: out c (0 .. C: dWo[c], C + 1: dbo) = blockIdx.x of this kernel, the sum of the nparts CTA
// partials of train_head_bwd_kernel<true> in double, in a fixed order (strided per thread, then block_sum)
__global__ void __launch_bounds__(256) train_head_sum_kernel(const double *__restrict__ part, int nparts, int C,
                                                             float *__restrict__ g_wo, float *__restrict__ g_bo)
{
    __shared__ double sh[8];
    const int c = blockIdx.x;
    double s = 0.0;
    for (int j = threadIdx.x; j < nparts; j += blockDim.x) s += part[(size_t)j * (C + 2) + c];
    const double t = block_sum(s, sh);
    if (threadIdx.x == 0) {
        if (c <= C) g_wo[c] = (float)t;
        else *g_bo = (float)t;
    }
}

// deterministic weight gradients: dw[i] = sum over the slices z = 0, 1, ... of part[z * n + i], in that order, in double
__global__ void train_slice_sum_kernel(const float *__restrict__ part, float *__restrict__ dw, int slices, long long n)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double s = 0.0;
    for (int z = 0; z < slices; ++z) s += (double)part[(size_t)z * n + i];
    dw[i] = (float)s;
}

// BatchNorm + LeakyReLU backward, reductions of channel c = blockIdx.x:
//   dy = da * (y >= 0 ? 1 : slope), y = gamma zh + beta, zh = (z - mean) invstd;   dbeta = sum dy;  dgamma = sum dy zh
__global__ void __launch_bounds__(256) train_bn_bwd_stats_kernel(const float *__restrict__ ga, const float *__restrict__ z,
                                                                 const float *__restrict__ mean, const float *__restrict__ invstd,
                                                                 const float *__restrict__ gamma, const float *__restrict__ beta,
                                                                 float *__restrict__ g_gamma, float *__restrict__ g_beta,
                                                                 float *__restrict__ s1, float *__restrict__ s2, int B, int C, int L)
{
    __shared__ double sh[8];
    const int c = blockIdx.x;
    const long long n = (long long)B * L;
    const float mu = mean[c], is = invstd[c], g = gamma[c], be = beta[c];
    double a1 = 0.0, a2 = 0.0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const int b = (int)(i / L), l = (int)(i - (long long)b * L);
        const size_t idx = ((size_t)b * C + c) * L + l;
        const float zh = (z[idx] - mu) * is;
        const float yv = fmaf(g, zh, be);
        const float dyv = yv >= 0.f ? ga[idx] : kLreluSlope * ga[idx];
        a1 += (double)dyv;
        a2 += (double)dyv * (double)zh;
    }
    const double t1 = block_sum(a1, sh);
    const double t2 = block_sum(a2, sh);
    if (threadIdx.x == 0) {
        if (g_beta) g_beta[c] = (float)t1;                     // null under TRAIN_NO_PARAM_GRADS
        if (g_gamma) g_gamma[c] = (float)t2;
        s1[c] = (float)(t1 / (double)n);                        // mean(dy), mean(dy zh): what the input gradient needs
        s2[c] = (float)(t2 / (double)n);
    }
}

// The same reductions synchronised over data-parallel ranks (BnSync), train_bn_bwd_stats_kernel's loop and block_sum order:
// g_beta, g_gamma get the LOCAL sums (the gradient all-reduce averages them, as with nn.SyncBatchNorm under DDP);
// buf = [sum dy | sum dy zh | B L] (2C + 1)                                            -> hook(buf, 2C + 1)
__global__ void __launch_bounds__(256) train_bn_sync_bwd_sums_kernel(const float *__restrict__ ga, const float *__restrict__ z,
                                                                     const float *__restrict__ mean, const float *__restrict__ invstd,
                                                                     const float *__restrict__ gamma, const float *__restrict__ beta,
                                                                     float *__restrict__ g_gamma, float *__restrict__ g_beta,
                                                                     double *__restrict__ buf, int B, int C, int L)
{
    __shared__ double sh[8];
    const int c = blockIdx.x;
    const long long n = (long long)B * L;
    const float mu = mean[c], is = invstd[c], g = gamma[c], be = beta[c];
    double a1 = 0.0, a2 = 0.0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const int b = (int)(i / L), l = (int)(i - (long long)b * L);
        const size_t idx = ((size_t)b * C + c) * L + l;
        const float zh = (z[idx] - mu) * is;
        const float yv = fmaf(g, zh, be);
        const float dyv = yv >= 0.f ? ga[idx] : kLreluSlope * ga[idx];
        a1 += (double)dyv;
        a2 += (double)dyv * (double)zh;
    }
    const double t1 = block_sum(a1, sh);
    const double t2 = block_sum(a2, sh);
    if (threadIdx.x == 0) {
        if (g_beta) g_beta[c] = (float)t1;                     // null under TRAIN_NO_PARAM_GRADS
        if (g_gamma) g_gamma[c] = (float)t2;
        buf[c] = t1;
        buf[C + c] = t2;
        if (c == 0) buf[2 * C] = (double)n;
    }
}

// s1 = mean(dy), s2 = mean(dy zh) over every rank's frames, from the global sums
__global__ void train_bn_sync_bwd_finalize_kernel(const double *__restrict__ buf, int C, float *__restrict__ s1,
                                                  float *__restrict__ s2)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    s1[c] = (float)(buf[c] / buf[2 * C]);
    s2[c] = (float)(buf[C + c] / buf[2 * C]);
}

//   dz = invstd gamma (dy - mean(dy) - zh mean(dy zh))      of element i of [B][C][L], from da = ga[i]
// With s1 = s2 = 0 this is the eval-mode (frozen statistics) BatchNorm backward, dz = invstd gamma dy.
__device__ __forceinline__ float bn_bwd_dz(const float *__restrict__ ga, const float *__restrict__ z, const float *__restrict__ mean,
                                           const float *__restrict__ invstd, const float *__restrict__ gamma,
                                           const float *__restrict__ beta, const float *__restrict__ s1,
                                           const float *__restrict__ s2, long long i, int C, int L)
{
    const int c = (int)((i / L) % C);
    const float zh = (z[i] - mean[c]) * invstd[c];
    const float yv = fmaf(gamma[c], zh, beta[c]);
    const float dyv = yv >= 0.f ? ga[i] : kLreluSlope * ga[i];
    return invstd[c] * gamma[c] * (dyv - s1[c] - zh * s2[c]);
}

// dz written over ga (in place)
__global__ void train_bn_bwd_apply_kernel(float *__restrict__ ga, const float *__restrict__ z, const float *__restrict__ mean,
                                          const float *__restrict__ invstd, const float *__restrict__ gamma,
                                          const float *__restrict__ beta, const float *__restrict__ s1,
                                          const float *__restrict__ s2, int B, int C, int L)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * C * L) return;
    ga[i] = bn_bwd_dz(ga, z, mean, invstd, gamma, beta, s1, s2, i, C, L);
}

// max |v| of a thread's values (as bits: non-negative floats order as their bits, NaN above inf) -> *amax, one atomicMax per
// warp (*amax zeroed first); every lane of the warp calls it
__device__ __forceinline__ void warp_amax_combine(unsigned m, float *amax)
{
    m = __reduce_max_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0 && m) atomicMax(reinterpret_cast<unsigned *>(amax), m);
}
constexpr int kAmaxCtas = 8 * 132;         // grid of the max |dz| kernels (grid-stride): a few thousand atomics per block

// TRAIN_FP16_SCALED: train_bn_bwd_apply_kernel's dz, and max |dz| of the block -> *amax (the block's scale slot)
__global__ void __launch_bounds__(256) train_bn_bwd_apply_amax_kernel(float *__restrict__ ga, const float *__restrict__ z,
                                                                      const float *__restrict__ mean, const float *__restrict__ invstd,
                                                                      const float *__restrict__ gamma, const float *__restrict__ beta,
                                                                      const float *__restrict__ s1, const float *__restrict__ s2,
                                                                      int B, int C, int L, float *__restrict__ amax)
{
    const long long n = (long long)B * C * L;
    unsigned m = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float d = bn_bwd_dz(ga, z, mean, invstd, gamma, beta, s1, s2, i, C, L);
        ga[i] = d;
        m = max(m, __float_as_uint(fabsf(d)));
    }
    warp_amax_combine(m, amax);
}

// max |src[i]| over n values -> *amax (zeroed first): the scale of dz in wunet_debug_train_conv
__global__ void __launch_bounds__(256) train_amax_kernel(const float *__restrict__ src, long long n, float *__restrict__ amax)
{
    unsigned m = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        m = max(m, __float_as_uint(fabsf(src[i])));
    warp_amax_combine(m, amax);
}

// out[c] = sum over (b, l) of src[b][c][l]      (conv bias gradient: db = sum dz)
__global__ void __launch_bounds__(256) train_channel_sum_kernel(const float *__restrict__ src, float *__restrict__ out, int B, int C, int L)
{
    __shared__ double sh[8];
    const int c = blockIdx.x;
    const long long n = (long long)B * L;
    double s = 0.0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const int b = (int)(i / L), l = (int)(i - (long long)b * L);
        s += (double)src[((size_t)b * C + c) * L + l];
    }
    const double t = block_sum(s, sh);
    if (threadIdx.x == 0) out[c] = (float)t;
}

// din[b][ci][l] = sum_co sum_k dz[b][co][l - k + pad] * w[co][ci][k]      (gradient of the block input, dense [B][Cin][L])
template <int KS>
__global__ void __launch_bounds__(128) train_conv_bwd_data_kernel(const float *__restrict__ dz, const float *__restrict__ w,
                                                                  float *__restrict__ din, int B, int Cin, int Cout, int L)
{
    constexpr int PAD = (KS - 1) / 2, CI = 8;
    const int l = blockIdx.x * 128 + threadIdx.x;
    const int ci0 = blockIdx.y * CI;
    const int b = blockIdx.z;
    float acc[CI];
#pragma unroll
    for (int j = 0; j < CI; ++j) acc[j] = 0.f;
    for (int co = 0; co < Cout; ++co) {
        float d[KS];
        const float *dr = dz + ((size_t)b * Cout + co) * L;
#pragma unroll
        for (int k = 0; k < KS; ++k) {
            const int p = l - k + PAD;
            d[k] = (p >= 0 && p < L) ? __ldg(dr + p) : 0.f;
        }
#pragma unroll
        for (int j = 0; j < CI; ++j) {
            if (ci0 + j < Cin) {
                const float *wr = w + ((size_t)co * Cin + ci0 + j) * KS;
#pragma unroll
                for (int k = 0; k < KS; ++k) acc[j] = fmaf(d[k], __ldg(wr + k), acc[j]);
            }
        }
    }
    if (l < L) {
#pragma unroll
        for (int j = 0; j < CI; ++j)
            if (ci0 + j < Cin) din[((size_t)b * Cin + ci0 + j) * L + l] = acc[j];
    }
}

// dW[co][ci][k] = sum_b sum_l dz[b][co][l] * in(b, ci, l + k - pad).  Block = (co, group of 4 ci, slice of the batch);
// the slices are combined with atomicAdd (dW is zeroed first); there is no deterministic form (TRAIN_DETERMINISTIC refuses it).
template <int KS, int MODE>
__global__ void __launch_bounds__(128) train_conv_bwd_weight_kernel(const ConvArgs a, const float *__restrict__ dz, float *__restrict__ dw)
{
    constexpr int PAD = (KS - 1) / 2, CI = 4;
    __shared__ float sh[4][CI * KS];
    const int co = blockIdx.x;
    const int ci0 = blockIdx.y * CI;
    float acc[CI][KS];
#pragma unroll
    for (int j = 0; j < CI; ++j)
#pragma unroll
        for (int k = 0; k < KS; ++k) acc[j][k] = 0.f;
    for (int b = blockIdx.z; b < a.B; b += gridDim.z) {
        const float *dr = dz + ((size_t)b * a.Cout + co) * a.L;
        for (int l = threadIdx.x; l < a.L; l += 128) {
            const float d = __ldg(dr + l);
#pragma unroll
            for (int j = 0; j < CI; ++j) {
                if (ci0 + j < a.Cin) {
#pragma unroll
                    for (int k = 0; k < KS; ++k) acc[j][k] = fmaf(d, fetch_src<MODE>(a, b, ci0 + j, l + k - PAD), acc[j][k]);
                }
            }
        }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int j = 0; j < CI; ++j)
#pragma unroll
        for (int k = 0; k < KS; ++k) {
            float v = acc[j][k];
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0) sh[warp][j * KS + k] = v;
        }
    __syncthreads();
    if (threadIdx.x < CI * KS) {
        const int j = threadIdx.x / KS, k = threadIdx.x - j * KS;
        if (ci0 + j < a.Cin) {
            const float v = sh[0][threadIdx.x] + sh[1][threadIdx.x] + sh[2][threadIdx.x] + sh[3][threadIdx.x];
            atomicAdd(dw + ((size_t)co * a.Cin + ci0 + j) * KS + k, v);
        }
    }
}

// adjoint of o[:, :, ::2]  (model/unet_basic.py:86):  g_prev[b][c][2l] += din[b][c][l]
__global__ void train_decim_adjoint_kernel(const float *__restrict__ din, float *__restrict__ g_prev, int B, int C, int L)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;      // over [B][C][L]
    if (i >= (long long)B * C * L) return;
    const long long bc = i / L;
    const int l = (int)(i - bc * L);
    g_prev[bc * (2LL * L) + 2 * l] += din[i];
}

// decoder block input = cat([interp2x(prev), skip]) (model/unet_basic.py:93-95): the skip half of din is the gradient of the
// encoder activation (first contribution: plain store) ...
__global__ void train_skip_grad_kernel(const float *__restrict__ din, float *__restrict__ g_skip, int B, int Cin, int Cin0, int L)
{
    const int Cs = Cin - Cin0;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;      // over [B][Cs][L]
    if (i >= (long long)B * Cs * L) return;
    const int l = (int)(i % L);
    const int c = (int)((i / L) % Cs);
    const int b = (int)(i / ((long long)L * Cs));
    g_skip[i] = din[((size_t)b * Cin + Cin0 + c) * L + l];
}
// ... and the first Cin0 channels go through the adjoint of the linear interpolation (align_corners=True, fp32 index math
// as in the forward): g_prev[b][c][m] = sum_l U[l][m] din[b][c][l], gathered over the few l whose i0 or i1 equals m.
__global__ void train_upsample_adjoint_kernel(const float *__restrict__ din, float *__restrict__ g_prev, int B, int Cin, int Cin0,
                                              int L, float up_scale)
{
    const int Lin = L >> 1;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;      // over [B][Cin0][Lin]
    if (i >= (long long)B * Cin0 * Lin) return;
    const int m = (int)(i % Lin);
    const int c = (int)((i / Lin) % Cin0);
    const int b = (int)(i / ((long long)Lin * Cin0));
    const float *dr = din + ((size_t)b * Cin + c) * L;
    float acc = 0.f;
    for (int l = 2 * m - 2; l <= 2 * m + 3; ++l) {
        if (l < 0 || l >= L) continue;
        const float s = up_scale * (float)l;
        const int i0 = (int)s;
        const int i1 = i0 + (i0 < Lin - 1 ? 1 : 0);
        const float lam1 = s - (float)i0;
        const float lam0 = 1.f - lam1;
        const float d = dr[l];
        if (i0 == m) acc = fmaf(lam0, d, acc);
        if (i1 == m) acc = fmaf(lam1, d, acc);
    }
    g_prev[i] = acc;
}

// gradient of the network input x [B][1][T]: the head's raw-input channel (model/unet_basic.py:98-99) plus the input gradient
// of block 0 (Cin = 1, a transposed convolution of dz0 = the block's dz):
//   dx[b][t] = Wo[C] dy (1 - y^2) + sum_co sum_k w0[co][0][k] dz0[b][co][t + PAD - k]
// One thread per sample; each step of the channel loop stages IN_CH channels of a dz0 tile with its KS - 1 halo and their
// weights in shared memory, so dz0 is read once. fp32 at both training precisions (block 0 always runs fp32).
template <int KS>
__global__ void __launch_bounds__(256) train_input_grad_kernel(const float *__restrict__ dz0, const float *__restrict__ w0,
                                                               const float *__restrict__ dy, const float *__restrict__ y,
                                                               const float *__restrict__ wo, float *__restrict__ dx, int C0,
                                                               int C, int T)
{
    constexpr int PAD = (KS - 1) / 2, TILE = 256, IN_CH = 8, W = TILE + KS - 1;
    __shared__ float ds[IN_CH][W];
    __shared__ float ws[IN_CH][KS];
    const int tid = threadIdx.x, b = blockIdx.y;
    const int l0 = blockIdx.x * TILE, l = l0 + tid;
    float acc = 0.f;
    for (int c0 = 0; c0 < C0; c0 += IN_CH) {
        __syncthreads();
        for (int i = tid; i < IN_CH * W; i += TILE) {
            const int c = i / W, j = i - c * W, p = l0 - PAD + j;
            ds[c][j] = (c0 + c < C0 && p >= 0 && p < T) ? __ldg(dz0 + ((size_t)b * C0 + c0 + c) * T + p) : 0.f;
        }
        if (tid < IN_CH * KS) {
            const int c = tid / KS, k = tid - c * KS;
            ws[c][k] = c0 + c < C0 ? __ldg(w0 + (size_t)(c0 + c) * KS + k) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int c = 0; c < IN_CH; ++c)
#pragma unroll
            for (int k = 0; k < KS; ++k) acc = fmaf(ds[c][tid + 2 * PAD - k], ws[c][k], acc);
    }
    if (l < T) {
        const size_t i = (size_t)b * T + l;
        const float yv = y[i];
        dx[i] = fmaf(wo[C], dy[i] * (1.f - yv * yv), acc);
    }
}

// both packings of a block's weights, every step (the parameters change every step):
//   wf[(ci*K + k)*Cout + co] = w[co][ci][k]            forward conv, operand layout of wunet_fp32.cu
//   wb[(co*K + k)*Cin + ci]  = w[co][ci][K-1-k]        input gradient = conv of dz with the transposed, flipped weights
__global__ void train_pack_kernel(const float *__restrict__ w, float *__restrict__ wf, float *__restrict__ wb, int Cout, int Cin, int K)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)Cout * Cin * K) return;
    const int k = (int)(i % K);
    const int ci = (int)((i / K) % Cin);
    const int co = (int)(i / ((long long)K * Cin));
    const float v = w[i];
    wf[((size_t)ci * K + k) * Cout + co] = v;
    wb[((size_t)co * K + (K - 1 - k)) * Cin + ci] = v;
}

__global__ void train_fill_kernel(float *__restrict__ p, float v, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// dW[co][ci][k] = sum_b sum_l dz[b][co][l] * in(b, ci, l + k - pad).
// Block = 16 co x 64 ci; thread = 2 co x 2 ci x KS taps of accumulators (a warp shares its co pair: dz reads are broadcasts;
// its lanes own ci = lane and lane + 32: conflict-free rows). The reduction runs over tiles of `lt` positions of one frame,
// staged in shared memory (the block input is built on the fly by fetch_src: decimate / interpolate + cat), 4 positions per
// inner step: 2 x (4 + KS - 1) + 8 shared loads for 16 KS FFMA. gridDim.z slices of the (frame, tile) list are combined
// with atomicAdd (dW is zeroed first) or, with SLICES (deterministic mode), each slice stores its partial sums to its own
// copy of dW at dw + blockIdx.z * Cout Cin KS.
template <int KS, int MODE, bool SLICES>
__global__ void __launch_bounds__(256) train_wgrad_kernel(const ConvArgs a, const float *__restrict__ dz, float *__restrict__ dw, int lt)
{
    constexpr int PAD = (KS - 1) / 2, CO_T = 16, CI_T = 64, LT_MAX = 128;
    constexpr int XP = LT_MAX + KS - 1 + ((LT_MAX + KS - 1) % 2 == 0 ? 1 : 0);      // odd row pitch
    __shared__ float xs[CI_T][XP];
    __shared__ float ds[CO_T][LT_MAX];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int co0 = blockIdx.x * CO_T, ci0 = blockIdx.y * CI_T;
    const int tiles_per_frame = (a.L + lt - 1) / lt;
    const int ntiles = a.B * tiles_per_frame;
    float acc[2][2][KS];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int k = 0; k < KS; ++k) acc[i][j][k] = 0.f;
    const int lt4 = (lt + 3) & ~3;                    // the inner loop takes 4 positions at a time: frames of 1 or 2 samples are
    const int xw = lt4 + KS - 1;                       // padded with zero gradients / out-of-frame (zero) inputs
    for (int t = blockIdx.z; t < ntiles; t += gridDim.z) {
        const int b = t / tiles_per_frame;
        const int l0 = (t - b * tiles_per_frame) * lt;
        __syncthreads();
        for (int i = tid; i < CI_T * xw; i += 256) {
            const int ci = i / xw, j = i - ci * xw;
            xs[ci][j] = (ci0 + ci < a.Cin) ? fetch_src<MODE>(a, b, ci0 + ci, l0 - PAD + j) : 0.f;
        }
        for (int i = tid; i < CO_T * lt4; i += 256) {
            const int co = i / lt4, j = i - co * lt4;
            ds[co][j] = (co0 + co < a.Cout && j < lt && l0 + j < a.L) ? __ldg(dz + ((size_t)b * a.Cout + co0 + co) * a.L + l0 + j) : 0.f;
        }
        __syncthreads();
#pragma unroll 1
        for (int l = 0; l < lt; l += 4) {
            float x0[4 + KS - 1], x1[4 + KS - 1], d0[4], d1[4];
#pragma unroll
            for (int j = 0; j < 4 + KS - 1; ++j) { x0[j] = xs[lane][l + j]; x1[j] = xs[lane + 32][l + j]; }
#pragma unroll
            for (int j = 0; j < 4; ++j) { d0[j] = ds[2 * warp][l + j]; d1[j] = ds[2 * warp + 1][l + j]; }
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int k = 0; k < KS; ++k) {
                    acc[0][0][k] = fmaf(d0[j], x0[j + k], acc[0][0][k]);
                    acc[0][1][k] = fmaf(d0[j], x1[j + k], acc[0][1][k]);
                    acc[1][0][k] = fmaf(d1[j], x0[j + k], acc[1][0][k]);
                    acc[1][1][k] = fmaf(d1[j], x1[j + k], acc[1][1][k]);
                }
        }
    }
    if (SLICES) dw += (size_t)blockIdx.z * a.Cout * a.Cin * KS;
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int co = co0 + 2 * warp + i, ci = ci0 + lane + 32 * j;
            if (co < a.Cout && ci < a.Cin) {
#pragma unroll
                for (int k = 0; k < KS; ++k) {
                    float *d = dw + ((size_t)co * a.Cin + ci) * KS + k;
                    if (SLICES) *d = acc[i][j][k];
                    else atomicAdd(d, acc[i][j][k]);
                }
            }
        }
}

template <bool SLICES>
void launch_wgrad_fp32_as(const ConvArgs &a, const float *dz, float *dw, int mode, cudaStream_t st)
{
    const WgradGrid g = wgrad_grid_fp32(a.B, a.L, a.Cin, a.Cout);
    if (mode == SRC_DIRECT) train_wgrad_kernel<15, SRC_DIRECT, SLICES><<<g.grid, 256, 0, st>>>(a, dz, dw, g.positions);
    else if (mode == SRC_DECIM) train_wgrad_kernel<15, SRC_DECIM, SLICES><<<g.grid, 256, 0, st>>>(a, dz, dw, g.positions);
    else train_wgrad_kernel<5, SRC_UPCAT, SLICES><<<g.grid, 256, 0, st>>>(a, dz, dw, g.positions);
}

// the tiled fp32 weight gradient (dw zeroed first; with `slices`, the per-slice partial sums of train_wgrad_kernel<.., true>);
// mode DIRECT / DECIM: 15 taps, UPCAT: 5
void launch_wgrad_fp32(const ConvArgs &a, const float *dz, float *dw, int mode, cudaStream_t st, bool slices = false)
{
    if (slices) launch_wgrad_fp32_as<true>(a, dz, dw, mode, st);
    else launch_wgrad_fp32_as<false>(a, dz, dw, mode, st);
}

struct Shape { int cin, cout, k, L, mode, cin0, cin1; };

void shapes_of(int n, int ci, int T, std::vector<Shape> &sh)
{
    sh.clear();
    for (int i = 0; i < n; ++i) sh.push_back(Shape{i == 0 ? 1 : i * ci, (i + 1) * ci, 15, T >> i, i == 0 ? SRC_DIRECT : SRC_DECIM, i == 0 ? 1 : i * ci, 0});
    sh.push_back(Shape{n * ci, n * ci, 15, T >> n, SRC_DECIM, n * ci, 0});
    for (int j = 0; j < n; ++j) {
        const int cin = j == 0 ? 2 * n * ci : (2 * (n - j) + 1) * ci;
        const int cprev = j == 0 ? n * ci : (n - j + 1) * ci;         // channels of the previous block's output
        sh.push_back(Shape{cin, (n - j) * ci, 5, T >> (n - 1 - j), SRC_UPCAT, cprev, cin - cprev});
    }
}

struct Layout {
    std::vector<size_t> z, act, ga;      // float offsets of the pre-BN outputs, activations, activation gradients
    std::vector<size_t> mean, invstd, s1, s2;
    std::vector<size_t> wf, wb;          // the step's packed weights: forward / input-gradient operand layouts
    std::vector<size_t> wftc, wbtc;      // the tensor-core precisions only (appended after the fp32 layout): the tensor-core
                                         // packings at that precision
    size_t din, ones, zeros, total;      // ones / zeros: [kMaxC] identity scale and zero shift for the linear conv epilogue
    size_t amax;                         // TRAIN_FP16_SCALED only (after the packings): [2n+1] max |dz| of each block (0 = none)
};
constexpr int kMaxC = 2048;

// the first block (Cin = 1: a degenerate GEMM) stays on the fp32 kernels at every precision
bool on_tc(int prec, int i) { return (prec == TRAIN_BF16 || prec == TRAIN_TF32 || prec == TRAIN_FP16_SCALED) && i > 0; }

// launch geometry of block i's weight gradient at `prec`
WgradGrid wgrad_grid_of(int prec, int i, int B, int L, int cin, int cout, int k)
{
    return on_tc(prec, i) ? wgrad_grid_tc(B, L, cin, cout, k) : wgrad_grid_fp32(B, L, cin, cout);
}

void layout_of(const std::vector<Shape> &sh, int B, Layout &lo, int prec = TRAIN_FP32)
{
    const size_t nb = sh.size();
    lo.z.resize(nb); lo.act.resize(nb); lo.ga.resize(nb); lo.mean.resize(nb); lo.invstd.resize(nb); lo.s1.resize(nb); lo.s2.resize(nb); lo.wf.resize(nb); lo.wb.resize(nb);
    size_t cur = 0, din_max = 0;
    auto take = [&](size_t n) { const size_t o = cur; cur += (n + 63) / 64 * 64; return o; };
    for (size_t i = 0; i < nb; ++i) {
        const size_t n = (size_t)B * sh[i].cout * sh[i].L;
        lo.z[i] = take(n); lo.act[i] = take(n); lo.ga[i] = take(n);
        lo.mean[i] = take(sh[i].cout); lo.invstd[i] = take(sh[i].cout); lo.s1[i] = take(sh[i].cout); lo.s2[i] = take(sh[i].cout);
        lo.wf[i] = take((size_t)sh[i].cout * sh[i].cin * sh[i].k); lo.wb[i] = take((size_t)sh[i].cout * sh[i].cin * sh[i].k);
        din_max = std::max(din_max, (size_t)B * sh[i].cin * sh[i].L);
    }
    lo.din = take(din_max);
    lo.ones = take(kMaxC); lo.zeros = take(kMaxC);
    lo.wftc.assign(nb, 0); lo.wbtc.assign(nb, 0);
    for (size_t i = 0; i < nb; ++i) {
        if (!on_tc(prec, (int)i)) continue;
        lo.wftc[i] = take((train_tc_packed_bytes(prec, sh[i].cout, sh[i].cin, sh[i].k) + 3) / 4);       // float units
        lo.wbtc[i] = take((train_tc_packed_bytes(prec, sh[i].cin, sh[i].cout, sh[i].k) + 3) / 4);
    }
    lo.amax = prec == TRAIN_FP16_SCALED ? take(nb) : 0;
    lo.total = cur;
}

ConvArgs conv_args(const std::vector<Shape> &sh, const Layout &lo, float *ws, const float *x, int i, int n, int B)
{
    ConvArgs a{};
    const Shape &s = sh[i];
    a.B = B; a.L = s.L; a.Cin = s.cin; a.Cin0 = s.cin0; a.Cin1 = s.cin1; a.Cout = s.cout;
    if (s.mode == SRC_DIRECT) a.src0 = x;
    else if (s.mode == SRC_DECIM) a.src0 = ws + lo.act[i - 1];
    else {
        a.src0 = ws + lo.act[i - 1];
        a.src1 = ws + lo.act[2 * n - i];                    // skip = encoder 2n - i (model/unet_basic.py:95)
        const int Lin = s.L / 2;
        a.up_scale = s.L > 1 ? (float)(Lin - 1) / (float)(s.L - 1) : 0.f;
    }
    return a;
}

unsigned blocks_for(long long n, int per) { return (unsigned)((n + per - 1) / per); }

// TRAIN_DETERMINISTIC scratch in floats, placed at lo.total: the larger of one block's per-slice weight-gradient partials
// (gridDim.z copies of its dW; the grids depend on the shapes only) and the head's CTA partials (doubles). The blocks use it
// one after another on the stream.
size_t det_scratch_floats(const std::vector<Shape> &sh, int B, int T, int prec)
{
    const int last = (int)sh.size() - 1;
    size_t m = 2 * (size_t)blocks_for((long long)B * T, 256) * (sh[last].cout + 2);
    for (int i = 0; i <= last; ++i) {
        const Shape &s = sh[i];
        const WgradGrid g = wgrad_grid_of(prec, i, B, s.L, s.cin, s.cout, s.k);
        m = std::max(m, (size_t)g.grid.z * s.cout * s.cin * s.k);
    }
    return m;
}

// WUNET_TRAIN_NAIVE=1: the one-thread-per-output reference kernels instead of the tuned ones (cross-check)
bool train_naive()
{
    const char *e = getenv("WUNET_TRAIN_NAIVE");
    return e && e[0] == '1';
}

}  // namespace

const char *train_error() { return g_train_err; }

// CTA = 16 co x 64 ci; tiles of min(L, 128) positions of one frame, split over gridDim.z
WgradGrid wgrad_grid_fp32(int B, int L, int Cin, int Cout)
{
    const int lt = std::min(L, 128);
    const int nco = (Cout + 15) / 16, nci = (Cin + 63) / 64;
    const int ntiles = B * ((L + lt - 1) / lt);
    const int slices = std::max(1, std::min(ntiles, 1184 / (nco * nci)));           // ~4 blocks per SM over the grid
    return WgradGrid{dim3((unsigned)nco, (unsigned)nci, (unsigned)slices), ntiles, lt};
}

int train_debug_layout(int n, int ci, int B, int T, int prec, int block, long long *f, int capacity)
{
    if (block < 0 || block > 2 * n) return train_fail("layout query: block %d outside 0 .. %d", block, 2 * n);
    if (!f || capacity < kTrainLayoutFields) return train_fail("layout query: needs room for %d fields", kTrainLayoutFields);
    std::vector<Shape> sh;
    shapes_of(n, ci, T, sh);
    Layout lo;
    layout_of(sh, B, lo, prec);
    const Shape &s = sh[block];
    const bool tc = on_tc(prec, block);
    const WgradGrid g = wgrad_grid_of(prec, block, B, s.L, s.cin, s.cout, s.k);
    const long long b = sizeof(float), gz = g.grid.z;
    const long long v[kTrainLayoutFields] = {
        (long long)lo.z[block] * b, (long long)lo.act[block] * b, (long long)lo.ga[block] * b, (long long)lo.mean[block] * b,
        (long long)lo.invstd[block] * b, (long long)lo.s1[block] * b, (long long)lo.s2[block] * b,
        s.cin, s.cin0, s.cin1, s.cout, s.L, s.k, s.mode,
        tc ? prec : 0 /* the field's 1 = bf16, 2 = tf32, 3 = fp16 are TRAIN_BF16, TRAIN_TF32, TRAIN_FP16_SCALED */, g.grid.x, g.grid.y, gz, g.items, g.positions, (g.items + gz - 1) / gz, (long long)lo.total * b};
    for (int i = 0; i < kTrainLayoutFields; ++i) f[i] = v[i];
    if (capacity > kTrainLayoutFields) f[kTrainLayoutFields] = (prec == TRAIN_FP16_SCALED && tc) ? (long long)(lo.amax + block) * b : -1;
    return 0;
}

size_t train_workspace_bytes(int n, int ci, int B, int T, int prec, int flags)
{
    std::vector<Shape> sh;
    shapes_of(n, ci, T, sh);
    Layout lo;
    layout_of(sh, B, lo, prec);
    const size_t scratch = (flags & TRAIN_DETERMINISTIC) ? det_scratch_floats(sh, B, T, prec) : 0;
    return (lo.total + scratch) * sizeof(float);
}

int train_forward(int n, int ci, const float *x, float *y, int B, int T, const TrainParams &P, const float *momentum,
                  void *workspace, cudaStream_t st, int prec, int flags, const BnSync *sync, const unsigned char *bn_frozen)
{
    // block i normalises by its running statistics (eval-mode container) or by batch statistics; only the latter synchronise
    auto frozen_at = [&](int i) { return (flags & TRAIN_FROZEN_BN) || (bn_frozen && bn_frozen[i]); };
    bool any_frozen = false;
    for (int i = 0; i < 2 * n + 1; ++i) any_frozen = any_frozen || frozen_at(i);
    std::vector<Shape> sh;
    shapes_of(n, ci, T, sh);
    Layout lo;
    layout_of(sh, B, lo, prec);
    float *ws = static_cast<float *>(workspace);
    const bool naive = train_naive() && prec == TRAIN_FP32;
    // the ones / zeros vectors serve the linear conv epilogue and, as s1 = s2 = 0, the frozen-statistics BatchNorm backward
    if (sh[0].cout * (2 * n) > kMaxC && (!naive || any_frozen)) return train_fail("channel plan too wide for the training kernels (%d channels)", sh[0].cout * 2 * n);
    if (!naive || any_frozen) {
        train_fill_kernel<<<(kMaxC + 255) / 256, 256, 0, st>>>(ws + lo.ones, 1.f, kMaxC);
        train_fill_kernel<<<(kMaxC + 255) / 256, 256, 0, st>>>(ws + lo.zeros, 0.f, kMaxC);
    }
    for (int i = 0; i < 2 * n + 1; ++i) {
        const Shape &s = sh[i];
        ConvArgs a = conv_args(sh, lo, ws, x, i, n, B);
        float *z = ws + lo.z[i];
        const dim3 grid((unsigned)((s.L + 127) / 128), (unsigned)((s.cout + 7) / 8), (unsigned)B);
        if (on_tc(prec, i)) {
            // z = conv(round(in), round(w)) + bias on the tensor cores (fp32 accumulate); both packings for this step
            if (train_tc_pack(prec, P.conv_w[i], ws + lo.wftc[i], ws + lo.wbtc[i], s.cout, s.cin, s.k, st) < 0) return train_fail("training forward, block %d: tensor-core pack failed", i);
            a.wp = ws + lo.wftc[i]; a.scale = ws + lo.ones; a.shift = P.conv_b[i]; a.out = z; a.linear = 1;
            if (launch_train_conv_tc(prec, a, s.k, s.mode, st) < 0) return train_fail("training forward, block %d: tensor-core conv launch failed", i);
        } else if (!naive) {
            // z = conv(in, w) + bias through the tuned fp32 conv kernels: identity scale, shift = conv bias, no activation
            const long long nw = (long long)s.cout * s.cin * s.k;
            train_pack_kernel<<<blocks_for(nw, 256), 256, 0, st>>>(P.conv_w[i], ws + lo.wf[i], ws + lo.wb[i], s.cout, s.cin, s.k);
            a.wp = ws + lo.wf[i]; a.scale = ws + lo.ones; a.shift = P.conv_b[i]; a.out = z; a.linear = 1;
            if (launch_conv_fp32(a, s.k, s.mode, st) < 0) return train_fail("training forward, block %d: conv launch failed", i);
        } else if (s.mode == SRC_DIRECT) train_conv_fwd_kernel<15, SRC_DIRECT><<<grid, 128, 0, st>>>(a, P.conv_w[i], P.conv_b[i], z);
        else if (s.mode == SRC_DECIM) train_conv_fwd_kernel<15, SRC_DECIM><<<grid, 128, 0, st>>>(a, P.conv_w[i], P.conv_b[i], z);
        else train_conv_fwd_kernel<5, SRC_UPCAT><<<grid, 128, 0, st>>>(a, P.conv_w[i], P.conv_b[i], z);
        if (frozen_at(i))
            train_bn_frozen_stats_kernel<<<blocks_for(s.cout, 256), 256, 0, st>>>(P.bn_mean[i], P.bn_var[i], ws + lo.mean[i],
                                                                                   ws + lo.invstd[i], s.cout);
        else if (sync) {
            double *buf = sync->buf;
            train_bn_sync_sum_kernel<<<(unsigned)s.cout, 256, 0, st>>>(z, B, s.cout, s.L, buf);
            if (const int rc = sync->fn(sync->user, buf, (size_t)s.cout + 1, st))
                return train_fail("training forward, block %d: the BatchNorm all-reduce hook failed on the sums (status %d)", i, rc);
            train_bn_sync_centred_kernel<<<(unsigned)s.cout, 256, 0, st>>>(z, B, s.cout, s.L, buf);
            if (const int rc = sync->fn(sync->user, buf + s.cout + 1, (size_t)s.cout, st))
                return train_fail("training forward, block %d: the BatchNorm all-reduce hook failed on the variances (status %d)", i, rc);
            train_bn_sync_finalize_kernel<<<blocks_for(s.cout, 256), 256, 0, st>>>(buf, s.cout, momentum[i], ws + lo.mean[i],
                                                                                    ws + lo.invstd[i], P.bn_mean[i], P.bn_var[i]);
        } else
            train_bn_stats_kernel<<<(unsigned)s.cout, 256, 0, st>>>(z, B, s.cout, s.L, momentum[i], ws + lo.mean[i], ws + lo.invstd[i],
                                                                     P.bn_mean[i], P.bn_var[i]);
        const long long nel = (long long)B * s.cout * s.L;
        train_bn_act_kernel<<<blocks_for(nel, 256), 256, 0, st>>>(z, ws + lo.mean[i], ws + lo.invstd[i], P.bn_w[i], P.bn_b[i],
                                                                  ws + lo.act[i], B, s.cout, s.L);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return train_fail("training forward, block %d: %s", i, cudaGetErrorString(e));
    }
    if (launch_out_fp32(ws + lo.act[2 * n], x, P.out_w, P.out_b, y, B, sh[2 * n].cout, T, st) < 0)
        return train_fail("training forward, head: %s", cudaGetErrorString(cudaGetLastError()));
    return 0;
}

int train_backward(int n, int ci, const float *x, const float *y, const float *dy, int B, int T, const TrainParams &P,
                   const TrainGrads &G, void *workspace, cudaStream_t st, int part, int prec, float *dx, int flags,
                   const BnSync *sync, const unsigned char *bn_frozen, bool early_stop, const float *const *g_act)
{
    std::vector<Shape> sh;
    shapes_of(n, ci, T, sh);
    Layout lo;
    layout_of(sh, B, lo, prec);
    float *ws = static_cast<float *>(workspace);
    const int last = 2 * n, C = sh[last].cout;
    const bool naive = train_naive() && prec == TRAIN_FP32;
    const bool pgrads = !(flags & TRAIN_NO_PARAM_GRADS);
    auto frozen_at = [&](int i) { return (flags & TRAIN_FROZEN_BN) || (bn_frozen && bn_frozen[i]); };
    // the gradient slots this call fills: a null array or entry is a frozen parameter (nothing computed, nothing written)
    auto slot = [&](float *const *g, int i) { return pgrads && g ? g[i] : nullptr; };
    float *const g_wo = pgrads ? G.out_w : nullptr, *const g_bo = pgrads ? G.out_b : nullptr;
    auto block_wants = [&](int i) { return slot(G.conv_w, i) || slot(G.conv_b, i) || slot(G.bn_w, i) || slot(G.bn_b, i); };
    // early stop: j = the lowest block (the last in backward order) that still needs something — a parameter gradient or,
    // through block 0, dx. Block j skips its input gradient; blocks below j issue nothing. Without early_stop every block runs
    // (the _ex entry points: their split backward's part 0 cannot know whether part 1 will ask for dx).
    int j = 0;
    if (early_stop && !dx) {
        j = last + 1;
        for (int i = 0; i <= last && j > last; ++i)
            if (block_wants(i)) j = i;
    }
    bool any_grad = g_wo || g_bo;
    for (int i = 0; i <= last; ++i) any_grad = any_grad || block_wants(i);
    const bool det = any_grad && (flags & TRAIN_DETERMINISTIC);    // without parameter gradients nothing is summed atomically
    float *scratch = ws + lo.total;                                 // TRAIN_DETERMINISTIC only (det_scratch_floats)
    if (part < -1 || part > 1) return train_fail("training backward: part must be -1, 0 or 1 (got %d)", part);
    if (dx && part == 0 && !early_stop) return train_fail("training backward: dx is written by part 1 (or -1), not part 0");
    if (det && naive) return train_fail("training backward: WUNET_TRAIN_NAIVE=1 has no deterministic weight gradient");
    if (part != 1 && (g_wo || g_bo || j <= last)) {
        const unsigned hb = blocks_for((long long)B * T, 256);
        // one head parameter frozen, the other not: the kernel computes both, the frozen one into the (idle) din region
        float *hw = g_wo ? g_wo : ws + lo.din, *hbias = g_bo ? g_bo : ws + lo.din;
        if (det && (g_wo || g_bo)) {
            double *hp = reinterpret_cast<double *>(scratch);
            train_head_bwd_kernel<true><<<hb, 256, 0, st>>>(dy, y, ws + lo.act[last], x, P.out_w, ws + lo.ga[last], hw, hbias, hp,
                                                            B, C, T);
            train_head_sum_kernel<<<(unsigned)(C + 2), 256, 0, st>>>(hp, (int)hb, C, hw, hbias);
        } else {
            if (g_wo || g_bo) {
                cudaMemsetAsync(hw, 0, (C + 1) * sizeof(float), st);
                cudaMemsetAsync(hbias, 0, sizeof(float), st);
            }
            train_head_bwd_kernel<false><<<hb, 256, 0, st>>>(dy, y, ws + lo.act[last], x, P.out_w, ws + lo.ga[last],
                                                             (g_wo || g_bo) ? hw : nullptr, hbias, nullptr, B, C, T);
        }
    }
    const int i_hi = (part == 1) ? n : last, i_lo = std::max((part == 0) ? n + 1 : 0, j);
    const bool scaled = prec == TRAIN_FP16_SCALED;
    if (scaled && i_hi >= i_lo) cudaMemsetAsync(ws + lo.amax + i_lo, 0, (size_t)(i_hi - i_lo + 1) * sizeof(float), st);
    for (int i = i_hi; i >= i_lo; --i) {
        const Shape &s = sh[i];
        float *ga = ws + lo.ga[i];                               // gradient of the activation; becomes dz in place
        const float *z = ws + lo.z[i];
        const long long nel = (long long)B * s.cout * s.L;
        float *g_gamma = slot(G.bn_w, i), *g_beta = slot(G.bn_b, i), *g_cb = slot(G.conv_b, i), *g_cw = slot(G.conv_w, i);
        const bool frozen = frozen_at(i);
        // a forward hook's upstream gradient of this block's output: ga is complete here (head or upsample adjoint, skip and
        // decimation adjoints), so the sum is the same whatever the launch order of the others
        if (g_act && g_act[i] && launch_grad_inject(ga, g_act[i], nel, st) < 0)
            return train_fail("training backward, block %d: gradient injection launch failed", i);
        // batch statistics: dz needs mean(dy) and mean(dy zh) (s1, s2); frozen statistics: they are constants, dz = invstd
        // gamma dy (s1 = s2 = 0), and the reductions only serve the BatchNorm parameter gradients
        if (sync && !frozen) {
            train_bn_sync_bwd_sums_kernel<<<(unsigned)s.cout, 256, 0, st>>>(ga, z, ws + lo.mean[i], ws + lo.invstd[i], P.bn_w[i],
                                                                             P.bn_b[i], g_gamma, g_beta, sync->buf, B, s.cout, s.L);
            if (const int rc = sync->fn(sync->user, sync->buf, 2 * (size_t)s.cout + 1, st))
                return train_fail("training backward, block %d: the BatchNorm all-reduce hook failed (status %d)", i, rc);
            train_bn_sync_bwd_finalize_kernel<<<blocks_for(s.cout, 256), 256, 0, st>>>(sync->buf, s.cout, ws + lo.s1[i], ws + lo.s2[i]);
        } else if (!frozen || g_gamma || g_beta)
            train_bn_bwd_stats_kernel<<<(unsigned)s.cout, 256, 0, st>>>(ga, z, ws + lo.mean[i], ws + lo.invstd[i], P.bn_w[i], P.bn_b[i],
                                                                         g_gamma, g_beta, ws + lo.s1[i], ws + lo.s2[i], B, s.cout, s.L);
        const float *s1 = frozen ? ws + lo.zeros : ws + lo.s1[i], *s2 = frozen ? ws + lo.zeros : ws + lo.s2[i];
        // the scaled passes of this block read its max |dz| (wunet_train_tc_kernels.cuh)
        float *amax = scaled && on_tc(prec, i) ? ws + lo.amax + i : nullptr;
        if (amax)
            train_bn_bwd_apply_amax_kernel<<<std::min(blocks_for(nel, 256), (unsigned)kAmaxCtas), 256, 0, st>>>(
                ga, z, ws + lo.mean[i], ws + lo.invstd[i], P.bn_w[i], P.bn_b[i], s1, s2, B, s.cout, s.L, amax);
        else
            train_bn_bwd_apply_kernel<<<blocks_for(nel, 256), 256, 0, st>>>(ga, z, ws + lo.mean[i], ws + lo.invstd[i], P.bn_w[i],
                                                                            P.bn_b[i], s1, s2, B, s.cout, s.L);
        ConvArgs a = conv_args(sh, lo, ws, x, i, n, B);
        if (g_cb) train_channel_sum_kernel<<<(unsigned)s.cout, 256, 0, st>>>(ga, g_cb, B, s.cout, s.L);
        if (g_cw) {
            // weight gradient: gridDim.z slices combined with atomicAdd into the zeroed dW or, in deterministic mode, stored to
            // the scratch and summed in slice order
            const long long nw = (long long)s.cout * s.cin * s.k;
            float *wdst = det ? scratch : g_cw;
            if (!det) cudaMemsetAsync(g_cw, 0, (size_t)nw * sizeof(float), st);
            const dim3 gw((unsigned)s.cout, (unsigned)((s.cin + 3) / 4), (unsigned)std::min(B, 8));
            if (on_tc(prec, i)) {
                a.scale = amax;                                          // the weight gradient has no epilogue
                if (launch_train_wgrad_tc(prec, a, ga, wdst, s.k, s.mode, st, det) < 0) return train_fail("training backward, block %d: tensor-core weight-gradient launch failed", i);
            } else if (!naive) {
                launch_wgrad_fp32(a, ga, wdst, s.mode, st, det);
            } else if (s.mode == SRC_DIRECT) train_conv_bwd_weight_kernel<15, SRC_DIRECT><<<gw, 128, 0, st>>>(a, ga, g_cw);
            else if (s.mode == SRC_DECIM) train_conv_bwd_weight_kernel<15, SRC_DECIM><<<gw, 128, 0, st>>>(a, ga, g_cw);
            else train_conv_bwd_weight_kernel<5, SRC_UPCAT><<<gw, 128, 0, st>>>(a, ga, g_cw);
            if (det) {
                const WgradGrid g = wgrad_grid_of(prec, i, B, s.L, s.cin, s.cout, s.k);
                train_slice_sum_kernel<<<blocks_for(nw, 256), 256, 0, st>>>(scratch, g_cw, (int)g.grid.z, nw);
            }
        }
        // input gradient and its routing to the producers of the block input (none below block j needs it)
        if (s.mode != SRC_DIRECT && i > j) {
            float *din = ws + lo.din;
            const dim3 gd((unsigned)((s.L + 127) / 128), (unsigned)((s.cin + 7) / 8), (unsigned)B);
            if (!naive) {
                // din = conv(dz, transposed + flipped weights): the forward conv kernels with dz as a plain [B][Cout][L] input
                ConvArgs d{};
                d.src0 = ga; d.wp = ws + lo.wb[i]; d.scale = ws + lo.ones; d.shift = ws + lo.zeros; d.out = din;
                d.B = B; d.L = s.L; d.Cin = s.cout; d.Cin0 = s.cout; d.Cin1 = 0; d.Cout = s.cin; d.linear = 1;
                if (on_tc(prec, i)) {
                    d.wp = ws + lo.wbtc[i];                                     // the packing the forward wrote
                    d.src1 = amax;                                              // (DIRECT mode reads no skip input)
                    if (launch_train_conv_tc(prec, d, s.k, SRC_DIRECT, st) < 0) return train_fail("training backward, block %d: tensor-core input-gradient launch failed", i);
                } else if (launch_conv_fp32(d, s.k, SRC_DIRECT, st) < 0) return train_fail("training backward, block %d: input-gradient conv launch failed", i);
            } else if (s.k == 15) train_conv_bwd_data_kernel<15><<<gd, 128, 0, st>>>(ga, P.conv_w[i], din, B, s.cin, s.cout, s.L);
            else train_conv_bwd_data_kernel<5><<<gd, 128, 0, st>>>(ga, P.conv_w[i], din, B, s.cin, s.cout, s.L);
            if (s.mode == SRC_DECIM) {
                // encoder i >= 1 or the middle block: its input is act[i-1][:, :, ::2]; ga[i-1] already holds the skip gradient
                train_decim_adjoint_kernel<<<blocks_for((long long)B * s.cin * s.L, 256), 256, 0, st>>>(din, ws + lo.ga[i - 1], B, s.cin, s.L);
            } else {
                const int e = 2 * n - i;
                if (e >= j)
                    train_skip_grad_kernel<<<blocks_for((long long)B * s.cin1 * s.L, 256), 256, 0, st>>>(din, ws + lo.ga[e], B, s.cin,
                                                                                                         s.cin0, s.L);
                train_upsample_adjoint_kernel<<<blocks_for((long long)B * s.cin0 * (s.L / 2), 256), 256, 0, st>>>(
                    din, ws + lo.ga[i - 1], B, s.cin, s.cin0, s.L, a.up_scale);
            }
        }
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return train_fail("training backward, block %d: %s", i, cudaGetErrorString(e));
    }
    if (dx && part != 0) {
        // part -1 or 1: ga[0] now holds block 0's dz
        const dim3 gx(blocks_for(T, 256), (unsigned)B);
        train_input_grad_kernel<15><<<gx, 256, 0, st>>>(ws + lo.ga[0], P.conv_w[0], dy, y, P.out_w, dx, sh[0].cout, C, T);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return train_fail("training backward, input gradient: %s", cudaGetErrorString(e));
    }
    return 0;
}

int train_debug_conv(int pass, int prec, int mode, int ksize, int B, int L, int Cin0, int Cin1, int Cout, const float *src0,
                     const float *src1, const float *w, const float *dz, float *out)
{
    const bool ok_mode = (ksize == 15 && (mode == SRC_DIRECT || mode == SRC_DECIM)) || (ksize == 5 && mode == SRC_UPCAT) ||
                         (ksize == 5 && mode == SRC_DIRECT && pass == 1);
    if (pass < 0 || pass > 2 || (prec != TRAIN_FP32 && prec != TRAIN_BF16 && prec != TRAIN_TF32 && prec != TRAIN_FP16_SCALED) || !ok_mode || B < 1 || L < 1 || Cin0 < 1 ||
        Cin1 < 0 || Cout < 1 || (mode != SRC_UPCAT && Cin1 != 0) || (mode == SRC_UPCAT && (L < 2 || L % 2 != 0 || Cin1 < 1)) ||
        !w || !out || (pass != 1 && !src0) || (pass != 1 && mode == SRC_UPCAT && !src1) || (pass != 0 && !dz))
        return train_fail("debug conv: bad arguments");
    const int Cin = Cin0 + Cin1, K = ksize, cmax = std::max(Cin, Cout);
    ConvArgs a{};
    a.src0 = src0; a.src1 = src1; a.B = B; a.L = L; a.Cin = Cin; a.Cin0 = mode == SRC_UPCAT ? Cin0 : Cin; a.Cin1 = Cin1; a.Cout = Cout;
    a.up_scale = (mode == SRC_UPCAT && L > 1) ? (float)(L / 2 - 1) / (float)(L - 1) : 0.f;
    float *buf = nullptr;
    const size_t nw = (size_t)Cout * Cin * K, cpad = (cmax + 63) / 64 * 64, wpad = (nw + 63) / 64 * 64;      // 256-byte aligned parts
    const bool tc = prec != TRAIN_FP32;
    const size_t ntcf = tc ? train_tc_packed_bytes(prec, Cout, Cin, K) / sizeof(float) : 0;     // float units
    const size_t ntc = tc ? ntcf + train_tc_packed_bytes(prec, Cin, Cout, K) / sizeof(float) : 0;
    if (cudaMalloc(&buf, (2 * cpad + 2 * wpad + ntc + 64) * sizeof(float)) != cudaSuccess)
        return train_fail("debug conv: %s", cudaGetErrorString(cudaGetLastError()));
    float *ones = buf, *zeros = buf + cpad, *wf = zeros + cpad, *wb = wf + wpad, *wtc_f = wb + wpad, *wtc_b = wtc_f + ntcf;
    const cudaStream_t st = 0;
    train_fill_kernel<<<(cmax + 255) / 256, 256, 0, st>>>(ones, 1.f, cmax);
    train_fill_kernel<<<(cmax + 255) / 256, 256, 0, st>>>(zeros, 0.f, cmax);
    // TRAIN_FP16_SCALED: the passes that read dz scale it by 2^k of its max |dz|, as the step does per block
    float *amax = prec == TRAIN_FP16_SCALED && pass != 0 ? wtc_f + ntc : nullptr;
    if (amax) {
        const long long ndz = (long long)B * Cout * L;
        cudaMemsetAsync(amax, 0, sizeof(float), st);
        train_amax_kernel<<<std::min(blocks_for(ndz, 256), (unsigned)kAmaxCtas), 256, 0, st>>>(dz, ndz, amax);
    }
    if (mode != SRC_UPCAT) a.src1 = nullptr;                  // no skip input (and no scale: the forward conv is unscaled)
    int rc = 0;
    if (pass == 2) {
        cudaMemsetAsync(out, 0, nw * sizeof(float), st);
        a.scale = amax;
        if (tc) rc = launch_train_wgrad_tc(prec, a, dz, out, K, mode, st, false);
        else launch_wgrad_fp32(a, dz, out, mode, st);
    } else {
        if (tc) rc = train_tc_pack(prec, w, wtc_f, wtc_b, Cout, Cin, K, st);
        else train_pack_kernel<<<blocks_for((long long)nw, 256), 256, 0, st>>>(w, wf, wb, Cout, Cin, K);
        if (pass == 0) {
            a.wp = tc ? wtc_f : wf; a.scale = ones; a.shift = zeros; a.out = out; a.linear = 1;
            if (rc >= 0) rc = tc ? launch_train_conv_tc(prec, a, K, mode, st) : launch_conv_fp32(a, K, mode, st);
        } else {
            ConvArgs d{};
            d.src0 = dz; d.src1 = amax; d.wp = tc ? wtc_b : wb; d.scale = ones; d.shift = zeros; d.out = out;
            d.B = B; d.L = L; d.Cin = Cout; d.Cin0 = Cout; d.Cin1 = 0; d.Cout = Cin; d.linear = 1;
            if (rc >= 0) rc = tc ? launch_train_conv_tc(prec, d, K, SRC_DIRECT, st) : launch_conv_fp32(d, K, SRC_DIRECT, st);
        }
    }
    const cudaError_t e = cudaDeviceSynchronize();
    cudaFree(buf);
    if (rc < 0) return train_fail("debug conv: launch failed");
    if (e != cudaSuccess) return train_fail("debug conv: %s", cudaGetErrorString(e));
    return 0;
}

}  // namespace wunet
