// wunet_train.cu — training step of the Wave-U-Net (SURVEY.md §8f row N1): forward with BatchNorm1d in training mode and the
// backward pass, fp32, NCL layout, CUDA cores (one formula per kernel, in the order autograd would replay them); checked
// against float64 golden steps (tests/test_train_gpu.py). The three convolution-shaped passes carry ~99 % of the work:
//   forward conv and input gradient  -> the tuned fp32 kernels of wunet_fp32.cu (sliding-window / implicit GEMM) with a linear
//                                       epilogue; the input gradient is the same convolution with the weights transposed and
//                                       flipped, read from dz (train_pack_kernel writes both packings every step);
//   weight gradient                  -> train_wgrad_kernel below (register-tiled reduction over (batch, position) tiles staged in
//                                       shared memory, split over the batch, combined with atomicAdd).
// The naive one-thread-per-output kernels they replace are kept as WUNET_TRAIN_NAIVE=1 (cross-check, tests).
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
__global__ void __launch_bounds__(256) train_head_bwd_kernel(const float *__restrict__ dy, const float *__restrict__ y,
                                                             const float *__restrict__ a_last, const float *__restrict__ x,
                                                             const float *__restrict__ wo, float *__restrict__ ga_last,
                                                             float *__restrict__ g_wo, float *__restrict__ g_bo, int B, int C, int T)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;      // over [B][T]
    const bool ok = i < (long long)B * T;
    const int b = ok ? (int)(i / T) : 0, l = ok ? (int)(i - (long long)b * T) : 0;
    const float yv = ok ? y[i] : 0.f;
    const float dpre = ok ? dy[i] * (1.f - yv * yv) : 0.f;
    for (int c = 0; c <= C; ++c) {
        float v;
        if (c < C) {
            const size_t idx = ((size_t)b * C + c) * T + l;
            v = ok ? dpre * a_last[idx] : 0.f;
            if (ok) ga_last[idx] = wo[c] * dpre;
        } else {
            v = ok ? dpre * x[i] : 0.f;
        }
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) atomicAdd(g_wo + c, v);
    }
    float v = dpre;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(g_bo, v);
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
        g_beta[c] = (float)t1;
        g_gamma[c] = (float)t2;
        s1[c] = (float)(t1 / (double)n);                        // mean(dy), mean(dy zh): what the input gradient needs
        s2[c] = (float)(t2 / (double)n);
    }
}

//   dz = invstd gamma (dy - mean(dy) - zh mean(dy zh))      written over ga (in place)
__global__ void train_bn_bwd_apply_kernel(float *__restrict__ ga, const float *__restrict__ z, const float *__restrict__ mean,
                                          const float *__restrict__ invstd, const float *__restrict__ gamma,
                                          const float *__restrict__ beta, const float *__restrict__ s1,
                                          const float *__restrict__ s2, int B, int C, int L)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * C * L) return;
    const int c = (int)((i / L) % C);
    const float zh = (z[i] - mean[c]) * invstd[c];
    const float yv = fmaf(gamma[c], zh, beta[c]);
    const float dyv = yv >= 0.f ? ga[i] : kLreluSlope * ga[i];
    ga[i] = invstd[c] * gamma[c] * (dyv - s1[c] - zh * s2[c]);
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
// the slices are combined with atomicAdd (dW is zeroed first).
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
// with atomicAdd (dW is zeroed first).
template <int KS, int MODE>
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
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int co = co0 + 2 * warp + i, ci = ci0 + lane + 32 * j;
            if (co < a.Cout && ci < a.Cin) {
#pragma unroll
                for (int k = 0; k < KS; ++k) atomicAdd(dw + ((size_t)co * a.Cin + ci) * KS + k, acc[i][j][k]);
            }
        }
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
    size_t din, ones, zeros, total;      // ones / zeros: [kMaxC] identity scale and zero shift for the linear conv epilogue
};
constexpr int kMaxC = 2048;

void layout_of(const std::vector<Shape> &sh, int B, Layout &lo)
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

// WUNET_TRAIN_NAIVE=1: the one-thread-per-output reference kernels instead of the tuned ones (cross-check)
bool train_naive()
{
    const char *e = getenv("WUNET_TRAIN_NAIVE");
    return e && e[0] == '1';
}

}  // namespace

const char *train_error() { return g_train_err; }

size_t train_workspace_bytes(int n, int ci, int B, int T)
{
    std::vector<Shape> sh;
    shapes_of(n, ci, T, sh);
    Layout lo;
    layout_of(sh, B, lo);
    return lo.total * sizeof(float);
}

int train_forward(int n, int ci, const float *x, float *y, int B, int T, const TrainParams &P, float momentum, void *workspace,
                  cudaStream_t st)
{
    std::vector<Shape> sh;
    shapes_of(n, ci, T, sh);
    Layout lo;
    layout_of(sh, B, lo);
    float *ws = static_cast<float *>(workspace);
    const bool naive = train_naive();
    if (sh[0].cout * (2 * n) > kMaxC && !naive) return train_fail("channel plan too wide for the training kernels (%d channels)", sh[0].cout * 2 * n);
    if (!naive) {
        train_fill_kernel<<<(kMaxC + 255) / 256, 256, 0, st>>>(ws + lo.ones, 1.f, kMaxC);
        train_fill_kernel<<<(kMaxC + 255) / 256, 256, 0, st>>>(ws + lo.zeros, 0.f, kMaxC);
    }
    for (int i = 0; i < 2 * n + 1; ++i) {
        const Shape &s = sh[i];
        ConvArgs a = conv_args(sh, lo, ws, x, i, n, B);
        float *z = ws + lo.z[i];
        const dim3 grid((unsigned)((s.L + 127) / 128), (unsigned)((s.cout + 7) / 8), (unsigned)B);
        if (!naive) {
            // z = conv(in, w) + bias through the tuned fp32 conv kernels: identity scale, shift = conv bias, no activation
            const long long nw = (long long)s.cout * s.cin * s.k;
            train_pack_kernel<<<blocks_for(nw, 256), 256, 0, st>>>(P.conv_w[i], ws + lo.wf[i], ws + lo.wb[i], s.cout, s.cin, s.k);
            a.wp = ws + lo.wf[i]; a.scale = ws + lo.ones; a.shift = P.conv_b[i]; a.out = z; a.linear = 1;
            if (launch_conv_fp32(a, s.k, s.mode, st) < 0) return train_fail("training forward, block %d: conv launch failed", i);
        } else if (s.mode == SRC_DIRECT) train_conv_fwd_kernel<15, SRC_DIRECT><<<grid, 128, 0, st>>>(a, P.conv_w[i], P.conv_b[i], z);
        else if (s.mode == SRC_DECIM) train_conv_fwd_kernel<15, SRC_DECIM><<<grid, 128, 0, st>>>(a, P.conv_w[i], P.conv_b[i], z);
        else train_conv_fwd_kernel<5, SRC_UPCAT><<<grid, 128, 0, st>>>(a, P.conv_w[i], P.conv_b[i], z);
        train_bn_stats_kernel<<<(unsigned)s.cout, 256, 0, st>>>(z, B, s.cout, s.L, momentum, ws + lo.mean[i], ws + lo.invstd[i],
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
                   const TrainGrads &G, void *workspace, cudaStream_t st, int part)
{
    std::vector<Shape> sh;
    shapes_of(n, ci, T, sh);
    Layout lo;
    layout_of(sh, B, lo);
    float *ws = static_cast<float *>(workspace);
    const int last = 2 * n, C = sh[last].cout;
    const bool naive = train_naive();
    if (part < -1 || part > 1) return train_fail("training backward: part must be -1, 0 or 1 (got %d)", part);
    if (part != 1) {
        cudaMemsetAsync(G.out_w, 0, (C + 1) * sizeof(float), st);
        cudaMemsetAsync(G.out_b, 0, sizeof(float), st);
        train_head_bwd_kernel<<<blocks_for((long long)B * T, 256), 256, 0, st>>>(dy, y, ws + lo.act[last], x, P.out_w, ws + lo.ga[last],
                                                                                 G.out_w, G.out_b, B, C, T);
    }
    const int i_hi = (part == 1) ? n : last, i_lo = (part == 0) ? n + 1 : 0;
    for (int i = i_hi; i >= i_lo; --i) {
        const Shape &s = sh[i];
        float *ga = ws + lo.ga[i];                               // gradient of the activation; becomes dz in place
        const float *z = ws + lo.z[i];
        const long long nel = (long long)B * s.cout * s.L;
        train_bn_bwd_stats_kernel<<<(unsigned)s.cout, 256, 0, st>>>(ga, z, ws + lo.mean[i], ws + lo.invstd[i], P.bn_w[i], P.bn_b[i],
                                                                     G.bn_w[i], G.bn_b[i], ws + lo.s1[i], ws + lo.s2[i], B, s.cout, s.L);
        train_bn_bwd_apply_kernel<<<blocks_for(nel, 256), 256, 0, st>>>(ga, z, ws + lo.mean[i], ws + lo.invstd[i], P.bn_w[i], P.bn_b[i],
                                                                        ws + lo.s1[i], ws + lo.s2[i], B, s.cout, s.L);
        train_channel_sum_kernel<<<(unsigned)s.cout, 256, 0, st>>>(ga, G.conv_b[i], B, s.cout, s.L);
        // weight gradient
        const ConvArgs a = conv_args(sh, lo, ws, x, i, n, B);
        cudaMemsetAsync(G.conv_w[i], 0, (size_t)s.cout * s.cin * s.k * sizeof(float), st);
        const dim3 gw((unsigned)s.cout, (unsigned)((s.cin + 3) / 4), (unsigned)std::min(B, 8));
        if (!naive) {
            const int lt = std::min(s.L, 128);
            const int nco = (s.cout + 15) / 16, nci = (s.cin + 63) / 64;
            const int ntiles = B * ((s.L + lt - 1) / lt);
            const int slices = std::max(1, std::min(ntiles, 1184 / (nco * nci)));           // ~4 blocks per SM over the grid
            const dim3 gt((unsigned)nco, (unsigned)nci, (unsigned)slices);
            if (s.mode == SRC_DIRECT) train_wgrad_kernel<15, SRC_DIRECT><<<gt, 256, 0, st>>>(a, ga, G.conv_w[i], lt);
            else if (s.mode == SRC_DECIM) train_wgrad_kernel<15, SRC_DECIM><<<gt, 256, 0, st>>>(a, ga, G.conv_w[i], lt);
            else train_wgrad_kernel<5, SRC_UPCAT><<<gt, 256, 0, st>>>(a, ga, G.conv_w[i], lt);
        } else if (s.mode == SRC_DIRECT) train_conv_bwd_weight_kernel<15, SRC_DIRECT><<<gw, 128, 0, st>>>(a, ga, G.conv_w[i]);
        else if (s.mode == SRC_DECIM) train_conv_bwd_weight_kernel<15, SRC_DECIM><<<gw, 128, 0, st>>>(a, ga, G.conv_w[i]);
        else train_conv_bwd_weight_kernel<5, SRC_UPCAT><<<gw, 128, 0, st>>>(a, ga, G.conv_w[i]);
        // input gradient and its routing to the producers of the block input
        if (s.mode != SRC_DIRECT) {
            float *din = ws + lo.din;
            const dim3 gd((unsigned)((s.L + 127) / 128), (unsigned)((s.cin + 7) / 8), (unsigned)B);
            if (!naive) {
                // din = conv(dz, transposed + flipped weights): the forward conv kernels with dz as a plain [B][Cout][L] input
                ConvArgs d{};
                d.src0 = ga; d.wp = ws + lo.wb[i]; d.scale = ws + lo.ones; d.shift = ws + lo.zeros; d.out = din;
                d.B = B; d.L = s.L; d.Cin = s.cout; d.Cin0 = s.cout; d.Cin1 = 0; d.Cout = s.cin; d.linear = 1;
                if (launch_conv_fp32(d, s.k, SRC_DIRECT, st) < 0) return train_fail("training backward, block %d: input-gradient conv launch failed", i);
            } else if (s.k == 15) train_conv_bwd_data_kernel<15><<<gd, 128, 0, st>>>(ga, P.conv_w[i], din, B, s.cin, s.cout, s.L);
            else train_conv_bwd_data_kernel<5><<<gd, 128, 0, st>>>(ga, P.conv_w[i], din, B, s.cin, s.cout, s.L);
            if (s.mode == SRC_DECIM) {
                // encoder i >= 1 or the middle block: its input is act[i-1][:, :, ::2]; ga[i-1] already holds the skip gradient
                train_decim_adjoint_kernel<<<blocks_for((long long)B * s.cin * s.L, 256), 256, 0, st>>>(din, ws + lo.ga[i - 1], B, s.cin, s.L);
            } else {
                const int e = 2 * n - i;
                train_skip_grad_kernel<<<blocks_for((long long)B * s.cin1 * s.L, 256), 256, 0, st>>>(din, ws + lo.ga[e], B, s.cin, s.cin0, s.L);
                train_upsample_adjoint_kernel<<<blocks_for((long long)B * s.cin0 * (s.L / 2), 256), 256, 0, st>>>(
                    din, ws + lo.ga[i - 1], B, s.cin, s.cin0, s.L, a.up_scale);
            }
        }
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return train_fail("training backward, block %d: %s", i, cudaGetErrorString(e));
    }
    return 0;
}

}  // namespace wunet
