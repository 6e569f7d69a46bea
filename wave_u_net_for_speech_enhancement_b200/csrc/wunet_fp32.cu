// wunet_fp32.cu — exact-fp32 (FFMA) kernels of the Wave-U-Net forward: the parity anchor
// (BASELINE.json config 2: <= 1e-4 max-abs vs the reference's fp32 CPU forward).
//
// Replaces, per block, the reference's op sequence
//   [decimate o[:, :, ::2] | F.interpolate + torch.cat] -> nn.Conv1d -> nn.BatchNorm1d(eval) -> nn.LeakyReLU(0.1)
// (model/unet_basic.py:83-86, :93-96, :10-13, :23-26) with ONE kernel: the producer-side reshuffle is
// fused into the operand load (fetch_src), BatchNorm/LeakyReLU into the epilogue.
//
// Two kernels:
//   conv_slide_kernel  L >= 256: sliding-window direct convolution. A warp owns 8 output channels x
//                      256 positions (8 per lane); per input channel the lane keeps its 8+K-1 input
//                      window in registers and sweeps the K taps -> 64*K FFMA per 6 (K=15) LDS.128 of
//                      inputs + 2K broadcast LDS.128 of weights. 89 % of the network's FLOPs.
//   conv_gen_kernel    any shape: implicit GEMM over flattened (b,l) positions with an im2col gather
//                      into shared memory (handles frames shorter than a tile, L down to 1).
#include "wunet_common.cuh"

namespace wunet {

// -------------------------------------------------------------------------------------------
// sliding-window kernel
// -------------------------------------------------------------------------------------------
template <int KS, int MODE, int LW, typename IO = float>
__global__ void __launch_bounds__(96 * LW) conv_slide_kernel(const ConvArgs a)
{
    constexpr int PAD = (KS - 1) / 2;
    constexpr int CI = 8;
    constexpr int COT = 24;
    constexpr int LT = 256 * LW;
    constexpr int XW = LT + KS - 1;
    constexpr int NX = (8 + KS - 1 + 3) & ~3;          // register window, rounded to float4s
    constexpr int XWP = LT - 8 + NX;                    // last float4 over-read stays inside the row
    constexpr int NT = 96 * LW;
    static_assert(XWP >= XW, "row too short");

    __shared__ __align__(16) float Xs[CI][XWP];
    __shared__ __align__(16) float Ws[CI][KS][COT];

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const int wc = warp % 3, wl = warp / 3;
    const int lbase = wl * 256 + lane * 8;
    const int b = blockIdx.z;
    const int co0 = blockIdx.y * COT;
    const int l0 = blockIdx.x * LT;

    float acc[8][8];
#pragma unroll
    for (int m = 0; m < 8; ++m)
#pragma unroll
        for (int n = 0; n < 8; ++n) acc[m][n] = 0.f;

    // zero the over-read tail once (never used by an FFMA, but keep it finite)
    if constexpr (XWP > XW) {
        constexpr int TAIL = XWP - XW;
        for (int i = tid; i < CI * TAIL; i += NT) Xs[i / TAIL][XW + i % TAIL] = 0.f;
    }

    for (int c0 = 0; c0 < a.Cin; c0 += CI) {
        const int nci = min(CI, a.Cin - c0);
        __syncthreads();
        for (int i = tid; i < nci * XW; i += NT) {
            const int ci = i / XW, j = i - ci * XW;
            Xs[ci][j] = fetch_src<MODE, IO>(a, b, c0 + ci, l0 - PAD + j);
        }
        for (int i = tid; i < nci * KS * (COT / 4); i += NT) {
            const int row = i / (COT / 4), q = i - row * (COT / 4);      // row = ci*KS + k
            const float4 v = __ldg(reinterpret_cast<const float4 *>(a.wp + ((size_t)c0 * KS + row) * a.Cout + co0) + q);
            reinterpret_cast<float4 *>(&Ws[0][0][0] + row * COT)[q] = v;
        }
        __syncthreads();

#pragma unroll 1
        for (int ci = 0; ci < nci; ++ci) {
            float xr[NX];
#pragma unroll
            for (int q = 0; q < NX / 4; ++q) {
                const float4 v = *reinterpret_cast<const float4 *>(&Xs[ci][lbase + 4 * q]);
                xr[4 * q + 0] = v.x; xr[4 * q + 1] = v.y; xr[4 * q + 2] = v.z; xr[4 * q + 3] = v.w;
            }
#pragma unroll
            for (int k = 0; k < KS; ++k) {
                const float4 w0 = *reinterpret_cast<const float4 *>(&Ws[ci][k][wc * 8]);
                const float4 w1 = *reinterpret_cast<const float4 *>(&Ws[ci][k][wc * 8 + 4]);
                const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
                for (int m = 0; m < 8; ++m)
#pragma unroll
                    for (int n = 0; n < 8; ++n) acc[m][n] = fmaf(w[m], xr[n + k], acc[m][n]);
            }
        }
    }

    // epilogue: eval-BatchNorm scale/shift (+conv bias) and LeakyReLU(0.1), NCL fp32 store
#pragma unroll
    for (int m = 0; m < 8; ++m) {
        const int co = co0 + wc * 8 + m;
        const float s = __ldg(a.scale + co), t = __ldg(a.shift + co);
        float4 v0, v1;
        v0.x = bn_lrelu(acc[m][0], s, t, a.linear); v0.y = bn_lrelu(acc[m][1], s, t, a.linear);
        v0.z = bn_lrelu(acc[m][2], s, t, a.linear); v0.w = bn_lrelu(acc[m][3], s, t, a.linear);
        v1.x = bn_lrelu(acc[m][4], s, t, a.linear); v1.y = bn_lrelu(acc[m][5], s, t, a.linear);
        v1.z = bn_lrelu(acc[m][6], s, t, a.linear); v1.w = bn_lrelu(acc[m][7], s, t, a.linear);
        float4 *dst = reinterpret_cast<float4 *>(a.out + ((size_t)b * a.Cout + co) * a.L + l0 + lbase);
        dst[0] = v0;
        dst[1] = v1;
    }
}

// -------------------------------------------------------------------------------------------
// generic implicit-GEMM kernel (im2col gather); positions p = b*L + l flattened over the batch
// -------------------------------------------------------------------------------------------
template <int KS, int MODE, typename IO = float>
__global__ void __launch_bounds__(128) conv_gen_kernel(const ConvArgs a)
{
    constexpr int PAD = (KS - 1) / 2;
    constexpr int BM = 48, BN = 64;
    constexpr int CI = (KS == 15) ? 4 : 8;
    constexpr int KC = CI * KS;                       // 60 / 40 rows per chunk
    static_assert(KC % 2 == 0, "KC must be even");
    __shared__ __align__(16) float Xs[KC][BN];
    __shared__ __align__(16) float Ws[KC][BM];

    const int tid = threadIdx.x;
    const int tn = tid & 15, tm = tid >> 4;           // 16 x 8 threads; thread tile 6 co x 4 positions
    const int n0 = tn * 4, m0 = tm * 6;
    const int co0 = blockIdx.y * BM;
    const long long P = (long long)a.B * a.L;
    const long long p0 = (long long)blockIdx.x * BN;

    // loader role: fixed column, rows tid/64 + 2j
    const int ln = tid & 63;
    const long long lp = p0 + ln;
    const bool lvalid = lp < P;
    const int lb = lvalid ? (int)(lp / a.L) : 0;
    const int ll = lvalid ? (int)(lp - (long long)lb * a.L) : 0;

    float acc[6][4];
#pragma unroll
    for (int m = 0; m < 6; ++m)
#pragma unroll
        for (int n = 0; n < 4; ++n) acc[m][n] = 0.f;

    for (int c0 = 0; c0 < a.Cin; c0 += CI) {
        const int nci = min(CI, a.Cin - c0);
        const int nk = nci * KS;
        __syncthreads();
        for (int kk = (tid >> 6); kk < nk; kk += 2) {
            const int ci = kk / KS, k = kk - ci * KS;
            Xs[kk][ln] = lvalid ? fetch_src<MODE, IO>(a, lb, c0 + ci, ll + k - PAD) : 0.f;
        }
        for (int i = tid; i < nk * BM; i += 128) {
            const int kk = i / BM, m = i - kk * BM;
            const int co = co0 + m;
            Ws[kk][m] = (co < a.Cout) ? __ldg(a.wp + ((size_t)c0 * KS + kk) * a.Cout + co) : 0.f;
        }
        __syncthreads();
#pragma unroll 4
        for (int kk = 0; kk < nk; ++kk) {
            const float4 xv = *reinterpret_cast<const float4 *>(&Xs[kk][n0]);
            const float2 wa = *reinterpret_cast<const float2 *>(&Ws[kk][m0]);
            const float2 wb = *reinterpret_cast<const float2 *>(&Ws[kk][m0 + 2]);
            const float2 wc = *reinterpret_cast<const float2 *>(&Ws[kk][m0 + 4]);
            const float w[6] = {wa.x, wa.y, wb.x, wb.y, wc.x, wc.y};
            const float x[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
            for (int m = 0; m < 6; ++m)
#pragma unroll
                for (int n = 0; n < 4; ++n) acc[m][n] = fmaf(w[m], x[n], acc[m][n]);
        }
    }

#pragma unroll
    for (int n = 0; n < 4; ++n) {
        const long long p = p0 + n0 + n;
        if (p >= P) continue;
        const int b = (int)(p / a.L);
        const int l = (int)(p - (long long)b * a.L);
#pragma unroll
        for (int m = 0; m < 6; ++m) {
            const int co = co0 + m0 + m;
            if (co < a.Cout)
                a.out[((size_t)b * a.Cout + co) * a.L + l] = bn_lrelu(acc[m][n], __ldg(a.scale + co), __ldg(a.shift + co), a.linear);
        }
    }
}

// -------------------------------------------------------------------------------------------
// out: cat([o, input], 1) -> Conv1d(C+1 -> 1, k=1) -> Tanh      (model/unet_basic.py:98-99, :72-75); x, y: IO elements
// -------------------------------------------------------------------------------------------
template <typename IO = float>
__global__ void __launch_bounds__(256) out_kernel(const float *__restrict__ dec, const IO *__restrict__ x,
                                                  const float *__restrict__ w, const float *__restrict__ bias,
                                                  IO *__restrict__ y, int B, int C, int T)
{
    const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // float4 index over [B][T/4]
    const long long n4 = (long long)B * (T / 4);
    if (i4 >= n4) return;
    const int b = (int)(i4 / (T / 4));
    const int l = (int)(i4 - (long long)b * (T / 4)) * 4;
    const float bv = __ldg(bias);
    float4 acc = make_float4(bv, bv, bv, bv);
    for (int c = 0; c < C; ++c) {
        const float wv = __ldg(w + c);
        const float4 v = __ldg(reinterpret_cast<const float4 *>(dec + ((size_t)b * C + c) * T + l));
        acc.x = fmaf(wv, v.x, acc.x); acc.y = fmaf(wv, v.y, acc.y);
        acc.z = fmaf(wv, v.z, acc.z); acc.w = fmaf(wv, v.w, acc.w);
    }
    const float wx = __ldg(w + C);
    const float4 xv = io_ld4(x + (size_t)b * T + l);
    acc.x = tanhf(fmaf(wx, xv.x, acc.x)); acc.y = tanhf(fmaf(wx, xv.y, acc.y));
    acc.z = tanhf(fmaf(wx, xv.z, acc.z)); acc.w = tanhf(fmaf(wx, xv.w, acc.w));
    io_st4(y + (size_t)b * T + l, acc);
}

// -------------------------------------------------------------------------------------------
// weight packing: [Cout][Cin][K] -> [Cin][K][Cout]; eval BatchNorm folded to scale/shift
// -------------------------------------------------------------------------------------------
__global__ void pack_fp32_kernel(const float *__restrict__ w, const float *__restrict__ bias,
                                 const float *__restrict__ g, const float *__restrict__ beta,
                                 const float *__restrict__ mean, const float *__restrict__ var,
                                 float *__restrict__ wp, float *__restrict__ scale, float *__restrict__ shift,
                                 int Cout, int Cin, int K)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n = (long long)Cout * Cin * K;
    if (i < n) {
        const int k = (int)(i % K);
        const int ci = (int)((i / K) % Cin);
        const int co = (int)(i / ((long long)K * Cin));
        wp[((size_t)ci * K + k) * Cout + co] = w[i];
    }
    if (i < Cout) {
        // y = (conv + bias - mean) * g / sqrt(var + eps) + beta
        const float s = g[i] / sqrtf(var[i] + kBnEps);
        scale[i] = s;
        shift[i] = fmaf(bias[i] - mean[i], s, beta[i]);
    }
}

// -------------------------------------------------------------------------------------------
// launchers
// -------------------------------------------------------------------------------------------
template <int KS, int MODE, typename IO = float>
static int launch_conv_mode(const ConvArgs &a, cudaStream_t st)
{
    if (a.L % 512 == 0 && a.Cout % 24 == 0) {
        dim3 grid(a.L / 512, a.Cout / 24, a.B);
        conv_slide_kernel<KS, MODE, 2, IO><<<grid, 192, 0, st>>>(a);
    } else if (a.L % 256 == 0 && a.Cout % 24 == 0) {
        dim3 grid(a.L / 256, a.Cout / 24, a.B);
        conv_slide_kernel<KS, MODE, 1, IO><<<grid, 96, 0, st>>>(a);
    } else {
        const long long P = (long long)a.B * a.L;
        dim3 grid((unsigned)((P + 63) / 64), (a.Cout + 47) / 48, 1);
        conv_gen_kernel<KS, MODE, IO><<<grid, 128, 0, st>>>(a);
    }
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_conv_fp32_generic(const ConvArgs &a, int ksize, int mode, cudaStream_t st);

int launch_conv_fp32(const ConvArgs &a, int ksize, int mode, cudaStream_t st)
{
    if (ksize == 15) {
        if (mode == SRC_DIRECT) return launch_conv_mode<15, SRC_DIRECT>(a, st);
        if (mode == SRC_DECIM) return launch_conv_mode<15, SRC_DECIM>(a, st);
    } else if (ksize == 5) {
        if (mode == SRC_UPCAT) return launch_conv_mode<5, SRC_UPCAT>(a, st);
        if (mode == SRC_DIRECT) return launch_conv_mode<5, SRC_DIRECT>(a, st);      // training: input gradient of a decoder block
    }
    return -1;
}

// force the generic kernel (tests cross-check the two kernels against each other)
int launch_conv_fp32_generic(const ConvArgs &a, int ksize, int mode, cudaStream_t st)
{
    const long long P = (long long)a.B * a.L;
    dim3 grid((unsigned)((P + 63) / 64), (a.Cout + 47) / 48, 1);
    if (ksize == 15 && mode == SRC_DIRECT) conv_gen_kernel<15, SRC_DIRECT><<<grid, 128, 0, st>>>(a);
    else if (ksize == 15 && mode == SRC_DECIM) conv_gen_kernel<15, SRC_DECIM><<<grid, 128, 0, st>>>(a);
    else if (ksize == 5 && mode == SRC_UPCAT) conv_gen_kernel<5, SRC_UPCAT><<<grid, 128, 0, st>>>(a);
    else return -1;
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_out_fp32(const float *dec, const float *x, const float *out_w, const float *out_b, float *y, int B,
                    int C, int T, cudaStream_t st)
{
    const long long n4 = (long long)B * (T / 4);
    out_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, st>>>(dec, x, out_w, out_b, y, B, C, T);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_conv_fp32_io(const ConvArgs &a, int io, cudaStream_t st)
{
    if (io == IO_F16) return launch_conv_mode<15, SRC_DIRECT, __half>(a, st);
    if (io == IO_BF16) return launch_conv_mode<15, SRC_DIRECT, __nv_bfloat16>(a, st);
    return launch_conv_fp32(a, 15, SRC_DIRECT, st);
}

int launch_out_fp32_io(const float *dec, const void *x, const float *out_w, const float *out_b, void *y, int B, int C, int T,
                       int io, cudaStream_t st)
{
    const long long n4 = (long long)B * (T / 4);
    const unsigned grid = (unsigned)((n4 + 255) / 256);
    if (io == IO_F16)
        out_kernel<<<grid, 256, 0, st>>>(dec, static_cast<const __half *>(x), out_w, out_b, static_cast<__half *>(y), B, C, T);
    else if (io == IO_BF16)
        out_kernel<<<grid, 256, 0, st>>>(dec, static_cast<const __nv_bfloat16 *>(x), out_w, out_b, static_cast<__nv_bfloat16 *>(y), B, C, T);
    else
        return launch_out_fp32(dec, static_cast<const float *>(x), out_w, out_b, static_cast<float *>(y), B, C, T, st);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_pack_fp32(const float *w, const float *bias, const float *g, const float *beta, const float *mean,
                     const float *var, float *wp, float *scale, float *shift, int Cout, int Cin, int K,
                     cudaStream_t st)
{
    const long long n = (long long)Cout * Cin * K;
    pack_fp32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(w, bias, g, beta, mean, var, wp, scale, shift, Cout,
                                                                  Cin, K);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace wunet
