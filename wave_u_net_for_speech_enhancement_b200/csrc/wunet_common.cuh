// wunet_common.cuh — shared host/device declarations of the H100 Wave-U-Net forward library.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stddef.h>

namespace wunet {

constexpr float kBnEps = 1e-5f;       // torch.nn.BatchNorm1d default; reference model/unet_basic.py:12,25,55
constexpr float kLreluSlope = 0.1f;   // reference model/unet_basic.py:13,26,56

// Where a conv block reads its input from (what the reference does between two Conv1d calls).
enum SrcMode : int {
    SRC_DIRECT = 0,   // x[b][ci][l]                                   (enc0: the raw input)
    SRC_DECIM = 1,    // prev[b][ci][2l]            o = o[:, :, ::2]   (model/unet_basic.py:86)
    SRC_UPCAT = 2,    // cat([interp2x(prev), skip], dim=1)            (model/unet_basic.py:93-95)
};

// One conv + eval-BN + LeakyReLU block on the fp32 path. All activations NCL fp32 (reference layout).
struct ConvArgs {
    const float *src0;   // DIRECT: [B][Cin][L]; DECIM: [B][Cin][2L]; UPCAT: prev [B][Cin0][L/2]
    const float *src1;   // UPCAT: skip [B][Cin1][L]
    const float *wp;     // packed weights [Cin][K][Cout]  (Cout contiguous)
    const float *scale;  // [Cout]  gamma / sqrt(var + eps)
    const float *shift;  // [Cout]  beta - mean*scale + bias*scale
    float *out;          // [B][Cout][L]
    int B, L;            // L = output length of this block
    int Cin, Cin0, Cin1; // Cin = Cin0 + Cin1 (Cin1 = 0 unless UPCAT)
    int Cout;
    float up_scale;      // UPCAT: (L/2 - 1) / (L - 1) in fp32, like ATen's area_pixel_compute_scale
    int linear;          // 0: LeakyReLU(0.1) epilogue (the forward blocks); 1: out = acc * scale + shift (training: pre-BatchNorm
                         // conv output, input gradients)
};

// x -> NCL element fetch with zero padding outside [0, L)  (Conv1d padding, per frame)
template <int MODE>
__device__ __forceinline__ float fetch_src(const ConvArgs &a, int b, int ci, int l)
{
    if (l < 0 || l >= a.L) return 0.f;
    if (MODE == SRC_DIRECT) {
        return __ldg(a.src0 + ((size_t)b * a.Cin + ci) * a.L + l);
    } else if (MODE == SRC_DECIM) {
        return __ldg(a.src0 + ((size_t)b * a.Cin + ci) * (2 * (size_t)a.L) + 2 * l);
    } else {
        if (ci < a.Cin0) {
            // F.interpolate(scale_factor=2, mode="linear", align_corners=True), index math in fp32
            const int Lin = a.L >> 1;
            const float s = a.up_scale * (float)l;
            const int i0 = (int)s;
            const int i1 = i0 + (i0 < Lin - 1 ? 1 : 0);
            const float lam1 = s - (float)i0;
            const float lam0 = 1.f - lam1;
            const float *p = a.src0 + ((size_t)b * a.Cin0 + ci) * Lin;
            return lam0 * __ldg(p + i0) + lam1 * __ldg(p + i1);
        } else {
            return __ldg(a.src1 + ((size_t)b * a.Cin1 + (ci - a.Cin0)) * a.L + l);
        }
    }
}

__device__ __forceinline__ float bn_lrelu(float acc, float scale, float shift, int linear = 0)
{
    const float v = fmaf(acc, scale, shift);
    return (v >= 0.f || linear) ? v : kLreluSlope * v;
}

// ---- launchers implemented in wunet_fp32.cu -------------------------------------------------
// returns number of kernel launches enqueued, or -1 on launch error
int launch_conv_fp32(const ConvArgs &a, int ksize, int mode, cudaStream_t st);
int launch_out_fp32(const float *dec, const float *x, const float *out_w, const float *out_b, float *y,
                    int B, int C, int T, cudaStream_t st);
int launch_pack_fp32(const float *w, const float *bias, const float *g, const float *beta, const float *mean,
                     const float *var, float *wp, float *scale, float *shift, int Cout, int Cin, int K,
                     cudaStream_t st);

}  // namespace wunet
