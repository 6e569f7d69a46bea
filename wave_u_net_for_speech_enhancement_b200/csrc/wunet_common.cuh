// wunet_common.cuh — shared host/device declarations of the H100 Wave-U-Net forward library.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stddef.h>

namespace wunet {

constexpr float kBnEps = 1e-5f;       // torch.nn.BatchNorm1d default; reference model/unet_basic.py:12,25,55
constexpr float kLreluSlope = 0.1f;   // reference model/unet_basic.py:13,26,56

// Element type of the network input x and output y (WUNET_IO_* in include/wunet_b200.h). The kernels that read x or write y
// take it as a template argument IO (float, __half or __nv_bfloat16): a sample is widened to fp32 on load (exact) and a result
// rounded once to IO on store (round to nearest even); everything in between is the fp32-I/O computation.
enum IoType : int { IO_F32 = 0, IO_F16 = 1, IO_BF16 = 2 };
inline size_t io_bytes(int io) { return io == IO_F32 ? 4 : 2; }

__device__ __forceinline__ float io_f32(float v) { return v; }
__device__ __forceinline__ float io_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float io_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float io_ld(const float *p) { return __ldg(p); }
__device__ __forceinline__ float io_ld(const __half *p) { return __half2float(__ldg(p)); }
__device__ __forceinline__ float io_ld(const __nv_bfloat16 *p) { return __bfloat162float(__ldg(p)); }
__device__ __forceinline__ void io_st(float *p, float v) { *p = v; }
__device__ __forceinline__ void io_st(__half *p, float v) { *p = __float2half_rn(v); }
__device__ __forceinline__ void io_st(__nv_bfloat16 *p, float v) { *p = __float2bfloat16_rn(v); }
// four consecutive elements (16-byte aligned for float, 8-byte aligned for the 16-bit types)
__device__ __forceinline__ float4 io_ld4(const float *p) { return __ldg(reinterpret_cast<const float4 *>(p)); }
__device__ __forceinline__ float4 io_ld4(const __half *p)
{
    const uint2 u = __ldg(reinterpret_cast<const uint2 *>(p));
    const float2 a = __half22float2(*reinterpret_cast<const __half2 *>(&u.x)), b = __half22float2(*reinterpret_cast<const __half2 *>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float4 io_ld4(const __nv_bfloat16 *p)
{
    const uint2 u = __ldg(reinterpret_cast<const uint2 *>(p));
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&u.x));
    const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ void io_st4(float *p, float4 v) { *reinterpret_cast<float4 *>(p) = v; }
__device__ __forceinline__ void io_st4(__half *p, float4 v)
{
    const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
    *reinterpret_cast<uint2 *>(p) = make_uint2(*reinterpret_cast<const uint32_t *>(&a), *reinterpret_cast<const uint32_t *>(&b));
}
__device__ __forceinline__ void io_st4(__nv_bfloat16 *p, float4 v)
{
    const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    *reinterpret_cast<uint2 *>(p) = make_uint2(*reinterpret_cast<const uint32_t *>(&a), *reinterpret_cast<const uint32_t *>(&b));
}

// Where a conv block reads its input from (what the reference does between two Conv1d calls).
enum SrcMode : int {
    SRC_DIRECT = 0,   // x[b][ci][l]                                   (enc0: the raw input)
    SRC_DECIM = 1,    // prev[b][ci][2l]            o = o[:, :, ::2]   (model/unet_basic.py:86)
    SRC_UPCAT = 2,    // cat([interp2x(prev), skip], dim=1)            (model/unet_basic.py:93-95)
};

// One conv + eval-BN + LeakyReLU block on the fp32 path. All activations NCL fp32 (reference layout).
struct ConvArgs {
    const float *src0;   // DIRECT: [B][Cin][L] (elements of the kernel's IO type: block 0 reads the network input); DECIM: [B][Cin][2L]; UPCAT: prev [B][Cin0][L/2]
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

// x -> NCL element fetch with zero padding outside [0, L)  (Conv1d padding, per frame); IO: element type of a DIRECT source
template <int MODE, typename IO = float>
__device__ __forceinline__ float fetch_src(const ConvArgs &a, int b, int ci, int l)
{
    if (l < 0 || l >= a.L) return 0.f;
    if (MODE == SRC_DIRECT) {
        return io_ld(reinterpret_cast<const IO *>(a.src0) + ((size_t)b * a.Cin + ci) * a.L + l);
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
// block 0 (ksize 15, SRC_DIRECT) and the head with a 16-bit network input / output: a.src0, x and y hold IO elements (IoType io)
int launch_conv_fp32_io(const ConvArgs &a, int io, cudaStream_t st);
int launch_out_fp32_io(const float *dec, const void *x, const float *out_w, const float *out_b, void *y, int B, int C, int T,
                       int io, cudaStream_t st);
int launch_pack_fp32(const float *w, const float *bias, const float *g, const float *beta, const float *mean,
                     const float *var, float *wp, float *scale, float *shift, int Cout, int Cin, int K,
                     cudaStream_t st);

// ---- tensor-core training convolutions, implemented in wunet_train_tc.cu ------------------------------------------------
// prec (TrainPrec, wunet_train.cuh) is TRAIN_BF16 (bf16 operands, round to nearest), TRAIN_TF32 (tf32 operands, round to
// nearest, ties away: cvt.rna.tf32.f32) or TRAIN_FP16_SCALED (fp16 operands, round to nearest even; dz staged at its block's
// power-of-two scale, wunet_train_tc_kernels.cuh); products are accumulated in fp32.
// launch_train_conv_tc: launch_conv_fp32's operator with a.wp pointing at the forward (or input-gradient) packing written by
// train_tc_pack at the same precision; ksize 15 (DIRECT, DECIM) or 5 (DIRECT, UPCAT).
int launch_train_conv_tc(int prec, const ConvArgs &a, int ksize, int mode, cudaStream_t st);
// dw[co][ci][k] += sum_{b,l} dz[b][co][l] * in(b, ci, l + k - pad), in read through `a` as the forward reads it (dw zeroed first).
// slices = true: slice z of the grid stores its partial sums to dw + z * Cout * Cin * K instead (nothing zeroed first)
int launch_train_wgrad_tc(int prec, const ConvArgs &a, const float *dz, float *dw, int ksize, int mode, cudaStream_t st,
                          bool slices = false);
// Launch geometry of the weight-gradient kernels, the one definition their launchers and wunet_debug_train_layout use:
// grid, number of (frame, position tile) work items that gridDim.z slices share, and positions per item.
struct WgradGrid { dim3 grid; int items, positions; };
WgradGrid wgrad_grid_fp32(int B, int L, int Cin, int Cout);             // train_wgrad_kernel (wunet_train.cu)
WgradGrid wgrad_grid_tc(int B, int L, int Cin, int Cout, int ksize);    // the tensor-core ones, at every precision
// bytes of one packing of a [cout][cin][k] weight (forward: (cout, cin); input gradient: (cin, cout)); a multiple of 256
size_t train_tc_packed_bytes(int prec, int cout, int cin, int k);
int train_tc_pack(int prec, const float *w, void *wf, void *wb, int Cout, int Cin, int K, cudaStream_t st);
// the TRAIN_FP16_SCALED instances of the three (wunet_train_tc_f16.cu)
int train_tc_pack_f16(const float *w, void *wf, void *wb, int Cout, int Cin, int K, cudaStream_t st);
int launch_train_conv_tc_f16(const ConvArgs &a, int ksize, int mode, cudaStream_t st);
int launch_train_wgrad_tc_f16(const ConvArgs &a, const float *dz, float *dw, int ksize, int mode, cudaStream_t st, bool slices);

// ---- block forward hooks, implemented in wunet_hooks.cu ---------------------------------------------------------------------
// How a block output is stored in an inference workspace: channels-last bf16 or fp16 [B][L][C], the split-precision [B][L][hi C |
// lo C] bf16 halves, or fp32 [B][C][L] (the fp32 path).
enum LevelKind : int { LEVEL_BF16 = 0, LEVEL_SPLIT = 1, LEVEL_F16 = 2, LEVEL_F32_NCL = 3 };
// dst [B][C][L] of IoType io (IO_F16 or IO_BF16): each element widened exactly to fp32, then rounded once to io. 1 launch, or -1.
int launch_level_export_io(const void *src, int kind, void *dst, int io, int B, int L, int C, cudaStream_t st);
// ga[0 .. n) += g[0 .. n), element by element. 1 launch, or -1.
int launch_grad_inject(float *ga, const float *g, long long n, cudaStream_t st);

}  // namespace wunet
