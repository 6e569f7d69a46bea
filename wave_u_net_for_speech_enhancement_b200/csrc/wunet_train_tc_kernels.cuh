// wunet_train_tc_kernels.cuh — the tensor-core convolutions of the training step, templated on the operand type: bf16 and tf32
// (instantiated in wunet_train_tc.cu) and fp16 with per-block dz scaling (wunet_train_tc_f16.cu). DESIGN.md §5.4.
//
// Arithmetic: the operands of the three convolution-shaped passes (block input, weights, dz) are rounded to the operand type
// (bf16: round to nearest; tf32: 10 explicit mantissa bits, round to nearest with ties away from zero, cvt.rna.tf32.f32, done
// here at staging and packing time rather than left to the MMA, as cuDNN does for Conv1d with torch.backends.cudnn.allow_tf32;
// fp16: round to nearest even, beyond +-65504 to +-inf, no saturation) and the products are accumulated in fp32 by sm_90a wgmma;
// everything around them (z, BatchNorm, the adjoints of decimation / interpolation / concat, all gradients) stays fp32 in
// wunet_train.cu, over the same fp32 NCL workspace. A 128B-swizzled K row holds 64 bf16 / fp16 or 32 fp32 elements, so one K
// step (bf16 / fp16 K16, tf32 K8) is 32 bytes of it in all three.
// fp16 (Op::kScaled) has too little range for dz (about 1e-7 at the reference's batch), so the two passes that read dz stage
// fp16(dz 2^k) and multiply their fp32 results by 2^-k, k = dz_scale_exp(max |dz|) of the block (wunet_train.cuh); powers of
// two are exact in fp32, so the pass computes sum fp16(dz 2^k) fp16(x) 2^-k. The block's max |dz| reaches the kernels through a
// ConvArgs pointer the pass does not otherwise read (null = unscaled): a.src1 of the input-gradient conv (DIRECT mode, no skip
// input) and a.scale of the weight gradient (no epilogue).
//
//   train_conv_tc_kernel<Op>  implicit-GEMM conv with a linear epilogue, out = conv(in, w) * scale + shift, the interface of
//                             launch_conv_fp32: the forward conv (z, modes DIRECT / DECIM / UPCAT) and the input gradient (DIRECT
//                             over dz with the transposed, flipped weights). M = 128 output positions of one frame, N = Cout
//                             (16 .. 64 columns per CTA), K = Op::kChunk-channel chunks x taps. All 256 threads stage the operand
//                             tile: the block input is read from fp32 NCL (decimation / interpolation + concat as in fetch_src),
//                             rounded and written K-major as 128B-swizzled [position][kChunk channels] rows, so a tap is the A
//                             descriptor advanced by one 128-byte row. The weights come pre-packed (train_tc_pack_kernel) and are
//                             staged five taps at a time. Each of the two warpgroups owns one m64 half of the tile.
//   train_wgrad_tc_kernel<Op> (bf16, fp16) dW[co][ci][k] = sum_{b,l} dz[b][co][l] in(b, ci, l + k - pad): per tap a GEMM with M = co,
//                             N = ci and K = (b, l). The tap shift lies along K, so both operands are staged channels-last, dz as
//                             [position][64 co] and the input as [position][64 ci] (128B-swizzled), and fed MN-major
//                             (imm-trans = 1): a tap advances the B descriptor by one 128-byte row, exactly as in the forward.
//   train_wgrad_tf32_kernel   the same GEMMs with tf32 operands, which must be K-major (the PTX has no transpose immediates for
//                             tf32). K is the position axis here, so a tap is a shift of ONE element (4 bytes) along K, which no
//                             descriptor can express (start addresses move in 16-byte steps). The CTA therefore stages dz as
//                             [64 co][64 positions] and, per tap of its group, one shifted copy of the block input as
//                             [64 ci][64 positions] (16 KB each): every thread reads one element of the 68-position input window
//                             once and stores it into the five copies.
// A weight-gradient CTA owns 64 co x 64 ci x 5 taps (160 accumulator registers per thread); the (frame, 64-position) items are
// split over gridDim.z and combined with fp32 atomicAdd or, in deterministic mode, stored per slice and summed in slice order
// by wunet_train.cu.
//
// Tiles never straddle two frames: a tile's rows past the frame end are computed and discarded, and positions outside
// [0, L) read as zero (Conv1d padding, per frame), so frames shorter than a tile (the bottom of the U) are padded, never packed.
#pragma once
#include "wunet_common.cuh"
#include "wunet_train.cuh"
#include "wunet_wgmma.cuh"

#include <algorithm>
#include <type_traits>

namespace wunet {

namespace {

constexpr int kRows = 128;        // output positions per forward tile (two m64 halves, one per warpgroup)
constexpr int kTapGroup = 5;      // taps per staged weight group / per weight-gradient CTA (both kernel sizes are multiples)
constexpr int kWgPos = 64;        // positions per weight-gradient item
constexpr uint32_t kAtomBytes = 64 * 128;      // one [64 rows][32 fp32] swizzled K atom of the tf32 weight gradient

// descriptor words of a 128B-swizzled operand: hi = SBO(1024 B) | SWIZZLE_128B; lo = (addr >> 4) | LBO << 16. K-major operands
// ignore LBO; the MN-major ones of the bf16 weight gradient hold exactly one 64-element atom along M / N, so LBO is never
// followed either (set to 1024 B all the same).
constexpr uint32_t kDescHi = (uint32_t)(1024 >> 4) | (1u << 30);
__device__ __forceinline__ uint32_t desc_lo(uint32_t addr) { return ((addr >> 4) & 0x3FFFu) | ((uint32_t)(1024 >> 4) << 16); }

// Operand types: the elements of one 128-byte K row (2^kLogChunk), the storage of a packed weight, the rounding of one value,
// the byte offset of (row, element) in a [rows][kChunk] 128B-swizzled tile whose base is 1024-byte aligned, and one K step's MMA.
// kScaled: dz is staged at its block's power-of-two scale (see above).
struct Bf16 {
    static constexpr bool kScaled = false;
    static constexpr int kLogChunk = 6, kChunk = 1 << kLogChunk;
    using W = __nv_bfloat16;
    __device__ __forceinline__ static W round(float v) { return __float2bfloat16_rn(v); }
    __device__ __forceinline__ static uint32_t swz(int row, int e) { return (uint32_t)(row * 128 + ((((e >> 3) ^ row) & 7) << 4) + (e & 7) * 2); }
    template <int N>
    __device__ __forceinline__ static void mma(float (&acc)[N / 2], uint32_t a_lo, uint32_t b_lo) { wgmma_m64nNk16<N>(acc, a_lo, b_lo, kDescHi); }
};
struct Tf32 {
    static constexpr bool kScaled = false;
    static constexpr int kLogChunk = 5, kChunk = 1 << kLogChunk;
    using W = float;
    __device__ __forceinline__ static W round(float v)
    {
        uint32_t r;
        asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
        return __uint_as_float(r);
    }
    __device__ __forceinline__ static uint32_t swz(int row, int e) { return (uint32_t)(row * 128 + ((((e >> 2) ^ row) & 7) << 4) + (e & 3) * 4); }
    template <int N>
    __device__ __forceinline__ static void mma(float (&acc)[N / 2], uint32_t a_lo, uint32_t b_lo) { wgmma_m64nNk8_tf32<N>(acc, a_lo, b_lo, kDescHi); }
};
struct F16 {
    static constexpr bool kScaled = true;
    static constexpr int kLogChunk = 6, kChunk = 1 << kLogChunk;
    using W = __half;
    __device__ __forceinline__ static W round(float v) { return __float2half_rn(v); }       // cvt.rn.f16.f32: overflow -> inf
    __device__ __forceinline__ static uint32_t swz(int row, int e) { return Bf16::swz(row, e); }
    template <int N>
    __device__ __forceinline__ static void mma(float (&acc)[N / 2], uint32_t a_lo, uint32_t b_lo) { wgmma_m64nNk16<N, 0, 0, __half>(acc, a_lo, b_lo, kDescHi); }
};

// an fp16 pair (round to nearest even, no saturation), low half = a
__device__ __forceinline__ uint32_t pack_f16(float a, float b)
{
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&h);
}

// 2^k of a block's dz from the max |dz| a scaled pass reads through `amax` (null: 1)
__device__ __forceinline__ float dz_scale_of(const float *amax) { return amax ? ldexpf(1.f, dz_scale_exp(__ldg(amax))) : 1.f; }

// the operand tiles are written with ordinary (generic-proxy) stores and read by wgmma through the async proxy: each writer
// fences before the barrier that hands the tiles to the MMAs
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ unsigned char *align1024(unsigned char *p)
{
    return p + ((1024u - (smem_u32(p) & 1023u)) & 1023u);
}

struct Cols { int nt, ntiles, npad; };
// Cout columns in CTA tiles of nt 16-column blocks (at most 4): as few tiles as possible, as evenly filled as possible
Cols cols_of(int cout)
{
    const int b16 = (cout + 15) / 16, ntiles = (b16 + 3) / 4, nt = (b16 + ntiles - 1) / ntiles;
    return Cols{nt, ntiles, nt * 16 * ntiles};
}

template <class Op, int KS, int MODE, int NT>
__global__ void __launch_bounds__(256, 2) train_conv_tc_kernel(const ConvArgs a, int npad, int nchunks, int tiles_per_frame)
{
    constexpr int PAD = (KS - 1) / 2, AROWS = (kRows + KS - 1 + 7) / 8 * 8, NG = KS / kTapGroup, CH = Op::kChunk;
    constexpr uint32_t TAP_BYTES = NT * 16 * 128;
    static_assert(KS % kTapGroup == 0, "kernel size must be a multiple of the tap group");
    extern __shared__ unsigned char smem_raw[];
    unsigned char *sa = align1024(smem_raw);
    unsigned char *sb = sa + AROWS * 128;
    const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
    const int b = blockIdx.x / tiles_per_frame, l0 = (blockIdx.x - b * tiles_per_frame) * kRows;
    const int n0 = blockIdx.y * NT * 16;
    const typename Op::W *wpk = reinterpret_cast<const typename Op::W *>(a.wp);
    const uint32_t a_lo = desc_lo(smem_u32(sa) + (uint32_t)wg * 64 * 128), b_lo = desc_lo(smem_u32(sb));
    float acc[NT * 8];
#pragma unroll
    for (int j = 0; j < NT * 8; ++j) acc[j] = 0.f;
    float sk = 1.f;                                            // scaled operand types: the input gradient's dz at 2^k
    if constexpr (Op::kScaled)
        if (MODE == SRC_DIRECT) sk = dz_scale_of(a.src1);
    for (int c = 0; c < nchunks; ++c) {
        __syncthreads();                                       // both warpgroups are done with the previous chunk's tiles
        // one 32-bit word per thread and step: a bf16 / fp16 channel pair or one tf32 channel (written here rather than through
        // a member of Op, which changes the instruction schedule of the bf16 kernels)
        for (int i = tid; i < AROWS * 32; i += 256) {
            const int r = i % AROWS, ch = CH / 32 * (i / AROWS), ci = c * CH + ch, l = l0 - PAD + r;
            const bool rok = r < kRows + KS - 1;
            if constexpr (Op::kScaled) {
                const float v0 = (rok && ci < a.Cin) ? fetch_src<MODE>(a, b, ci, l) : 0.f;
                const float v1 = (rok && ci + 1 < a.Cin) ? fetch_src<MODE>(a, b, ci + 1, l) : 0.f;
                *reinterpret_cast<uint32_t *>(sa + Op::swz(r, ch)) = pack_f16(v0 * sk, v1 * sk);
            } else if constexpr (CH == 64) {
                const float v0 = (rok && ci < a.Cin) ? fetch_src<MODE>(a, b, ci, l) : 0.f;
                const float v1 = (rok && ci + 1 < a.Cin) ? fetch_src<MODE>(a, b, ci + 1, l) : 0.f;
                *reinterpret_cast<uint32_t *>(sa + Op::swz(r, ch)) = pack_bf16(v0, v1);
            } else {
                const float v = (rok && ci < a.Cin) ? fetch_src<MODE>(a, b, ci, l) : 0.f;
                *reinterpret_cast<float *>(sa + Op::swz(r, ch)) = Op::round(v);
            }
        }
        for (int g = 0; g < NG; ++g) {
            if (g > 0) __syncthreads();                        // the previous weight group has been consumed
            const typename Op::W *src = wpk + ((size_t)c * KS + g * kTapGroup) * npad * CH;
            for (int i = tid; i < kTapGroup * NT * 16 * 8; i += 256) {
                const int v = i & 7, row = (i >> 3) % (NT * 16), tt = (i >> 3) / (NT * 16);
                const uint4 val = __ldg(reinterpret_cast<const uint4 *>(src + ((size_t)tt * npad + n0 + row) * CH) + v);
                *reinterpret_cast<uint4 *>(sb + tt * TAP_BYTES + Op::swz(row, CH / 8 * v)) = val;
            }
            fence_proxy_async();
            __syncthreads();
            wgmma_fence();
#pragma unroll
            for (int tt = 0; tt < kTapGroup; ++tt)
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    Op::template mma<16 * NT>(acc, a_lo + (uint32_t)(g * kTapGroup + tt) * 8u + 2u * k,   // tap: +128 B, K step: +32 B
                                              b_lo + (uint32_t)tt * (TAP_BYTES >> 4) + 2u * k);
            wgmma_commit();
            wgmma_wait0();
        }
    }
    if constexpr (Op::kScaled) {
        const float inv = 1.f / sk;                            // exact: sk is a normal power of two
#pragma unroll
        for (int j = 0; j < NT * 8; ++j) acc[j] *= inv;
    }
    // epilogue: thread (wq, lane) holds rows 16 wq + lane / 4 (+8) and columns 2 (lane % 4) (+1) of every 8-column group
#pragma unroll
    for (int j = 0; j < NT * 8; ++j) {
        const int row = wg * 64 + 16 * wq + (lane >> 2) + 8 * ((j >> 1) & 1);
        const int col = n0 + 8 * (j >> 2) + 2 * (lane & 3) + (j & 1);
        const int l = l0 + row;
        if (l < a.L && col < a.Cout)
            a.out[((size_t)b * a.Cout + col) * a.L + l] = bn_lrelu(acc[j], __ldg(a.scale + col), __ldg(a.shift + col), a.linear);
    }
}

// the dW of a weight-gradient CTA: thread (wq, lane) holds rows (co) 16 wq + lane / 4 (+8) and columns (ci) 2 (lane % 4) (+1) of
// every 8-column group of each tap's fragment. SLICES (deterministic mode): slice blockIdx.z stores its partial sums to its own
// copy of dW at dw + blockIdx.z * Cout Cin KS; otherwise they are added to dW with atomicAdd.
template <int KS, bool SLICES>
__device__ __forceinline__ void store_dw(const float (&acc)[kTapGroup][32], const ConvArgs &a, float *dw, int co0, int ci0, int t0,
                                         int wq, int lane)
{
    if (SLICES) dw += (size_t)blockIdx.z * a.Cout * a.Cin * KS;
#pragma unroll
    for (int tt = 0; tt < kTapGroup; ++tt)
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            const int co = co0 + 16 * wq + (lane >> 2) + 8 * ((j >> 1) & 1);
            const int ci = ci0 + 8 * (j >> 2) + 2 * (lane & 3) + (j & 1);
            if (co < a.Cout && ci < a.Cin) {
                float *d = dw + ((size_t)co * a.Cin + ci) * KS + t0 + tt;
                if (SLICES) *d = acc[tt][j];
                else atomicAdd(d, acc[tt][j]);
            }
        }
}

template <class Op, int KS, int MODE, bool SLICES>
__global__ void __launch_bounds__(128) train_wgrad_tc_kernel(const ConvArgs a, const float *__restrict__ dz, float *__restrict__ dw,
                                                               int chunks_per_frame)
{
    static_assert(Op::kChunk == 64, "MN-major operands of 64 two-byte elements per 128-byte row");
    constexpr int PAD = (KS - 1) / 2, XROWS = (kWgPos + KS - 1 + 7) / 8 * 8, NG = KS / kTapGroup;
    static_assert(KS % kTapGroup == 0, "kernel size must be a multiple of the tap group");
    extern __shared__ unsigned char smem_raw[];
    unsigned char *sd = align1024(smem_raw);                   // [kWgPos positions][64 co]
    unsigned char *sx = sd + kWgPos * 128;                     // [XROWS positions][64 ci], row r = position l0 - PAD + r
    const int tid = threadIdx.x, wq = tid >> 5, lane = tid & 31;
    const int co0 = (blockIdx.x / NG) * 64, t0 = (blockIdx.x % NG) * kTapGroup, ci0 = blockIdx.y * 64;
    const uint32_t d_lo = desc_lo(smem_u32(sd)), x_lo = desc_lo(smem_u32(sx));
    float acc[kTapGroup][32];
#pragma unroll
    for (int t = 0; t < kTapGroup; ++t)
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[t][j] = 0.f;
    float sk = 1.f;                                            // scaled operand types: dz at 2^k
    if constexpr (Op::kScaled) sk = dz_scale_of(a.scale);
    const int items = a.B * chunks_per_frame;
    for (int it = blockIdx.z; it < items; it += gridDim.z) {
        const int b = it / chunks_per_frame, l0 = (it - b * chunks_per_frame) * kWgPos;
        __syncthreads();
        for (int i = tid; i < kWgPos * 32; i += 128) {
            const int p = i % kWgPos, ch = 2 * (i / kWgPos), co = co0 + ch, l = l0 + p;
            const float *dr = dz + ((size_t)b * a.Cout + co) * a.L + l;
            const float v0 = (l < a.L && co < a.Cout) ? __ldg(dr) : 0.f;
            const float v1 = (l < a.L && co + 1 < a.Cout) ? __ldg(dr + a.L) : 0.f;
            if constexpr (Op::kScaled) *reinterpret_cast<uint32_t *>(sd + Bf16::swz(p, ch)) = pack_f16(v0 * sk, v1 * sk);
            else *reinterpret_cast<uint32_t *>(sd + Bf16::swz(p, ch)) = pack_bf16(v0, v1);
        }
        for (int i = tid; i < XROWS * 32; i += 128) {
            const int r = i % XROWS, ch = 2 * (i / XROWS), ci = ci0 + ch, l = l0 - PAD + r;
            const bool rok = r < kWgPos + KS - 1;
            const float v0 = (rok && ci < a.Cin) ? fetch_src<MODE>(a, b, ci, l) : 0.f;
            const float v1 = (rok && ci + 1 < a.Cin) ? fetch_src<MODE>(a, b, ci + 1, l) : 0.f;
            if constexpr (Op::kScaled) *reinterpret_cast<uint32_t *>(sx + Bf16::swz(r, ch)) = pack_f16(v0, v1);
            else *reinterpret_cast<uint32_t *>(sx + Bf16::swz(r, ch)) = pack_bf16(v0, v1);
        }
        fence_proxy_async();
        __syncthreads();
        wgmma_fence();
#pragma unroll
        for (int tt = 0; tt < kTapGroup; ++tt)
#pragma unroll
            for (int k = 0; k < 4; ++k)                          // K16 step: 16 position rows = 2048 B in both operands
                wgmma_m64nNk16<64, 1, 1, typename Op::W>(acc[tt], d_lo + 128u * k, x_lo + (uint32_t)(t0 + tt) * 8u + 128u * k, kDescHi);
        wgmma_commit();
        wgmma_wait0();
    }
    if constexpr (Op::kScaled) {
        const float inv = 1.f / sk;                            // exact: sk is a normal power of two
#pragma unroll
        for (int t = 0; t < kTapGroup; ++t)
#pragma unroll
            for (int j = 0; j < 32; ++j) acc[t][j] *= inv;
    }
    store_dw<KS, SLICES>(acc, a, dw, co0, ci0, t0, wq, lane);
}

template <int KS, int MODE, bool SLICES>
__global__ void __launch_bounds__(128) train_wgrad_tf32_kernel(const ConvArgs a, const float *__restrict__ dz, float *__restrict__ dw,
                                                               int chunks_per_frame)
{
    constexpr int PAD = (KS - 1) / 2, XW = kWgPos + kTapGroup - 1, NG = KS / kTapGroup;
    static_assert(KS % kTapGroup == 0, "kernel size must be a multiple of the tap group");
    extern __shared__ unsigned char smem_raw[];
    unsigned char *sd = align1024(smem_raw);                   // dz: 2 K atoms of [64 co][32 positions]
    unsigned char *sx = sd + 2 * kAtomBytes;                   // per tap tt: 2 K atoms of [64 ci][32 positions], position p
                                                               // holding in(ci, l0 + p + t0 + tt - PAD)
    const int tid = threadIdx.x, wq = tid >> 5, lane = tid & 31;
    const int co0 = (blockIdx.x / NG) * 64, t0 = (blockIdx.x % NG) * kTapGroup, ci0 = blockIdx.y * 64;
    const uint32_t d_lo = desc_lo(smem_u32(sd)), x_lo = desc_lo(smem_u32(sx));
    float acc[kTapGroup][32];
#pragma unroll
    for (int t = 0; t < kTapGroup; ++t)
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[t][j] = 0.f;
    const int items = a.B * chunks_per_frame;
    for (int it = blockIdx.z; it < items; it += gridDim.z) {
        const int b = it / chunks_per_frame, l0 = (it - b * chunks_per_frame) * kWgPos;
        __syncthreads();
        for (int i = tid; i < kWgPos * 64; i += 128) {
            const int p = i % kWgPos, co = co0 + i / kWgPos, l = l0 + p;
            const float v = (l < a.L && co < a.Cout) ? __ldg(dz + ((size_t)b * a.Cout + co) * a.L + l) : 0.f;
            *reinterpret_cast<float *>(sd + (p >> 5) * kAtomBytes + Tf32::swz(i / kWgPos, p & 31)) = Tf32::round(v);
        }
        // window element r = in(ci, l0 + t0 - PAD + r) is position p = r - tt of tap copy tt
        for (int i = tid; i < XW * 64; i += 128) {
            const int r = i % XW, cl = i / XW, ci = ci0 + cl;
            const float v = Tf32::round(ci < a.Cin ? fetch_src<MODE>(a, b, ci, l0 + t0 - PAD + r) : 0.f);
#pragma unroll
            for (int tt = 0; tt < kTapGroup; ++tt) {
                const int p = r - tt;
                if (p >= 0 && p < kWgPos)
                    *reinterpret_cast<float *>(sx + (tt * 2 + (p >> 5)) * kAtomBytes + Tf32::swz(cl, p & 31)) = v;
            }
        }
        fence_proxy_async();
        __syncthreads();
        wgmma_fence();
#pragma unroll
        for (int tt = 0; tt < kTapGroup; ++tt)
#pragma unroll
            for (int k = 0; k < 8; ++k) {                        // K8 step k: atom k / 4, +32 B within it
                const uint32_t off = (uint32_t)(k >> 2) * (kAtomBytes >> 4) + 2u * (k & 3);
                wgmma_m64nNk8_tf32<64>(acc[tt], d_lo + off, x_lo + (uint32_t)(2 * tt) * (kAtomBytes >> 4) + off, kDescHi);
            }
        wgmma_commit();
        wgmma_wait0();
    }
    store_dw<KS, SLICES>(acc, a, dw, co0, ci0, t0, wq, lane);
}

// both packings of a block's weights w[Cout][Cin][K], rounded to the operand type, every step (CH = Op::kChunk):
//   wf[((c K + t) npad(Cout) + co) CH + j] = w[co][CH c + j][t]          forward conv: [chunk][tap][Cout rows][CH channels]
//   wb[((c K + t) npad(Cin) + ci) CH + j]  = w[CH c + j][ci][K-1-t]      input gradient: transposed and flipped
// (zero where the channel or column is padding). The element index is split with shifts: i / CH on the signed 64-bit index
// compiles to a longer sequence.
template <class Op>
__global__ void train_tc_pack_kernel(const float *__restrict__ w, typename Op::W *__restrict__ wf, typename Op::W *__restrict__ wb,
                                     int Cout, int Cin, int K, int npad_f, int npad_b, long long nf, long long nb)
{
    constexpr int CH = Op::kChunk;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nf) {
        const int j = (int)(i & (CH - 1));
        const long long r = i >> Op::kLogChunk;
        const int row = (int)(r % npad_f);
        const int ct = (int)(r / npad_f), t = ct % K, c = ct / K;
        const int ci = c * CH + j;
        wf[i] = Op::round((row < Cout && ci < Cin) ? w[((size_t)row * Cin + ci) * K + t] : 0.f);
    } else if (i < nf + nb) {
        const long long q = i - nf;
        const int j = (int)(q & (CH - 1));
        const long long r = q >> Op::kLogChunk;
        const int row = (int)(r % npad_b);
        const int ct = (int)(r / npad_b), t = ct % K, c = ct / K;
        const int co = c * CH + j;
        wb[q] = Op::round((row < Cin && co < Cout) ? w[((size_t)co * Cin + row) * K + (K - 1 - t)] : 0.f);
    }
}

// bytes of one packing of a [cout][cin][k] weight (forward: (cout, cin); input gradient: (cin, cout)): 128-byte rows
template <class Op>
size_t packed_bytes(int cout, int cin, int k) { return (size_t)((cin + Op::kChunk - 1) / Op::kChunk) * k * cols_of(cout).npad * 128; }

template <class Op>
int pack(const float *w, void *wf, void *wb, int Cout, int Cin, int K, cudaStream_t st)
{
    using W = typename Op::W;
    const long long nf = (long long)(packed_bytes<Op>(Cout, Cin, K) / sizeof(W)), nb = (long long)(packed_bytes<Op>(Cin, Cout, K) / sizeof(W));
    train_tc_pack_kernel<Op><<<(unsigned)((nf + nb + 255) / 256), 256, 0, st>>>(w, static_cast<W *>(wf), static_cast<W *>(wb), Cout, Cin,
                                                                                K, cols_of(Cout).npad, cols_of(Cin).npad, nf, nb);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

template <class Op, int KS, int MODE, int NT>
int launch_conv(const ConvArgs &a, cudaStream_t st)
{
    constexpr int AROWS = (kRows + KS - 1 + 7) / 8 * 8;
    constexpr int smem = AROWS * 128 + kTapGroup * NT * 16 * 128 + 1024;
    if (cudaFuncSetAttribute(train_conv_tc_kernel<Op, KS, MODE, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
        return -1;                                             // (per device: set on every launch)
    const Cols cc = cols_of(a.Cout);
    const int tiles_per_frame = (a.L + kRows - 1) / kRows;
    const dim3 grid((unsigned)(a.B * tiles_per_frame), (unsigned)cc.ntiles);
    train_conv_tc_kernel<Op, KS, MODE, NT><<<grid, 256, smem, st>>>(a, cc.npad, (a.Cin + Op::kChunk - 1) / Op::kChunk, tiles_per_frame);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

template <class Op, int KS, int MODE>
int launch_conv_nt(const ConvArgs &a, cudaStream_t st)
{
    switch (cols_of(a.Cout).nt) {
    case 1: return launch_conv<Op, KS, MODE, 1>(a, st);
    case 2: return launch_conv<Op, KS, MODE, 2>(a, st);
    case 3: return launch_conv<Op, KS, MODE, 3>(a, st);
    default: return launch_conv<Op, KS, MODE, 4>(a, st);
    }
}

template <class Op>
int launch_conv_op(const ConvArgs &a, int ksize, int mode, cudaStream_t st)
{
    if (ksize == 15 && mode == SRC_DIRECT) return launch_conv_nt<Op, 15, SRC_DIRECT>(a, st);
    if (ksize == 15 && mode == SRC_DECIM) return launch_conv_nt<Op, 15, SRC_DECIM>(a, st);
    if (ksize == 5 && mode == SRC_DIRECT) return launch_conv_nt<Op, 5, SRC_DIRECT>(a, st);
    if (ksize == 5 && mode == SRC_UPCAT) return launch_conv_nt<Op, 5, SRC_UPCAT>(a, st);
    return -1;
}

template <class Op, int KS, int MODE>
int launch_wgrad(const ConvArgs &a, const float *dz, float *dw, cudaStream_t st, bool slices)
{
    constexpr int XROWS = (kWgPos + KS - 1 + 7) / 8 * 8;
    constexpr bool tf32 = std::is_same<Op, Tf32>::value;
    const int smem = tf32 ? (2 + 2 * kTapGroup) * kAtomBytes + 1024 : (kWgPos + XROWS) * 128 + 1024;
    void (*kern)(const ConvArgs, const float *, float *, int);
    if constexpr (tf32) kern = slices ? train_wgrad_tf32_kernel<KS, MODE, true> : train_wgrad_tf32_kernel<KS, MODE, false>;
    else kern = slices ? train_wgrad_tc_kernel<Op, KS, MODE, true> : train_wgrad_tc_kernel<Op, KS, MODE, false>;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return -1;
    const WgradGrid g = wgrad_grid_tc(a.B, a.L, a.Cin, a.Cout, KS);
    kern<<<g.grid, 128, smem, st>>>(a, dz, dw, (a.L + kWgPos - 1) / kWgPos);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

template <class Op>
int launch_wgrad_op(const ConvArgs &a, const float *dz, float *dw, int ksize, int mode, cudaStream_t st, bool slices)
{
    if (ksize == 15 && mode == SRC_DIRECT) return launch_wgrad<Op, 15, SRC_DIRECT>(a, dz, dw, st, slices);
    if (ksize == 15 && mode == SRC_DECIM) return launch_wgrad<Op, 15, SRC_DECIM>(a, dz, dw, st, slices);
    if (ksize == 5 && mode == SRC_UPCAT) return launch_wgrad<Op, 5, SRC_UPCAT>(a, dz, dw, st, slices);
    return -1;
}

}  // namespace

}  // namespace wunet
