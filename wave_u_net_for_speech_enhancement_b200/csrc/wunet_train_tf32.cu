// wunet_train_tf32.cu — tf32 tensor-core convolutions of the training step (Model(train_precision="tf32"), DESIGN.md §5.4).
//
// Arithmetic: the operands of the three convolution-shaped passes (block input, weights, dz) are rounded to tf32 (10 explicit
// mantissa bits, round to nearest with ties away from zero: cvt.rna.tf32.f32, done here at staging and packing time rather
// than left to the MMA) and the products are accumulated in fp32 by sm_90a wgmma (m64nNk8.f32.tf32.tf32); everything around
// them stays fp32 in wunet_train.cu, over the same fp32 NCL workspace. This is what cuDNN does for Conv1d with
// torch.backends.cudnn.allow_tf32 (PyTorch's default).
//
// 32-bit wgmma operands must be K-major (the PTX has no transpose immediates for tf32), and a 128B-swizzled row holds 32 fp32
// K elements (four K8 steps, 32 bytes each: the same descriptor advance as a bf16 K16 step).
//   train_conv_tf32_kernel    train_conv_tc_kernel's tiling with 32-channel K chunks: M = 128 output positions of one frame,
//                             N = Cout (16 .. 64 columns per CTA), K = 32-channel chunks x taps. The block input is staged
//                             K-major as [position][32 channels] rows, so a tap is still the A descriptor advanced by one
//                             128-byte row; the weights come pre-packed as tf32 [chunk][tap][Cout rows][32 channels].
//   train_wgrad_tf32_kernel   dW[co][ci][k] = sum_{b,l} dz[b][co][l] in(b, ci, l + k - pad): per tap a GEMM with M = co, N = ci,
//                             K = (b, l). K is the position axis here, so a tap is a shift of ONE element (4 bytes) along K,
//                             which no descriptor can express (start addresses move in 16-byte steps). The CTA (64 co x 64 ci x
//                             5 taps) therefore stages dz as [64 co][64 positions] and, per tap of its group, one shifted copy
//                             of the block input as [64 ci][64 positions] (16 KB each): every thread reads one element of the
//                             68-position input window once and stores it into the five copies. The (frame, 64-position) items
//                             are split over gridDim.z and combined with fp32 atomicAdd or, in deterministic mode, stored per
//                             slice and summed in slice order by wunet_train.cu.
//
// Tiles never straddle two frames: a tile's rows past the frame end are computed and discarded, and positions outside
// [0, L) read as zero (Conv1d padding, per frame).
#include "wunet_common.cuh"
#include "wunet_wgmma.cuh"

#include <algorithm>

namespace wunet {

namespace {

constexpr int kRows = 128;        // output positions per forward tile (two m64 halves, one per warpgroup)
constexpr int kChunk = 32;        // fp32 channels per 128-byte K-major row (forward K chunk)
constexpr int kTapGroup = 5;      // taps per staged weight group / per weight-gradient CTA (both kernel sizes are multiples)
constexpr int kWgPos = 64;        // positions per weight-gradient item (two 32-position K atoms, eight K8 steps)
constexpr uint32_t kAtomBytes = 64 * 128;      // one [64 rows][32 fp32] swizzled K atom of the weight gradient

// descriptor words of a K-major 128B-swizzled operand: hi = SBO(1024 B) | SWIZZLE_128B; lo = (addr >> 4) | LBO << 16 (LBO is
// not used by K-major swizzled operands)
constexpr uint32_t kDescHi = (uint32_t)(1024 >> 4) | (1u << 30);
__device__ __forceinline__ uint32_t desc_lo(uint32_t addr) { return ((addr >> 4) & 0x3FFFu) | ((uint32_t)(1024 >> 4) << 16); }

// byte offset of (row, element e) in a [rows][32 fp32] 128B-swizzled tile whose base is 1024-byte aligned
__device__ __forceinline__ uint32_t swz(int row, int e) { return (uint32_t)(row * 128 + ((((e >> 2) ^ row) & 7) << 4) + (e & 3) * 4); }

__device__ __forceinline__ float tf32_rna(float v)
{
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return __uint_as_float(r);
}

// the operand tiles are written with ordinary (generic-proxy) stores and read by wgmma through the async proxy
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

template <int KS, int MODE, int NT>
__global__ void __launch_bounds__(256, 2) train_conv_tf32_kernel(const ConvArgs a, int npad, int nchunks, int tiles_per_frame)
{
    constexpr int PAD = (KS - 1) / 2, AROWS = (kRows + KS - 1 + 7) / 8 * 8, NG = KS / kTapGroup;
    constexpr uint32_t TAP_BYTES = NT * 16 * 128;
    static_assert(KS % kTapGroup == 0, "kernel size must be a multiple of the tap group");
    extern __shared__ unsigned char smem_raw[];
    unsigned char *sa = align1024(smem_raw);
    unsigned char *sb = sa + AROWS * 128;
    const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
    const int b = blockIdx.x / tiles_per_frame, l0 = (blockIdx.x - b * tiles_per_frame) * kRows;
    const int n0 = blockIdx.y * NT * 16;
    const uint32_t a_lo = desc_lo(smem_u32(sa) + (uint32_t)wg * 64 * 128), b_lo = desc_lo(smem_u32(sb));
    float acc[NT * 8];
#pragma unroll
    for (int j = 0; j < NT * 8; ++j) acc[j] = 0.f;
    for (int c = 0; c < nchunks; ++c) {
        __syncthreads();                                       // both warpgroups are done with the previous chunk's tiles
        for (int i = tid; i < AROWS * kChunk; i += 256) {
            const int r = i % AROWS, ch = i / AROWS, ci = c * kChunk + ch, l = l0 - PAD + r;
            const float v = (r < kRows + KS - 1 && ci < a.Cin) ? fetch_src<MODE>(a, b, ci, l) : 0.f;
            *reinterpret_cast<float *>(sa + swz(r, ch)) = tf32_rna(v);
        }
        for (int g = 0; g < NG; ++g) {
            if (g > 0) __syncthreads();                        // the previous weight group has been consumed
            const float *src = a.wp + ((size_t)c * KS + g * kTapGroup) * npad * kChunk;
            for (int i = tid; i < kTapGroup * NT * 16 * 8; i += 256) {
                const int v = i & 7, row = (i >> 3) % (NT * 16), tt = (i >> 3) / (NT * 16);
                const uint4 val = __ldg(reinterpret_cast<const uint4 *>(src + ((size_t)tt * npad + n0 + row) * kChunk) + v);
                *reinterpret_cast<uint4 *>(sb + tt * TAP_BYTES + swz(row, 4 * v)) = val;
            }
            fence_proxy_async();
            __syncthreads();
            wgmma_fence();
#pragma unroll
            for (int tt = 0; tt < kTapGroup; ++tt)
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    wgmma_m64nNk8_tf32<16 * NT>(acc, a_lo + (uint32_t)(g * kTapGroup + tt) * 8u + 2u * k,   // tap: +128 B, K8: +32 B
                                                b_lo + (uint32_t)tt * (TAP_BYTES >> 4) + 2u * k, kDescHi);
            wgmma_commit();
            wgmma_wait0();
        }
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

// SLICES (deterministic mode): slice blockIdx.z stores its partial sums to its own copy of dW at dw + blockIdx.z * Cout Cin KS
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
            *reinterpret_cast<float *>(sd + (p >> 5) * kAtomBytes + swz(i / kWgPos, p & 31)) = tf32_rna(v);
        }
        // window element r = in(ci, l0 + t0 - PAD + r) is position p = r - tt of tap copy tt
        for (int i = tid; i < XW * 64; i += 128) {
            const int r = i % XW, cl = i / XW, ci = ci0 + cl;
            const float v = tf32_rna(ci < a.Cin ? fetch_src<MODE>(a, b, ci, l0 + t0 - PAD + r) : 0.f);
#pragma unroll
            for (int tt = 0; tt < kTapGroup; ++tt) {
                const int p = r - tt;
                if (p >= 0 && p < kWgPos)
                    *reinterpret_cast<float *>(sx + (tt * 2 + (p >> 5)) * kAtomBytes + swz(cl, p & 31)) = v;
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
    // fragment: row (co) = 16 wq + lane / 4 (+8), column (ci) = 2 (lane % 4) (+1) of every 8-column group
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

// both tf32 packings of a block's weights w[Cout][Cin][K], every step (128-byte K-major rows of 32 channels):
//   wf[((c K + t) npad(Cout) + co) 32 + j] = tf32(w[co][32 c + j][t])          forward conv: [chunk][tap][Cout rows][32 channels]
//   wb[((c K + t) npad(Cin) + ci) 32 + j]  = tf32(w[32 c + j][ci][K-1-t])      input gradient: transposed and flipped
// (zero where the channel or column is padding)
__global__ void train_tf32_pack_kernel(const float *__restrict__ w, float *__restrict__ wf, float *__restrict__ wb, int Cout, int Cin,
                                       int K, int npad_f, int npad_b, long long nf, long long nb)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nf) {
        const int j = (int)(i & 31);
        const long long r = i >> 5;
        const int row = (int)(r % npad_f);
        const int ct = (int)(r / npad_f), t = ct % K, c = ct / K;
        const int ci = c * kChunk + j;
        wf[i] = tf32_rna((row < Cout && ci < Cin) ? w[((size_t)row * Cin + ci) * K + t] : 0.f);
    } else if (i < nf + nb) {
        const long long q = i - nf;
        const int j = (int)(q & 31);
        const long long r = q >> 5;
        const int row = (int)(r % npad_b);
        const int ct = (int)(r / npad_b), t = ct % K, c = ct / K;
        const int co = c * kChunk + j;
        wb[q] = tf32_rna((row < Cin && co < Cout) ? w[((size_t)co * Cin + row) * K + (K - 1 - t)] : 0.f);
    }
}

template <int KS, int MODE, int NT>
int launch_conv(const ConvArgs &a, cudaStream_t st)
{
    constexpr int AROWS = (kRows + KS - 1 + 7) / 8 * 8;
    constexpr int smem = AROWS * 128 + kTapGroup * NT * 16 * 128 + 1024;
    if (cudaFuncSetAttribute(train_conv_tf32_kernel<KS, MODE, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
        return -1;                                             // (per device: set on every launch)
    const Cols cc = cols_of(a.Cout);
    const int tiles_per_frame = (a.L + kRows - 1) / kRows;
    const dim3 grid((unsigned)(a.B * tiles_per_frame), (unsigned)cc.ntiles);
    train_conv_tf32_kernel<KS, MODE, NT><<<grid, 256, smem, st>>>(a, cc.npad, (a.Cin + kChunk - 1) / kChunk, tiles_per_frame);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

template <int KS, int MODE>
int launch_conv_nt(const ConvArgs &a, cudaStream_t st)
{
    switch (cols_of(a.Cout).nt) {
    case 1: return launch_conv<KS, MODE, 1>(a, st);
    case 2: return launch_conv<KS, MODE, 2>(a, st);
    case 3: return launch_conv<KS, MODE, 3>(a, st);
    default: return launch_conv<KS, MODE, 4>(a, st);
    }
}

template <int KS, int MODE>
int launch_wgrad(const ConvArgs &a, const float *dz, float *dw, cudaStream_t st, bool slices)
{
    constexpr int smem = (2 + 2 * kTapGroup) * kAtomBytes + 1024;
    auto kern = slices ? train_wgrad_tf32_kernel<KS, MODE, true> : train_wgrad_tf32_kernel<KS, MODE, false>;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return -1;
    const WgradGrid g = wgrad_grid_tf32(a.B, a.L, a.Cin, a.Cout, KS);
    kern<<<g.grid, 128, smem, st>>>(a, dz, dw, (a.L + kWgPos - 1) / kWgPos);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace

// CTA = 64 co x 5 taps x 64 ci (97 KB of shared memory: two CTAs per SM); the (frame, 64-position) items are split over gridDim.z
WgradGrid wgrad_grid_tf32(int B, int L, int Cin, int Cout, int ksize)
{
    const int ntg = ksize / kTapGroup, nco = (Cout + 63) / 64, nci = (Cin + 63) / 64;
    const int items = B * ((L + kWgPos - 1) / kWgPos);
    const int base = nco * ntg * nci;
    const int slices = std::max(1, std::min(items, (2 * 132 + base - 1) / base));           // about two CTAs per SM
    return WgradGrid{dim3((unsigned)(nco * ntg), (unsigned)nci, (unsigned)slices), items, kWgPos};
}

size_t train_tf32_packed_elems(int cout, int cin, int k) { return (size_t)((cin + kChunk - 1) / kChunk) * k * cols_of(cout).npad * kChunk; }

int train_tf32_pack(const float *w, float *wf, float *wb, int Cout, int Cin, int K, cudaStream_t st)
{
    const long long nf = (long long)train_tf32_packed_elems(Cout, Cin, K), nb = (long long)train_tf32_packed_elems(Cin, Cout, K);
    train_tf32_pack_kernel<<<(unsigned)((nf + nb + 255) / 256), 256, 0, st>>>(w, wf, wb, Cout, Cin, K, cols_of(Cout).npad,
                                                                                cols_of(Cin).npad, nf, nb);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_conv_tf32(const ConvArgs &a, int ksize, int mode, cudaStream_t st)
{
    if (ksize == 15 && mode == SRC_DIRECT) return launch_conv_nt<15, SRC_DIRECT>(a, st);
    if (ksize == 15 && mode == SRC_DECIM) return launch_conv_nt<15, SRC_DECIM>(a, st);
    if (ksize == 5 && mode == SRC_DIRECT) return launch_conv_nt<5, SRC_DIRECT>(a, st);
    if (ksize == 5 && mode == SRC_UPCAT) return launch_conv_nt<5, SRC_UPCAT>(a, st);
    return -1;
}

int launch_wgrad_tf32(const ConvArgs &a, const float *dz, float *dw, int ksize, int mode, cudaStream_t st, bool slices)
{
    if (ksize == 15 && mode == SRC_DIRECT) return launch_wgrad<15, SRC_DIRECT>(a, dz, dw, st, slices);
    if (ksize == 15 && mode == SRC_DECIM) return launch_wgrad<15, SRC_DECIM>(a, dz, dw, st, slices);
    if (ksize == 5 && mode == SRC_UPCAT) return launch_wgrad<5, SRC_UPCAT>(a, dz, dw, st, slices);
    return -1;
}

}  // namespace wunet
