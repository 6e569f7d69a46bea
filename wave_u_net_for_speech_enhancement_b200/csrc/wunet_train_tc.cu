// wunet_train_tc.cu — bf16 tensor-core convolutions of the training step (Model(train_precision="bf16"), DESIGN.md §5.4).
//
// Arithmetic: the operands of the three convolution-shaped passes (block input, weights, dz) are rounded to bf16 (round to
// nearest) and the products are accumulated in fp32 by sm_90a wgmma; everything around them (z, BatchNorm, the adjoints of
// decimation / interpolation / concat, all gradients) stays fp32 in wunet_train.cu, over the same fp32 NCL workspace.
//
//   train_conv_tc_kernel    implicit-GEMM conv with a linear epilogue, out = conv(in, w) * scale + shift, the interface of
//                           launch_conv_fp32: the forward conv (z, modes DIRECT / DECIM / UPCAT) and the input gradient (DIRECT
//                           over dz with the transposed, flipped weights). M = 128 output positions of one frame, N = Cout
//                           (16 .. 64 columns per CTA), K = 64-channel chunks x taps. All 256 threads stage the operand tile:
//                           the block input is read from fp32 NCL (decimation / interpolation + concat as in fetch_src), rounded
//                           to bf16 and written K-major as 128B-swizzled [position][64 channels] rows, so a tap is the A
//                           descriptor advanced by one 128-byte row. The weights come pre-packed in bf16 (train_tc_pack_kernel)
//                           and are staged five taps at a time. Each of the two warpgroups owns one m64 half of the tile.
//   train_wgrad_tc_kernel   dW[co][ci][k] = sum_{b,l} dz[b][co][l] in(b, ci, l + k - pad): per tap a GEMM with M = co, N = ci
//                           and K = (b, l). The tap shift lies along K, so both operands are staged channels-last, dz as
//                           [position][64 co] and the input as [position][64 ci] (128B-swizzled), and fed MN-major
//                           (imm-trans = 1): a tap advances the B descriptor by one 128-byte row, exactly as in the forward. A
//                           CTA owns 64 co x 64 ci x 5 taps (160 accumulator registers per thread); the (frame, 64-position)
//                           chunks are split over gridDim.z and combined with fp32 atomicAdd or, in deterministic mode,
//                           stored per slice and summed in slice order by wunet_train.cu.
//
// Tiles never straddle two frames: a tile's rows past the frame end are computed and discarded, and positions outside
// [0, L) read as zero (Conv1d padding, per frame), so frames shorter than a tile (the bottom of the U) are padded, never packed.
#include "wunet_common.cuh"
#include "wunet_wgmma.cuh"

#include <algorithm>

namespace wunet {

namespace {

constexpr int kRows = 128;        // output positions per forward tile (two m64 halves, one per warpgroup)
constexpr int kTapGroup = 5;      // taps per staged weight group / per weight-gradient CTA (both kernel sizes are multiples)
constexpr int kWgPos = 64;        // positions per weight-gradient K chunk (four K16 steps)

// descriptor words of a 128B-swizzled operand: hi = SBO(1024 B) | SWIZZLE_128B; lo = (addr >> 4) | LBO << 16. K-major operands
// ignore LBO; the MN-major ones of the weight gradient hold exactly one 64-element atom along M / N, so LBO is never
// followed either (set to 1024 B all the same).
constexpr uint32_t kDescHi = (uint32_t)(1024 >> 4) | (1u << 30);
__device__ __forceinline__ uint32_t desc_lo(uint32_t addr) { return ((addr >> 4) & 0x3FFFu) | ((uint32_t)(1024 >> 4) << 16); }

// byte offset of (row, channel pair 2 cp) in a [rows][64 bf16] 128B-swizzled tile whose base is 1024-byte aligned
__device__ __forceinline__ uint32_t swz(int row, int ch) { return (uint32_t)(row * 128 + ((((ch >> 3) ^ row) & 7) << 4) + (ch & 7) * 2); }

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

template <int KS, int MODE, int NT>
__global__ void __launch_bounds__(256, 2) train_conv_tc_kernel(const ConvArgs a, int npad, int nchunks, int tiles_per_frame)
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
    const __nv_bfloat16 *wpk = reinterpret_cast<const __nv_bfloat16 *>(a.wp);
    const uint32_t a_lo = desc_lo(smem_u32(sa) + (uint32_t)wg * 64 * 128), b_lo = desc_lo(smem_u32(sb));
    float acc[NT * 8];
#pragma unroll
    for (int j = 0; j < NT * 8; ++j) acc[j] = 0.f;
    for (int c = 0; c < nchunks; ++c) {
        __syncthreads();                                       // both warpgroups are done with the previous chunk's tiles
        for (int i = tid; i < AROWS * 32; i += 256) {
            const int r = i % AROWS, ch = 2 * (i / AROWS), ci = c * 64 + ch, l = l0 - PAD + r;
            const bool rok = r < kRows + KS - 1;
            const float v0 = (rok && ci < a.Cin) ? fetch_src<MODE>(a, b, ci, l) : 0.f;
            const float v1 = (rok && ci + 1 < a.Cin) ? fetch_src<MODE>(a, b, ci + 1, l) : 0.f;
            *reinterpret_cast<uint32_t *>(sa + swz(r, ch)) = pack_bf16(v0, v1);
        }
        for (int g = 0; g < NG; ++g) {
            if (g > 0) __syncthreads();                        // the previous weight group has been consumed
            const __nv_bfloat16 *src = wpk + ((size_t)c * KS + g * kTapGroup) * npad * 64;
            for (int i = tid; i < kTapGroup * NT * 16 * 8; i += 256) {
                const int v = i & 7, row = (i >> 3) % (NT * 16), tt = (i >> 3) / (NT * 16);
                const uint4 val = __ldg(reinterpret_cast<const uint4 *>(src + ((size_t)tt * npad + n0 + row) * 64) + v);
                *reinterpret_cast<uint4 *>(sb + tt * TAP_BYTES + swz(row, 8 * v)) = val;
            }
            fence_proxy_async();
            __syncthreads();
            wgmma_fence();
#pragma unroll
            for (int tt = 0; tt < kTapGroup; ++tt)
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    wgmma_m64nNk16<16 * NT>(acc, a_lo + (uint32_t)(g * kTapGroup + tt) * 8u + 2u * k,   // tap: +128 B, K16: +32 B
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
__global__ void __launch_bounds__(128) train_wgrad_tc_kernel(const ConvArgs a, const float *__restrict__ dz, float *__restrict__ dw,
                                                             int chunks_per_frame)
{
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
    const int items = a.B * chunks_per_frame;
    for (int it = blockIdx.z; it < items; it += gridDim.z) {
        const int b = it / chunks_per_frame, l0 = (it - b * chunks_per_frame) * kWgPos;
        __syncthreads();
        for (int i = tid; i < kWgPos * 32; i += 128) {
            const int p = i % kWgPos, ch = 2 * (i / kWgPos), co = co0 + ch, l = l0 + p;
            const float *dr = dz + ((size_t)b * a.Cout + co) * a.L + l;
            const float v0 = (l < a.L && co < a.Cout) ? __ldg(dr) : 0.f;
            const float v1 = (l < a.L && co + 1 < a.Cout) ? __ldg(dr + a.L) : 0.f;
            *reinterpret_cast<uint32_t *>(sd + swz(p, ch)) = pack_bf16(v0, v1);
        }
        for (int i = tid; i < XROWS * 32; i += 128) {
            const int r = i % XROWS, ch = 2 * (i / XROWS), ci = ci0 + ch, l = l0 - PAD + r;
            const bool rok = r < kWgPos + KS - 1;
            const float v0 = (rok && ci < a.Cin) ? fetch_src<MODE>(a, b, ci, l) : 0.f;
            const float v1 = (rok && ci + 1 < a.Cin) ? fetch_src<MODE>(a, b, ci + 1, l) : 0.f;
            *reinterpret_cast<uint32_t *>(sx + swz(r, ch)) = pack_bf16(v0, v1);
        }
        fence_proxy_async();
        __syncthreads();
        wgmma_fence();
#pragma unroll
        for (int tt = 0; tt < kTapGroup; ++tt)
#pragma unroll
            for (int k = 0; k < 4; ++k)                          // K16 step: 16 position rows = 2048 B in both operands
                wgmma_m64nNk16<64, 1, 1>(acc[tt], d_lo + 128u * k, x_lo + (uint32_t)(t0 + tt) * 8u + 128u * k, kDescHi);
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

// both bf16 packings of a block's weights w[Cout][Cin][K], every step:
//   wf[((c K + t) npad(Cout) + co) 64 + j] = w[co][64 c + j][t]          forward conv: [chunk][tap][Cout rows][64 channels]
//   wb[((c K + t) npad(Cin) + ci) 64 + j]  = w[64 c + j][ci][K-1-t]      input gradient: transposed and flipped
// (zero where the channel or column is padding)
__global__ void train_tc_pack_kernel(const float *__restrict__ w, __nv_bfloat16 *__restrict__ wf, __nv_bfloat16 *__restrict__ wb,
                                     int Cout, int Cin, int K, int npad_f, int npad_b, long long nf, long long nb)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nf) {
        const int j = (int)(i & 63);
        const long long r = i >> 6;
        const int row = (int)(r % npad_f);
        const int ct = (int)(r / npad_f), t = ct % K, c = ct / K;
        const int ci = c * 64 + j;
        wf[i] = __float2bfloat16_rn((row < Cout && ci < Cin) ? w[((size_t)row * Cin + ci) * K + t] : 0.f);
    } else if (i < nf + nb) {
        const long long q = i - nf;
        const int j = (int)(q & 63);
        const long long r = q >> 6;
        const int row = (int)(r % npad_b);
        const int ct = (int)(r / npad_b), t = ct % K, c = ct / K;
        const int co = c * 64 + j;
        wb[q] = __float2bfloat16_rn((row < Cin && co < Cout) ? w[((size_t)co * Cin + row) * K + (K - 1 - t)] : 0.f);
    }
}

template <int KS, int MODE, int NT>
int launch_conv_tc(const ConvArgs &a, cudaStream_t st)
{
    constexpr int AROWS = (kRows + KS - 1 + 7) / 8 * 8;
    constexpr int smem = AROWS * 128 + kTapGroup * NT * 16 * 128 + 1024;
    if (cudaFuncSetAttribute(train_conv_tc_kernel<KS, MODE, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
        return -1;                                             // (per device: set on every launch)
    const Cols cc = cols_of(a.Cout);
    const int tiles_per_frame = (a.L + kRows - 1) / kRows;
    const dim3 grid((unsigned)(a.B * tiles_per_frame), (unsigned)cc.ntiles);
    train_conv_tc_kernel<KS, MODE, NT><<<grid, 256, smem, st>>>(a, cc.npad, (a.Cin + 63) / 64, tiles_per_frame);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

template <int KS, int MODE>
int launch_conv_tc_nt(const ConvArgs &a, cudaStream_t st)
{
    switch (cols_of(a.Cout).nt) {
    case 1: return launch_conv_tc<KS, MODE, 1>(a, st);
    case 2: return launch_conv_tc<KS, MODE, 2>(a, st);
    case 3: return launch_conv_tc<KS, MODE, 3>(a, st);
    default: return launch_conv_tc<KS, MODE, 4>(a, st);
    }
}

template <int KS, int MODE>
int launch_wgrad_tc(const ConvArgs &a, const float *dz, float *dw, cudaStream_t st, bool slices)
{
    constexpr int XROWS = (kWgPos + KS - 1 + 7) / 8 * 8;
    constexpr int smem = (kWgPos + XROWS) * 128 + 1024;
    const WgradGrid g = wgrad_grid_bf16(a.B, a.L, a.Cin, a.Cout, KS);
    const int cpf = (a.L + kWgPos - 1) / kWgPos;
    if (slices) train_wgrad_tc_kernel<KS, MODE, true><<<g.grid, 128, smem, st>>>(a, dz, dw, cpf);
    else train_wgrad_tc_kernel<KS, MODE, false><<<g.grid, 128, smem, st>>>(a, dz, dw, cpf);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

}  // namespace

// CTA = 64 co x 5 taps x 64 ci; the (frame, 64-position chunk) items are split over gridDim.z
WgradGrid wgrad_grid_bf16(int B, int L, int Cin, int Cout, int ksize)
{
    const int ntg = ksize / kTapGroup, nco = (Cout + 63) / 64, nci = (Cin + 63) / 64;
    const int items = B * ((L + kWgPos - 1) / kWgPos);
    const int base = nco * ntg * nci;
    const int slices = std::max(1, std::min(items, (2 * 132 + base - 1) / base));           // about two CTAs per SM
    return WgradGrid{dim3((unsigned)(nco * ntg), (unsigned)nci, (unsigned)slices), items, kWgPos};
}

size_t train_tc_packed_elems(int cout, int cin, int k) { return (size_t)((cin + 63) / 64) * k * cols_of(cout).npad * 64; }

int train_tc_pack(const float *w, __nv_bfloat16 *wf, __nv_bfloat16 *wb, int Cout, int Cin, int K, cudaStream_t st)
{
    const long long nf = (long long)train_tc_packed_elems(Cout, Cin, K), nb = (long long)train_tc_packed_elems(Cin, Cout, K);
    train_tc_pack_kernel<<<(unsigned)((nf + nb + 255) / 256), 256, 0, st>>>(w, wf, wb, Cout, Cin, K, cols_of(Cout).npad,
                                                                              cols_of(Cin).npad, nf, nb);
    return cudaGetLastError() == cudaSuccess ? 1 : -1;
}

int launch_conv_bf16(const ConvArgs &a, int ksize, int mode, cudaStream_t st)
{
    if (ksize == 15 && mode == SRC_DIRECT) return launch_conv_tc_nt<15, SRC_DIRECT>(a, st);
    if (ksize == 15 && mode == SRC_DECIM) return launch_conv_tc_nt<15, SRC_DECIM>(a, st);
    if (ksize == 5 && mode == SRC_DIRECT) return launch_conv_tc_nt<5, SRC_DIRECT>(a, st);
    if (ksize == 5 && mode == SRC_UPCAT) return launch_conv_tc_nt<5, SRC_UPCAT>(a, st);
    return -1;
}

int launch_wgrad_bf16(const ConvArgs &a, const float *dz, float *dw, int ksize, int mode, cudaStream_t st, bool slices)
{
    if (ksize == 15 && mode == SRC_DIRECT) return launch_wgrad_tc<15, SRC_DIRECT>(a, dz, dw, st, slices);
    if (ksize == 15 && mode == SRC_DECIM) return launch_wgrad_tc<15, SRC_DECIM>(a, dz, dw, st, slices);
    if (ksize == 5 && mode == SRC_UPCAT) return launch_wgrad_tc<5, SRC_UPCAT>(a, dz, dw, st, slices);
    return -1;
}

}  // namespace wunet
