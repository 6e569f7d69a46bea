// wunet_tc.cu — bf16 tensor-core path of the Wave-U-Net forward for sm_90a (wgmma + TMA + mbarrier).
//
// Data layout in HBM: every activation is channels-last bf16, [B][L][C] ("NLC"), C = the reference's
// channel count (24*m). A Conv1d tap shift is then a whole-row shift of the operand tile.
//
// Each conv block (reference: [decimate | interpolate+cat] -> Conv1d -> BatchNorm1d(eval) -> LeakyReLU,
// model/unet_basic.py:83-86, :93-96, :10-13, :23-26) is ONE kernel, an implicit GEMM
//     D[position, cout] = sum_taps sum_cin  X[position + tap - pad, cin] * W[tap][cout, cin]
// with M = 128 output positions per CTA tile, N = Cout (padded to 16, split over CTAs beyond the register budget) and the
// K loop running over 64-channel chunks x taps:
//   * the input tile (128 + K-1 rows x 64 channels, 128B-swizzled) is loaded ONCE per chunk by TMA;
//     out-of-range rows/channels are zero-filled by TMA = Conv1d zero padding, per frame;
//     every tap reuses it through a wgmma shared-memory descriptor whose start address is advanced by tap*128 B;
//   * encoder decimation o[:, :, ::2] is a tensor map with a doubled row stride (no copy);
//   * decoder: the K axis is [upsampled previous output | skip]. The skip half comes by TMA; the upsampled
//     half (F.interpolate linear, align_corners=True, index math in fp32 like ATen) is produced by the producer
//     warps straight into the swizzled operand tile — the interpolated/concatenated tensor never exists in HBM;
//   * weights come by TMA: either a ring of stages holding several taps of one [N x 64] chunk each, or — where the whole
//     packed weight set of the block fits next to the input ring — loaded once per persistent CTA;
//   * accumulators are registers of the consumer warpgroups that issue the wgmma; after the K loop the same threads apply
//     the folded BatchNorm scale/shift and LeakyReLU(0.1) and store bf16 NLC rows; the last decoder block also
//     applies the 1x1 conv over [decoder out | raw input] and tanh (model/unet_basic.py:98-99) so its 24-channel
//     output never reaches HBM.
//   * frames shorter than 128 samples (the bottom of the U) are packed several per tile with their own halo
//     rows; rows that straddle two frames are computed and discarded.
// Warp roles: consumer warpgroups (wgmma + epilogue), upsample-producer warps (decoder blocks), one TMA warp. Two kernel
// flavours per block type: "large" (one CTA per SM, two consumer warpgroups + 4 producer warps, up to 128 columns) and
// "small" (two CTAs per SM: one consumer warpgroup + 4 producer warps, up to 64 columns, half the shared memory), so that
// one CTA's pipeline bubbles are filled by the other's MMAs. build_plan() chooses tile shapes, ring depths and the flavour
// per block.
#include "wunet_tc.cuh"
#include "wunet_common.cuh"
#include "wunet_wgmma.cuh"

#include <cuda.h>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <map>
#include <string>
#include <vector>

namespace wunet {

namespace {

thread_local char g_tc_err[512] = "";
int tc_fail(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_tc_err, sizeof(g_tc_err), fmt, ap);
    va_end(ap);
    return -1;
}

constexpr int kEpiWarpsLarge = 8;                 // "large" flavour: two consumer warpgroups (one m64 half of the tile each) ...
constexpr int kProducerWarpsLarge = 4;            // ... plus four upsample-producer warps in decoder blocks (one item per thread)
constexpr int kEpiWarpsSmall = 4;                 // "small" flavour (two CTAs per SM): one consumer warpgroup (both m64 halves),
constexpr int kProducerWarpsSmall = 4;            // four producer warps
constexpr int kAccColsLarge = 128;                // accumulator columns per CTA: 64 fp32 registers per consumer thread in
constexpr int kAccColsSmall = 64;                 // either flavour
constexpr int kSmemLimitSmall = 113 * 1024;       // 2 x (dynamic + 1 KB reserved) <= 228 KB per SM
constexpr int kMaxBStages = 8;
constexpr int kSmemLimit = 227 * 1024;

inline int round_up(int v, int a) { return (v + a - 1) / a * a; }
inline size_t round_up_sz(size_t v, size_t a) { return (v + a - 1) / a * a; }

// -------------------------------------------------------------------------------------------------
// device helpers (raw PTX; forms taken from the PTX ISA as shipped in CUDA 12.9). smem_u32, pack_bf16 and the wgmma forms
// are in wunet_wgmma.cuh (shared with the training kernels).
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
// Waiting on an mbarrier phase. try_wait suspends the thread in hardware only for a short, system-defined time, so a plain
// retry loop is a hot spin that competes with the working roles for issue slots. With a suspend-time hint ptxas emits a
// sleep until the barrier's phase flips or the time is up. WUNET_WAIT_NS: hint in ns for every role; 0 = no hint.
#ifndef WUNET_WAIT_NS
#define WUNET_WAIT_NS 0
#endif
template <int NS>
__device__ __forceinline__ void mbar_wait_ns(uint32_t bar, uint32_t parity)
{
    uint32_t ok;
    do {
        if (NS > 0)
            asm volatile(
                "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\tselp.b32 %0, 1, 0, p;\n\t}"
                : "=r"(ok) : "r"(bar), "r"(parity), "r"((uint32_t)NS) : "memory");
        else
            asm volatile(
                "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
                : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) { mbar_wait_ns<WUNET_WAIT_NS>(bar, parity); }
__device__ __forceinline__ bool mbar_test(uint32_t bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1, int c2)
{
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// NK K16 steps x MB m64 row blocks of one operand pair, each one m64n(16 NT)k16 over all of the CTA's columns, issued back to
// back. acc[mb] is row block mb's fragment (columns past 16 NT untouched); a_lo addresses K step 0 of row block 0 (row blocks
// are 64 rows = 512 x 16 B apart), b_lo K step 0 of the [16 NT rows x 64] weight tile; a K16 step is +32 B in both. Straight-line
// code: ptxas serialises the wgmmas (waits for each one) when a branch it cannot prove warpgroup-uniform sits among them.
template <int NT, int NK, int MB, int ACC>
__device__ __forceinline__ void wgmma_batch(float (&acc)[MB][ACC], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
{
    static_assert(8 * NT <= ACC, "accumulator fragment narrower than the MMA");
#pragma unroll
    for (int k = 0; k < NK; ++k)
#pragma unroll
        for (int mb = 0; mb < MB; ++mb)
            wgmma_m64nNk16<16 * NT>(*reinterpret_cast<float (*)[8 * NT]>(&acc[mb][0]), a_lo + (uint32_t)(mb * 512 + 2 * k),
                                    b_lo + (uint32_t)(2 * k), hi);
}
// NTAP consecutive taps of wgmma_batch: tap t reads the A rows one 128-byte row further down (+8 in descriptor units) and the
// weight tile b_step (descriptor units) further on, in the same order as NTAP separate batches.
template <int NT, int NK, int NTAP, int MB, int ACC>
__device__ __forceinline__ void wgmma_batch_taps(float (&acc)[MB][ACC], uint32_t a_lo, uint32_t b_lo, uint32_t b_step, uint32_t hi)
{
#pragma unroll
    for (int t = 0; t < NTAP; ++t) wgmma_batch<NT, NK>(acc, a_lo + (uint32_t)t * 8u, b_lo + (uint32_t)t * b_step, hi);
}
// wgmma_batch_taps for run-time nt = columns / 16 (1 .. ACC / 8) and nk (1 .. 4): one fence, the batch, one commit (one wgmma
// group). The dispatch branches lie outside the fence ... commit region.
template <int MB, int ACC, int NTAP = 1, int NT = ACC / 8>
__device__ __forceinline__ void wgmma_group(int nt, int nk, float (&acc)[MB][ACC], uint32_t a_lo, uint32_t b_lo, uint32_t hi,
                                            uint32_t b_step = 0)
{
    if (NT == 1 || nt == NT) {
        switch (nk) {
        case 1: wgmma_fence(); wgmma_batch_taps<NT, 1, NTAP>(acc, a_lo, b_lo, b_step, hi); wgmma_commit(); break;
        case 2: wgmma_fence(); wgmma_batch_taps<NT, 2, NTAP>(acc, a_lo, b_lo, b_step, hi); wgmma_commit(); break;
        case 3: wgmma_fence(); wgmma_batch_taps<NT, 3, NTAP>(acc, a_lo, b_lo, b_step, hi); wgmma_commit(); break;
        default: wgmma_fence(); wgmma_batch_taps<NT, 4, NTAP>(acc, a_lo, b_lo, b_step, hi); wgmma_commit(); break;
        }
    } else if constexpr (NT > 1) {
        wgmma_group<MB, ACC, NTAP, NT - 1>(nt, nk, acc, a_lo, b_lo, hi, b_step);
    }
}
// wgmma_group for run-time ntap (1 .. NTAP) consecutive taps. Each wgmma group costs a fixed few hundred cycles on top of its
// MMAs (per-role trace, H100), which dominated the narrow decoder blocks when every tap was a group of its own.
constexpr int kMaxGroupTaps = 5;
template <int MB, int ACC, int NTAP = kMaxGroupTaps>
__device__ __forceinline__ void wgmma_group_taps(int ntap, int nt, int nk, float (&acc)[MB][ACC], uint32_t a_lo, uint32_t b_lo,
                                                 uint32_t hi, uint32_t b_step)
{
    if (NTAP == 1 || ntap == NTAP) wgmma_group<MB, ACC, NTAP>(nt, nk, acc, a_lo, b_lo, hi, b_step);
    else if constexpr (NTAP > 1) wgmma_group_taps<MB, ACC, NTAP - 1>(ntap, nt, nk, acc, a_lo, b_lo, hi, b_step);
}
__device__ __forceinline__ void st_shared_v4_if(uint32_t addr, const uint4 &v, bool pred)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %5, 0;\n\t@p st.shared.v4.b32 [%0], {%1, %2, %3, %4};\n\t}"
                 ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"((uint32_t)pred) : "memory");
}
__device__ __forceinline__ uint4 ld_shared_v4(uint32_t addr)
{
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}
#ifdef WUNET_TC_TRACE
#define TRACE(role, idx)                                                                      \
    do {                                                                                      \
        if (p.trace != nullptr && blockIdx.x == 0 && (idx) < 512) p.trace[(role) * 512 + (idx)++] = clock64(); \
    } while (0)
#else
#define TRACE(role, idx) do { } while (0)
#endif
__device__ __forceinline__ float lrelu(float v) { return fmaxf(v, kLreluSlope * v); }   // == v >= 0 ? v : slope * v (0 < slope < 1)
// tanh(x) = 1 - 2 / (exp(2x) + 1); saturates correctly at +-inf, abs error ~1e-6 (bf16 path only)
__device__ __forceinline__ float tanh_fast(float x) { return 1.f - __fdividef(2.f, __expf(2.f * x) + 1.f); }

}  // namespace

// -------------------------------------------------------------------------------------------------
// kernel parameters
// -------------------------------------------------------------------------------------------------
struct TcParams {
    // problem
    int B, L, Cout, T;
    int Cin0, Cin1;            // K segments: ENC: Cin0 = Cin, Cin1 = 0; DEC: Cin0 = upsampled prev, Cin1 = skip
    int nchunks0, nchunks;     // 64-channel chunks in segment 0 / in total
    unsigned char chunk_map[48]; // K-loop order: bit 7 = chunk of the upsampled segment, bits 0-4 = chunk index inside its segment;
                                 // bit 6: merged tail chunk (MG kernels) / low-part data (split-precision kernels); bit 5 (split
                                 // precision): the position re-uses the operand stage of the position before it
    // N tiling
    int Npad, Nh, Nstride;     // padded Cout, columns per CTA, column stride between sub-tile accumulators
    // M tiling
    int MT, packed, S, FR, tiles_per_frame;
    int m_tiles, nsplit, nacc; // M tiles in the problem, N halves, accumulator buffers (1)
    int tile_begin, tile_end;  // tiles [begin, end) handled by this launch (sub-ranges = batch chunks of the host pipeline)
    int nops, R1, a_tx_bytes;  // TMA ops per A chunk, rows advanced per op, bytes per chunk
    int rows_used;             // smem rows the producers must fill (upsample path)
    uint32_t a_stage_bytes, b_stage_bytes;
    int nb;                    // B ring depth
    int na;                    // A stages (1 or 2)
    int tg, ngroups;           // taps per weight stage, stages per chunk (= ceil(KS / tg))
    int n_epi;                 // consumer warps of this kernel flavour
    int bulk_store;            // always 0: the epilogue stores straight from the accumulator fragments
    int resident;              // 1: all weight tiles of the block stay in shared memory for the CTA's lifetime (no ring)
    uint32_t tmem_cols;
    // operands
    const __nv_bfloat16 *prev; // DEC: previous block output [B][L/2][Cin0]
    int Lin;
    float up_scale;
    const float2 *ss;          // [Npad] (scale, shift)
    __nv_bfloat16 *out;        // [B][L][Cout] or nullptr (fused head without debug store)
    // fused head (last decoder): y = tanh(out_w[:C] . v + out_w[C] * x + out_b)
    int head;
    const float *x;            // [B][T] raw input
    float *y;                  // [B][T]
    const float *head_w;       // [C+1]
    const float *head_b;       // [1]
    long long *trace;          // WUNET_TC_TRACE builds: per-role clock64 stamps of CTA 0 (development)
    // merged tail chunk (MG = 1 instantiations): the last K chunk of a decoder block is [skip tail (TMA) | upsampled tail
    // (producers)] in ONE stage - one K chunk fewer for dec6 / dec9 / dec10 of the reference architecture
    int pf_late;               // 1 (default): the producers' register prefetch of their next unit is issued when the K loop reaches that unit
                               // (after the TMA chunks in between have been handed on); 0: right after the previous unit's hand-off
    int split;                 // split-precision mode (SP kernels): activations are stored as [hi | lo] bf16 channel halves (2 C channels per
                               // row), the K loop runs [hi data x w_hi | lo data x w_hi | hi data x w_lo] and the epilogue stores hi and lo
    int mg;                    // 1: chunk_map's last entry (0x40) is such a merged chunk
    int mg_vo, mg_nvec;        // first 16-byte vector / number of vectors the producers write in it
    int mg_nk, mg_kslot;       // its K16 steps, its 64-wide slot in the packed weights
    int mg_skip_idx, mg_up_idx;// 64-channel chunk index of the tails inside their segments
    // head-only instantiation (HD = 1): the previous-level rows a tile interpolates between are staged in a shared-memory ring
    // by TMA (tmO = plain [B][Lin][Cin0] view of prev), several tiles ahead of the producers
    int hd;                    // 1: launch the HD instantiation
    int ps_n;                  // ring slots (0 = no ring); entries alternate [previous-level window | skip rows] of a tile
    int ps_rows, ps_rows2;     // box rows of the two entry kinds (previous-level rows / skip rows)
    uint32_t ps_bytes;         // slot pitch (128-byte multiple)
    uint32_t ps_tx, ps_tx2;    // bytes one TMA box of either kind delivers
};

// smem carve-up (offsets from the 1024-aligned base): A stages | B stages | ss | barriers
struct SmemMap {
    uint32_t a, b, ss, stg, ps, bars;
};
__host__ __device__ inline SmemMap smem_map(const TcParams &p)
{
    SmemMap m;
    m.a = 0;
    m.b = p.na * p.a_stage_bytes;
    m.ss = m.b + p.nb * p.b_stage_bytes;
    m.stg = (m.ss + (uint32_t)p.Npad * 8 + 64 * 4 + 1023) & ~1023u;   // after scale/shift + head weights
    m.ps = m.stg;
    m.ps = (m.ps + 127) & ~127u;
    m.bars = m.ps + (uint32_t)p.ps_n * p.ps_bytes;                       // HD: ring of previous-level row windows
    m.bars = (m.bars + 15) & ~15u;
    return m;
}
inline size_t smem_total(const TcParams &p)
{
    return smem_map(p).bars + 8 * (8 + 2 * kMaxBStages + 4) + 16 + ((p.mg || p.ps_n) ? 32 : 0) + (p.ps_n ? 128 : 0) + 1024;
}

// K-loop position c -> (segment, chunk index inside the segment, K16 steps, 64-wide slot in the packed weights)
struct ChunkInfo { bool up; int idx, nk, kslot; bool merged; int vo, nvec; bool lo, reuse; };
template <bool UPCAT, int MG, int SP = 0>
__device__ __forceinline__ ChunkInfo chunk_info(const TcParams &p, int c)
{
    ChunkInfo ci;
    const int m = p.chunk_map[c];
    ci.lo = false; ci.reuse = false;
    if (SP != 0) {                                // split precision: the weight slot is the K-loop position itself
        ci.merged = false;
        ci.up = UPCAT && (m & 0x80);
        ci.lo = (m & 0x40) != 0;
        ci.reuse = (m & 0x20) != 0;                // same operand stage as the position before (hi data x w_lo after hi data x w_hi)
        ci.idx = m & 0x1f;
        const int seg = (ci.up || !UPCAT) ? p.Cin0 - 64 * ci.idx : p.Cin1 - 64 * ci.idx;
        ci.nk = ((seg < 64 ? seg : 64) + 15) >> 4;
        ci.kslot = c;
        ci.vo = 0; ci.nvec = ci.nk * 2;
        return ci;
    }
    if (MG != 0 && UPCAT && (m & 0x40)) {          // merged tail chunk: TMA fills the leading vectors, the producers the next ones
        ci.up = true; ci.merged = true;
        ci.idx = p.mg_up_idx; ci.nk = p.mg_nk; ci.kslot = p.mg_kslot; ci.vo = p.mg_vo; ci.nvec = p.mg_nvec;
        return ci;
    }
    ci.merged = false;
    ci.up = UPCAT && (m & 0x80);
    ci.idx = m & 0x7f;
    const int seg_c = (ci.up || !UPCAT) ? p.Cin0 - 64 * ci.idx : p.Cin1 - 64 * ci.idx;
    ci.nk = ((seg_c < 64 ? seg_c : 64) + 15) >> 4;
    ci.kslot = (ci.up || !UPCAT) ? ci.idx : p.nchunks0 + ci.idx;
    ci.vo = 0; ci.nvec = ci.nk * 2;
    return ci;
}

// -------------------------------------------------------------------------------------------------
// the conv kernel
// -------------------------------------------------------------------------------------------------
// MG = 1: decoder instantiations whose K loop ends in a merged tail chunk (p.mg); MG = 0 everything else (kept in separate
// instantiations so that the code of the validated ones does not change while they are being developed).
// HD = 1: the last decoder block when only the network output is wanted (fused head, the block's own activations are not
// stored; Cout <= 32, one N tile): a straight-line head-only epilogue and 8-row producer items (see the roles below). The
// arithmetic and its order are those of the generic instantiation: bit-identical results.
// PR = 1 ("row-pair" instantiation, round 2 second half): the block is run on PAIRS of positions - operand row m holds positions
// 2m and 2m+1 side by side ([L/2][2 C] is the same memory as [L][C]), the output row their 2 Cout results, and the K = 5 taps
// become 3 taps over row pairs with Toeplitz-expanded weights (pair_weight() below). N doubles (the M=128 MMA of a narrow block
// is bound by its operand reads, 32 + N/4 cycles) and the K loop shrinks; for the decoder the producers write the upsampled
// half as [q0: 32 channels | q1: the same 32 channels] per 64-wide chunk and the fused head produces two samples per row.
template <int KS, bool UPCAT, int EW, int PW, int MG, int SP = 0, int HD = 0, int PR = 0>
__global__ void __launch_bounds__(32 + 32 * (EW + PW), EW == kEpiWarpsSmall ? 2 : 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
               const __grid_constant__ CUtensorMap tmO, const TcParams p)
{
    constexpr int PAD = (KS - 1) / 2;
    constexpr int kProducerWarps = PW;
    constexpr int NPROD = kProducerWarps * 32;
    constexpr int kEpilogueWarps = EW;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t *base_ptr = smem_raw + (base - smem_u32(smem_raw));
    const SmemMap sm = smem_map(p);
    const uint32_t bars = base + sm.bars;
    // barrier slots (8 B each): a_full[4] a_empty[4] b_full[8] b_empty[8] | 5 unused | a_tma[4] | p_full[8] p_empty[8]
    const uint32_t a_full = bars, a_empty = bars + 32, b_full = bars + 64, b_empty = bars + 64 + 8 * kMaxBStages;
    const uint32_t a_tma = bars + 64 + 16 * kMaxBStages + 48;   // [4], MG = 1 kernels (merged tail chunk) only (smem_total reserves them)
    const uint32_t p_full = a_tma + 32, p_empty = a_tma + 96;   // [8] each, HD = 1 kernels only: ring of row windows (see the TMA role)

    // Programmatic dependent launch: let the next block's kernel be scheduled as our CTAs retire, so its prologue (barrier
    // init, descriptor prefetch, resident weight preload) overlaps this kernel's tail.
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // warp roles: consumer warpgroups (wgmma + epilogue) first, so that they are aligned warpgroups, then the upsample producers
    // (decoder blocks) and the TMA warp, the last warp of the launch shape (32 + 32 (EW + PW) threads).
    constexpr int kFirstProducer = kEpilogueWarps;
    constexpr int kTmaWarp = kEpilogueWarps + (UPCAT ? kProducerWarps : 0);
    const int total_tiles = p.tile_end;
    const int first_tile = p.tile_begin + (int)blockIdx.x;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmW)) : "memory");
        for (int s = 0; s < 4; ++s) {
            mbar_init(a_full + 8 * s, HD != 0 ? kProducerWarps : (UPCAT ? 1 + kProducerWarps : 1));
            mbar_init(a_empty + 8 * s, kEpilogueWarps / 4);          // one arrival per consumer warpgroup
        }
        for (int s = 0; s < min(p.nb, kMaxBStages); ++s) { mbar_init(b_full + 8 * s, 1); mbar_init(b_empty + 8 * s, kEpilogueWarps / 4); }
        if (MG != 0 && p.mg)
            for (int s = 0; s < 4; ++s) mbar_init(a_tma + 8 * s, 1);
        if (HD != 0)
            for (int s = 0; s < 8; ++s) { mbar_init(p_full + 8 * s, 1); mbar_init(p_empty + 8 * s, kProducerWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    {   // folded BatchNorm scale/shift of all output columns
        if (HD != 0) {
            // head-only kernel: one float4 per output column {scale, shift, head weight, extra}; extra of column 0 = head bias,
            // of column 1 = head weight of the raw-input channel. Columns past Cout are zero.
            float4 *hp = reinterpret_cast<float4 *>(base_ptr + sm.ss);
            if (threadIdx.x < 32) {
                const int c = threadIdx.x;
                const float2 st = c < p.Npad ? p.ss[c] : make_float2(0.f, 0.f);
                hp[c] = make_float4(st.x, st.y, c < p.Cout ? p.head_w[c] : 0.f, c == 0 ? p.head_b[0] : (c == 1 ? p.head_w[p.Cout] : 0.f));
            }
        } else {
        float2 *ss = reinterpret_cast<float2 *>(base_ptr + sm.ss);
        for (int i = threadIdx.x; i < p.Npad; i += blockDim.x) ss[i] = p.ss[i];
        if (p.head) {
            float *hw = reinterpret_cast<float *>(base_ptr + sm.ss) + 2 * p.Npad;
            const int hc = PR != 0 ? p.Cout >> 1 : p.Cout;            // channels the 1x1 head sums over (row-pair mode: Cout = 2 hc)
            if ((int)threadIdx.x <= hc) hw[threadIdx.x] = p.head_w[threadIdx.x];
            if ((int)threadIdx.x == hc + 1) hw[threadIdx.x] = p.head_b[0];
        }
        }
    }
    __syncthreads();
    const bool pdl_early_weights = p.resident != 0;      // weights do not depend on the previous kernel's output
    if (!(warp == kTmaWarp && pdl_early_weights)) asm volatile("griddepcontrol.wait;" ::: "memory");

    // tile -> (frame / first row, column half)
    auto tile_coords = [&](int tile, int &b0, int &l0, int &n0) {
        const int mi = tile / p.nsplit;
        n0 = (tile - mi * p.nsplit) * p.Nh;
        if (p.packed) { b0 = mi * p.FR; l0 = 0; }
        else { b0 = mi / p.tiles_per_frame; l0 = (mi - b0 * p.tiles_per_frame) * 128 * p.MT; }
    };

    if (warp == kTmaWarp) {
        // ======================= TMA producer =======================
        if (lane == 0) {
            int sa = 0, pa = 0, sb = 0, pb = 0;
            int tr0 = 0; (void)tr0;
            // A tiles are issued one chunk ahead of the weight stream (across tile boundaries)
            int a_tile = first_tile, a_c = 0;
            // returns false if the stage is still in use and blocking == false
            auto issue_a = [&](bool blocking) -> bool {
                if (a_tile >= total_tiles) return true;
                if (!blocking && !mbar_test(a_empty + 8 * sa, pa ^ 1)) return false;
                int b0, l0, n0;
                tile_coords(a_tile, b0, l0, n0);
                const ChunkInfo aci = chunk_info<UPCAT, MG, SP>(p, a_c);
                if (SP != 0 && aci.reuse) {                      // no new operand data: the stage of the previous position is used again
                    if (++a_c == p.nchunks) { a_c = 0; a_tile += gridDim.x; }
                    return true;
                }
                const bool from_tma = !aci.up;
                TRACE(0, tr0);
                mbar_wait(a_empty + 8 * sa, pa ^ 1);
                TRACE(0, tr0);
                if (from_tma) {
                    const int cc = aci.idx;
                    const int lcoord = p.packed ? -PAD : l0 - PAD;
                    mbar_expect_tx(a_full + 8 * sa, p.a_tx_bytes);
                    for (int op = 0; op < p.nops; ++op)
                        tma_load_3d(base + sm.a + sa * p.a_stage_bytes + op * p.R1 * 128, &tmA, a_full + 8 * sa,
                                    cc * 64 + ((SP != 0 && aci.lo) ? (UPCAT ? p.Cin1 : p.Cin0) : 0),      // low part: second channel half
                                    lcoord + op * p.R1, b0);

                } else if (MG != 0 && aci.merged) {
                    // skip tail by TMA into the leading vectors of the stage (zero fill behind it), completion on a_tma: the
                    // producers add the upsampled tail once it has landed and complete a_full
                    const int lcoord = l0 - PAD;
                    mbar_expect_tx(a_tma + 8 * sa, p.a_tx_bytes);
                    for (int op = 0; op < p.nops; ++op)
                        tma_load_3d(base + sm.a + sa * p.a_stage_bytes + op * p.R1 * 128, &tmA, a_tma + 8 * sa, p.mg_skip_idx * 64,
                                    lcoord + op * p.R1, b0);
                    mbar_arrive(a_full + 8 * sa);
                } else {
                    mbar_arrive(a_full + 8 * sa);
                }
                if (++sa == p.na) { sa = 0; pa ^= 1; }
                if (++a_c == p.nchunks) { a_c = 0; a_tile += gridDim.x; }
                return true;
            };
            if (p.resident) {
                // the whole packed weight set of this block (nchunks x KS tiles of [Nh x 64]) is loaded once per CTA
                mbar_expect_tx(b_full, (uint32_t)p.nchunks * p.ngroups * p.tg * p.Nh * 128);
                for (int c = 0; c < p.nchunks; ++c) {
                    const int kslot = chunk_info<UPCAT, MG, SP>(p, c).kslot;
                    for (int g = 0; g < p.ngroups; ++g)
                        tma_load_3d(base + sm.b + (uint32_t)(c * p.ngroups + g) * p.b_stage_bytes, &tmW, b_full, kslot * 64, 0, g * p.tg);
                }
                asm volatile("griddepcontrol.wait;" ::: "memory");        // activations of the previous block from here on
            }
            if (HD != 0) {
                // head-only instantiation: BOTH operand chunks are written by the producer warps; this lane only feeds them. Per
                // tile two ring entries, in K-loop order: the window of previous-level rows the upsampled chunk interpolates
                // between (rows (l0 - PAD)/2 - 1 ..., tmO = plain [B][Lin][Cin0] view) and the tile's skip rows (l0 - PAD ...,
                // tmA = plain [B][L][Cin1] view; rows outside the frame are zero-filled = Conv1d padding). The lane runs as far
                // ahead as the ring has free slots (ps_n entries), so the DRAM latency of neither stream reaches the producers.
                int ps_i = 0, ps_par = 0;
                for (int tile = first_tile; tile < total_tiles; tile += gridDim.x) {
                    int b0, l0, n0;
                    tile_coords(tile, b0, l0, n0);
                    for (int half = 0; half < 2; ++half) {
                        TRACE(0, tr0);
                        mbar_wait(p_empty + 8 * ps_i, ps_par ^ 1);
                        TRACE(0, tr0);
                        const uint32_t dsts = base + sm.ps + (uint32_t)ps_i * p.ps_bytes;
                        if (half == 0) {
                            mbar_expect_tx(p_full + 8 * ps_i, p.ps_tx);
                            tma_load_3d(dsts, &tmO, p_full + 8 * ps_i, 0, ((l0 - PAD) >> 1) - 1, b0);
                        } else {
                            mbar_expect_tx(p_full + 8 * ps_i, p.ps_tx2);
                            tma_load_3d(dsts, &tmA, p_full + 8 * ps_i, 0, l0 - PAD, b0);
                        }
                        if (++ps_i == p.ps_n) { ps_i = 0; ps_par ^= 1; }
                    }
                }
            } else {
            for (int pre = 0; pre < p.na - 1; ++pre) issue_a(true);          // A tiles run na-1 chunks ahead of the weights
            if (p.na == 1) issue_a(true);
            for (int tile = first_tile; tile < total_tiles; tile += gridDim.x) {
                int b0, l0, n0;
                tile_coords(tile, b0, l0, n0);
                for (int c = 0; c < p.nchunks; ++c) {
                    // the weight groups of this chunk go out as soon as their ring slots free up; the A tile of the NEXT
                    // chunk is slipped in between them the moment its stage is released (it never blocks the weights)
                    bool a_done = false;
                    const int kslot = chunk_info<UPCAT, MG, SP>(p, c).kslot;
                    for (int g = 0; g < (p.resident ? 0 : p.ngroups); ++g) {
                        if (!a_done) a_done = issue_a(false);
                        mbar_wait(b_empty + 8 * sb, pb ^ 1);
                        TRACE(0, tr0);
                        mbar_expect_tx(b_full + 8 * sb, p.Nh * 128 * p.tg);          // taps past KS are zero-filled by TMA
                        tma_load_3d(base + sm.b + sb * p.b_stage_bytes, &tmW, b_full + 8 * sb, kslot * 64, n0, g * p.tg);
                        if (++sb == p.nb) { sb = 0; pb ^= 1; }
                    }
                    if (!a_done) issue_a(true);
                }
            }
            }
        }
    } else if (warp < kEpilogueWarps) {
        // ======================= consumer warpgroups: wgmma + epilogue =======================
        // The tile's 128 rows are split into m64 blocks over the warpgroups (large flavour: one block each, small: two); every
        // warpgroup runs the whole K loop for its rows with the accumulators in registers, each MMA as wide as the CTA's
        // columns, releases each operand stage once its wgmma groups have completed, then applies BatchNorm + LeakyReLU
        // straight from the fragments.
        // Fragment of m64nNk16 (f32): thread (warp wq, lane) holds rows 16 wq + lane / 4 (+8) and columns 2 (lane % 4) (+1) of
        // every 8-column group.
        constexpr int NWG = kEpilogueWarps / 4;
        constexpr int MB = 2 / NWG;
        constexpr int NB = (kEpilogueWarps == kEpiWarpsSmall ? kAccColsSmall : kAccColsLarge) / 16;
        const int wg = warp >> 2, wq = warp & 3;
        const bool wg_leader = (threadIdx.x & 127) == 0;
        const float2 *ss = reinterpret_cast<const float2 *>(base_ptr + sm.ss);
        const float *hw = reinterpret_cast<const float *>(base_ptr + sm.ss) + 2 * p.Npad;   // head: [C+1] weights, bias
        const uint32_t tile_bytes = (uint32_t)p.Nh * 128;
        const uint32_t b_step = tile_bytes >> 4;
        // descriptor words: hi = SBO(1024 B) | SWIZZLE_128B, lo = (addr >> 4) | LBO(1)
        const uint32_t hi = (uint32_t)(1024 >> 4) | (1u << 30);
        int sa = 0, pa = 0, sb = 0, pb = 0;
        int tr1 = 0, tr2 = 0; (void)tr1; (void)tr2;
        if (p.resident) mbar_wait(b_full, 0);
        for (int tile = first_tile; tile < total_tiles; tile += gridDim.x) {
            int b0, l0, n0;
            tile_coords(tile, b0, l0, n0);
            const int nt = min(p.Nh, p.Npad - n0) >> 4;     // 16-column blocks of this CTA (the last column split may be narrower)
            float acc[MB][8 * NB];
#pragma unroll
            for (int mb = 0; mb < MB; ++mb)
#pragma unroll
                for (int j = 0; j < 8 * NB; ++j) acc[mb][j] = 0.f;
            for (int c = 0; c < p.nchunks; ++c) {
                const ChunkInfo mci = chunk_info<UPCAT, MG, SP>(p, c);
                const int nk = mci.nk;
                if (threadIdx.x == 0) TRACE(1, tr1);
                if (!(SP != 0 && mci.reuse)) mbar_wait(a_full + 8 * sa, pa);
                if (threadIdx.x == 0) TRACE(1, tr1);
                const uint32_t a_base = base + sm.a + sa * p.a_stage_bytes + (uint32_t)(wg * MB * 64 * 128);
                const uint32_t a_lo0 = ((a_base >> 4) & 0x3FFFu) | (1u << 16);
                for (int g = 0; g < p.ngroups; ++g) {
                    uint32_t b_base;
                    if (p.resident) {
                        b_base = base + sm.b + (uint32_t)(c * p.ngroups + g) * p.b_stage_bytes;
                    } else {
                        mbar_wait(b_full + 8 * sb, pb);
                        b_base = base + sm.b + sb * p.b_stage_bytes;
                    }
                    const uint32_t b_lo0 = ((b_base >> 4) & 0x3FFFu) | (1u << 16);
                    const int t0 = g * p.tg, t_end = min(KS, (g + 1) * p.tg);
                    // one wgmma group per run of up to kMaxGroupTaps taps (a whole decoder stage): per tap nk K16 steps x MB row
                    // blocks, each as wide as the CTA's columns, in the order of one group per tap. The stage is released once all
                    // of them have completed. (Releasing it one group late, after a wgmma.wait_group 1 behind the next stage's first
                    // group, measured about 5 % slower end to end on an H100 at 400 W.)
#pragma unroll 1
                    for (int t = t0; t < t_end; t += kMaxGroupTaps)
                        wgmma_group_taps<MB, 8 * NB>(min(kMaxGroupTaps, t_end - t), nt, nk, acc, a_lo0 + (uint32_t)t * 8u,   // tap shift: +128 B
                                                     b_lo0 + (uint32_t)(t - t0) * b_step, hi, b_step);
                    wgmma_wait0();
                    if (!p.resident) {
                        if (wg_leader) mbar_arrive(b_empty + 8 * sb);
                        if (++sb == p.nb) { sb = 0; pb ^= 1; }
                    }
                }
                // split precision: the next position may multiply the same operand stage with the low weight part
                if (!(SP != 0 && c + 1 < p.nchunks && chunk_info<UPCAT, MG, SP>(p, c + 1).reuse)) {
                    if (wg_leader) mbar_arrive(a_empty + 8 * sa);
                    if (++sa == p.na) { sa = 0; pa ^= 1; }
                }
            }
            // epilogue
            if (threadIdx.x == 0) TRACE(2, tr2);
#pragma unroll
            for (int mb = 0; mb < MB; ++mb) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = (wg * MB + mb) * 64 + 16 * wq + (lane >> 2) + 8 * h;
                    int bb, l;
                    if (p.packed) { const int f = row / p.S; bb = b0 + f; l = row - f * p.S; if (f >= p.FR) l = p.L; }
                    else { bb = b0; l = l0 + row; }
                    const bool valid = (bb < p.B) && (l < p.L);
                    float hsum = 0.f;
#pragma unroll
                    for (int nb = 0; nb < NB; ++nb) {
                        if (nb >= nt) break;
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = nb * 16 + 8 * e + 2 * (lane & 3);            // column inside this CTA's N range
                            const float4 s2 = *reinterpret_cast<const float4 *>(&ss[n0 + col]);
                            const float f0 = lrelu(fmaf(acc[mb][8 * nb + 4 * e + 2 * h], s2.x, s2.y));
                            const float f1 = lrelu(fmaf(acc[mb][8 * nb + 4 * e + 2 * h + 1], s2.z, s2.w));
                            const bool col_ok = n0 + col < p.Cout;                        // Cout is even: both columns or none
                            if (p.out != nullptr && valid && col_ok) {
                                if (SP != 0) {
                                    // split precision: the row holds [hi(Cout) | lo(Cout)]; lo = bf16(v - hi)
                                    __nv_bfloat16 *orow = p.out + ((size_t)bb * p.L + l) * (2 * p.Cout) + n0 + col;
                                    *reinterpret_cast<uint32_t *>(orow) = pack_bf16(f0, f1);
                                    *reinterpret_cast<uint32_t *>(orow + p.Cout) =
                                        pack_bf16(f0 - __bfloat162float(__float2bfloat16_rn(f0)), f1 - __bfloat162float(__float2bfloat16_rn(f1)));
                                } else {
                                    *reinterpret_cast<uint32_t *>(p.out + ((size_t)bb * p.L + l) * p.Cout + n0 + col) = pack_bf16(f0, f1);
                                }
                            }
                            if (p.head && col_ok) hsum = fmaf(hw[col + 1], f1, fmaf(hw[col], f0, hsum));
                        }
                    }
                    if (p.head) {
                        // cat([o, input], 1) -> Conv1d(C+1 -> 1, k=1) -> Tanh   (model/unet_basic.py:98-99); the four threads of a
                        // row hold interleaved column pairs
                        hsum += __shfl_xor_sync(0xffffffffu, hsum, 1);
                        hsum += __shfl_xor_sync(0xffffffffu, hsum, 2);
                        if (valid && (lane & 3) == 0) {
                            const float hacc = fmaf(hw[p.Cout], __ldg(p.x + (size_t)bb * p.T + l), hw[p.Cout + 1] + hsum);
                            p.y[(size_t)bb * p.T + l] = tanh_fast(hacc);
                        }
                    }
                }
            }
        }
    } else if (UPCAT) {
        // ======================= upsample producers (decoder) =======================
        // F.interpolate(scale_factor=2, mode="linear", align_corners=True) of the previous block's output, written straight
        // into the swizzled operand tile. A thread owns (RPI = 16 consecutive output rows) x (one 16-byte channel vector): the
        // RPI/2 + 2 = 10 previous-level rows they interpolate between (row l lies between prev rows (l-1)>>1 and that + 1,
        // since src = l*(Lin-1)/(2Lin-1)) are fetched into registers one work unit AHEAD, so their DRAM latency overlaps the
        // wait for the shared-memory stage. The head-only instantiation (HD: 24 upsampled channels = 3 vectors per row) uses
        // 8-row items: with 16-row items only 48 of its 128 producer threads had work (ncu, round 2).
        // Row-pair instantiation (PR): operand row m = positions 2m (q = 0) and 2m+1 (q = 1), which interpolate between previous-level
        // rows (m-1, m) and (m, m+1). An item is 8 operand rows x one 16-byte vector of REAL channels and writes both q halves of
        // the chunk ([q0: range | q1: the same range], 32 channels per full chunk) from a window of 10 previous-level rows.
        constexpr int RPI = (HD != 0 || PR != 0) ? 8 : 16;   // rows per item
        constexpr int WR = PR != 0 ? 10 : RPI / 2 + 2;       // previous-level rows per item
        const int pt = (warp - kFirstProducer) * 32 + lane;
        int sa = 0, pa = 0;
        int tr4 = 0; (void)tr4;
        uint32_t tma_par = 0;                              // merged chunks: phase parity of a_tma[stage], one bit per stage
        uint4 xr[WR];
        bool pref = false;
        const int nruns = (p.rows_used + RPI - 1) / RPI;
        // a chunk whose first-round items can be prefetched into the register window one work unit ahead
        auto unit_fast = [&](int c) { return SP == 0 && !p.packed && chunk_info<UPCAT, MG, SP>(p, c).up; };
        // loads of item `item` of unit (frame ub0, first row ul0, K-loop position c) into the window
        auto fetch = [&](int ub0, int ul0, int c, int item) {
            const ChunkInfo u = chunk_info<UPCAT, MG, SP>(p, c);
            if (PR != 0) {
                // `item` counts through ALL upsampled chunks of the tile (K-loop positions 0 .. nchunks0 - 1, produced in one phase)
                int cc = 0, it = item;
                for (; cc < p.nchunks0; ++cc) {
                    const int nci = nruns * (chunk_info<UPCAT, MG, SP>(p, cc).nvec >> 1);
                    if (it < nci) break;
                    it -= nci;
                }
                if (cc >= p.nchunks0) return;
                const ChunkInfo uu = chunk_info<UPCAT, MG, SP>(p, cc);
                const int nvr = uu.nvec >> 1, creal = p.Cin0 >> 1;             // vectors of real channels in this chunk
                const int run = it / nvr, vec = it - run * nvr;
                const int ch = uu.idx * 32 + vec * 8;
                const int ms = ul0 - PAD + RPI * run;                          // operand row = previous-level row
                const bool chok = ch < creal && ub0 < p.B;
                const __nv_bfloat16 *pb = p.prev + (size_t)ub0 * p.Lin * creal + ch;
#pragma unroll
                for (int qq = 0; qq < WR; ++qq) {
                    int m = ms - 1 + qq;
                    m = m < 0 ? 0 : (m > p.Lin - 1 ? p.Lin - 1 : m);
                    xr[qq] = chok ? __ldg(reinterpret_cast<const uint4 *>(pb + (size_t)m * creal)) : make_uint4(0u, 0u, 0u, 0u);
                }
                return;
            }
            const int nvec = u.nvec;
            if (item >= nruns * nvec) return;
            const int run = item / nvec, vec = item - run * nvec;
            const int ch = u.idx * 64 + vec * 8;
            const int ms = (ul0 - PAD + RPI * run) >> 1;
            const bool chok = ch < p.Cin0 && ub0 < p.B;
            const __nv_bfloat16 *pb = p.prev + (size_t)ub0 * p.Lin * p.Cin0 + ch;
#pragma unroll
            for (int qq = 0; qq < WR; ++qq) {
                int m = ms - 1 + qq;
                m = m < 0 ? 0 : (m > p.Lin - 1 ? p.Lin - 1 : m);
                xr[qq] = chok ? __ldg(reinterpret_cast<const uint4 *>(pb + (size_t)m * p.Cin0)) : make_uint4(0u, 0u, 0u, 0u);
            }
        };
        // interpolate + store the 16 rows of one item from the register window. Straight-line code (masks and a predicated
        // store instead of branches): the 16 rows are independent, and a branch per row serialises their dependent chains
        // (trace: ~3600 cycles per item with branches, the stage hand-off was waiting on it).
        auto emit = [&](uint8_t *dst, int l0, int c, int item, const uint4 (&w)[WR]) {
            const ChunkInfo u = chunk_info<UPCAT, MG, SP>(p, c);
            if (PR != 0) {
                // dst = base of the operand ring, c = ring stage of the tile's first upsampled chunk; `item` as in fetch
                int cc = 0, it = item;
                for (; cc < p.nchunks0; ++cc) {
                    const int nci = nruns * (chunk_info<UPCAT, MG, SP>(p, cc).nvec >> 1);
                    if (it < nci) break;
                    it -= nci;
                }
                if (cc >= p.nchunks0) return;
                const ChunkInfo uu = chunk_info<UPCAT, MG, SP>(p, cc);
                int stg = c + cc;
                if (stg >= p.na) stg -= p.na;
                const int nvr = uu.nvec >> 1;
                const int run = it / nvr, vec = it - run * nvr;
                const bool chok = uu.idx * 32 + vec * 8 < (p.Cin0 >> 1);
                const int mstart = l0 - PAD + RPI * run;
                const uint32_t drow = smem_u32(dst) + (uint32_t)stg * p.a_stage_bytes + (uint32_t)(RPI * run) * 128u;
#pragma unroll
                for (int j = 0; j < RPI; ++j) {
                    const int m = mstart + j;
                    const uint32_t keep = (chok && (unsigned)m < (unsigned)p.L) ? 0xffffffffu : 0u;   // zero rows = Conv1d padding
#pragma unroll
                    for (int qh = 0; qh < 2; ++qh) {
                        // position l = 2m + qh lies between previous-level rows m - 1 + qh and m + qh = window rows j + qh, j + qh + 1;
                        // lam1 = up_scale * l - (m - 1 + qh): the generic instantiation's formula (one fused rounding), packed bf16
                        const float lam1 = fmaf(p.up_scale, (float)(2 * m + qh), -(float)(m - 1 + qh));
                        const __nv_bfloat162 lam = __float2bfloat162_rn(lam1);
                        const __nv_bfloat162 *a2 = reinterpret_cast<const __nv_bfloat162 *>(&w[j + qh]);
                        const __nv_bfloat162 *b2 = reinterpret_cast<const __nv_bfloat162 *>(&w[j + qh + 1]);
                        __nv_bfloat162 r2[4];
#pragma unroll
                        for (int q4 = 0; q4 < 4; ++q4) r2[q4] = __hfma2(lam, __hsub2(b2[q4], a2[q4]), a2[q4]);
                        uint4 o = *reinterpret_cast<const uint4 *>(r2);
                        o.x &= keep; o.y &= keep; o.z &= keep; o.w &= keep;
                        const int dvec = uu.vo + qh * nvr + vec;                    // q1 half follows the q0 half of the chunk
                        st_shared_v4_if(drow + (uint32_t)(j * 128 + ((dvec ^ (j & 7)) << 4)), o, RPI * run + j < p.rows_used);
                    }
                }
                return;
            }
            const int nvec = u.nvec;
            const int run = item / nvec, vec = item - run * nvec;
            const int ch = u.idx * 64 + vec * 8;
            const int dvec = u.vo + vec;                                       // 16-byte vector inside the stage row
            const int lstart = l0 - PAD + RPI * run;                           // even
            const int ms = lstart >> 1;
            const bool chok = ch < p.Cin0;
            const float lf0 = (float)lstart, mf0 = (float)(ms - 1);            // small integers: exact in fp32
            const uint32_t drow = smem_u32(dst) + (uint32_t)(RPI * run) * 128u;
#pragma unroll
            for (int j = 0; j < RPI; ++j) {
                const int l = lstart + j;
                const int qa = (j >> 1) + (j & 1);
                // out = a + lam1 * (b - a) in packed bf16 (HFMA2); lam1 = up_scale * l - (ms - 1 + qa), one fused rounding
                const float lam1 = fmaf(p.up_scale, lf0 + (float)j, -(mf0 + (float)qa));
                const __nv_bfloat162 lam = __float2bfloat162_rn(lam1);
                const __nv_bfloat162 *a2 = reinterpret_cast<const __nv_bfloat162 *>(&w[qa]);
                const __nv_bfloat162 *b2 = reinterpret_cast<const __nv_bfloat162 *>(&w[qa + 1]);
                __nv_bfloat162 r2[4];
#pragma unroll
                for (int q4 = 0; q4 < 4; ++q4) r2[q4] = __hfma2(lam, __hsub2(b2[q4], a2[q4]), a2[q4]);
                uint4 o = *reinterpret_cast<const uint4 *>(r2);
                const uint32_t keep = (chok && (unsigned)l < (unsigned)p.L) ? 0xffffffffu : 0u;   // zero rows = Conv1d padding
                o.x &= keep; o.y &= keep; o.z &= keep; o.w &= keep;
                // predicated (not branched) 16-byte store; (RPI * run + j) & 7 == j & 7
                st_shared_v4_if(drow + (uint32_t)(j * 128 + ((dvec ^ (j & 7)) << 4)), o, RPI * run + j < p.rows_used);
            }
        };
        if (HD != 0) {
            // head-only instantiation: both operand chunks come out of the ring the TMA lane fills several entries ahead - the
            // upsampled chunk is interpolated from its window of previous-level rows, the skip chunk is copied into the swizzled
            // stage layout - so no global-load latency sits between two hand-offs (the generic path's register prefetch leaves
            // ~3000 cycles of it exposed per unit). One ring entry per chunk, in K-loop order.
            int ps_i = 0, ps_par = 0;
            for (int tile = first_tile; tile < total_tiles; tile += gridDim.x) {
                int b0, l0, n0;
                tile_coords(tile, b0, l0, n0);
                const int base_m = ((l0 - PAD) >> 1) - 1;                           // previous-level row held by scratch row 0
                const int rlo = max(0, -base_m), rhi = min(p.ps_rows - 1, p.Lin - 1 - base_m);
                for (int c = 0; c < p.nchunks; ++c) {
                    const ChunkInfo cu = chunk_info<UPCAT, MG, SP>(p, c);
                    const uint32_t scr = base + sm.ps + (uint32_t)ps_i * p.ps_bytes;
                    if (pt == 0) TRACE(4, tr4);
                    mbar_wait(p_full + 8 * ps_i, ps_par);
                    if (pt == 0) TRACE(4, tr4);
                    mbar_wait(a_empty + 8 * sa, pa ^ 1);
                    if (pt == 0) TRACE(4, tr4);
                    uint8_t *dst = base_ptr + sm.a + sa * p.a_stage_bytes;
                    if (cu.up) {
                        const uint32_t rowb = (uint32_t)p.Cin0 * 2u;                // dense box rows
                        const int nvec = cu.nvec, nitems = nruns * nvec;
#pragma unroll 1
                        for (int itx = pt; itx < nitems; itx += NPROD) {
                            const int run = itx / nvec, vec = itx - run * nvec;
                            const bool chok = cu.idx * 64 + vec * 8 < p.Cin0;
#pragma unroll
                            for (int qq = 0; qq < WR; ++qq) {
                                int r = (RPI / 2) * run + qq;
                                r = r < rlo ? rlo : (r > rhi ? rhi : r);
                                xr[qq] = chok ? ld_shared_v4(scr + (uint32_t)r * rowb + (uint32_t)(cu.idx * 128 + vec * 16)) : make_uint4(0u, 0u, 0u, 0u);
                            }
                            emit(dst, l0, c, itx, xr);
                        }
                    } else {
                        // skip rows l0 - PAD ... (zero rows outside the frame) -> vectors 0 .. 2 nk - 1 of the stage rows, zeros
                        // past the last channel
                        const uint32_t rowb = (uint32_t)p.Cin1 * 2u;
                        const int nv = cu.nk * 2, nitems = p.rows_used * nv;
                        const uint32_t dsts = smem_u32(dst);
#pragma unroll 2
                        for (int itx = pt; itx < nitems; itx += NPROD) {
                            const int row = itx / nv, vec = itx - row * nv;
                            const uint4 v = (cu.idx * 64 + vec * 8 < p.Cin1)
                                                ? ld_shared_v4(scr + (uint32_t)row * rowb + (uint32_t)(cu.idx * 128 + vec * 16))
                                                : make_uint4(0u, 0u, 0u, 0u);
                            st_shared_v4_if(dsts + (uint32_t)(row * 128 + ((vec ^ (row & 7)) << 4)), v, true);
                        }
                    }
                    if (pt == 0) TRACE(4, tr4);
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");       // generic-proxy writes -> tensor core reads
                    __syncwarp();
                    if (pt == 0) TRACE(4, tr4);
                    if (lane == 0) { mbar_arrive(a_full + 8 * sa); mbar_arrive(p_empty + 8 * ps_i); }
                    if (++sa == p.na) { sa = 0; pa ^= 1; }
                    if (++ps_i == p.ps_n) { ps_i = 0; ps_par ^= 1; }
                }
            }
        } else
        for (int tile = first_tile; tile < total_tiles; tile += gridDim.x) {
            int b0, l0, n0;
            tile_coords(tile, b0, l0, n0);
            bool lo_done = false;                                                    // split precision: the lo stage of this chunk was
            for (int c = 0; c < p.nchunks; ++c) {                                    // written together with its hi stage
                if (SP != 0 && chunk_info<UPCAT, MG, SP>(p, c).reuse) continue;      // no new operand data for this position
                if (SP != 0 && lo_done) {                                            // (already arrived on its barrier)
                    lo_done = false;
                    if (++sa == p.na) { sa = 0; pa ^= 1; }
                    continue;
                }
                if (PR != 0 && c < p.nchunks0) {
                    // Row-pair instantiation: ALL upsampled chunks of the tile (K-loop positions 0 .. nchunks0 - 1, consecutive ring
                    // stages) are produced in ONE phase - one round of items over the producer threads, one fence, one hand-off. (Its
                    // first version produced them chunk by chunk: two phases per tile made the block 25 % slower than the plain form
                    // although it issues half the MMAs.)
                    if (c > 0) continue;
                    const int nup = p.nchunks0;
                    if (!pref) fetch(b0, l0, 0, pt);
                    {
                        int s2 = sa, par = pa;
                        for (int u2 = 0; u2 < nup; ++u2) {
                            mbar_wait(a_empty + 8 * s2, par ^ 1);
                            if (++s2 == p.na) { s2 = 0; par ^= 1; }
                        }
                    }
                    int nitems = 0;
                    for (int u2 = 0; u2 < nup; ++u2) nitems += nruns * (chunk_info<UPCAT, MG, SP>(p, u2).nvec >> 1);
#pragma unroll 1
                    for (int itx = pt; itx < nitems; itx += NPROD) {
                        if (itx != pt) fetch(b0, l0, 0, itx);
                        emit(base_ptr + sm.a, l0, sa, itx, xr);
                    }
                    pref = false;
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    __syncwarp();
                    for (int u2 = 0; u2 < nup; ++u2) {
                        if (lane == 0) mbar_arrive(a_full + 8 * sa);
                        if (++sa == p.na) { sa = 0; pa ^= 1; }
                    }
                    const int nt = tile + (int)gridDim.x;
                    if (nt < total_tiles) {
                        int nb0, nl0, nn0;
                        tile_coords(nt, nb0, nl0, nn0);
                        fetch(nb0, nl0, 0, pt);
                        pref = true;
                    }
                    continue;
                }
                const bool fast = unit_fast(c);
                if (fast && !pref) fetch(b0, l0, c, pt);
                if (pt == 0) TRACE(4, tr4);
                mbar_wait(a_empty + 8 * sa, pa ^ 1);
                if (pt == 0) TRACE(4, tr4);
                const ChunkInfo cu = chunk_info<UPCAT, MG, SP>(p, c);
                bool emitted_fast = false;
                if (cu.up) {
                    if (MG != 0 && cu.merged) {                               // the TMA part of this stage must have landed
                        mbar_wait(a_tma + 8 * sa, (tma_par >> sa) & 1u);
                        tma_par ^= 1u << sa;
                    }
                    const int nvec = cu.nvec;                                // 16-byte vectors per row
                    uint8_t *dst = base_ptr + sm.a + sa * p.a_stage_bytes;
                    if (fast) {
                        const int nitems = nruns * (PR != 0 ? nvec >> 1 : nvec);
#pragma unroll 1
                        for (int itx = pt; itx < nitems; itx += NPROD) {
                            if (itx != pt) fetch(b0, l0, c, itx);            // later rounds load on demand
                            emit(dst, l0, c, itx, xr);
                        }
                        pref = false;
                        emitted_fast = true;
                    } else {
                        // frames shorter than a tile (packed), and every level in split-precision mode: generic per-(row, vector)
                        // path, ATen index math in fp32
                        const int items = p.rows_used * nvec;
                        if (SP != 0) {
                            // the chunk's lo-data position follows two positions later ([hi x w_hi, re-use x w_lo, lo x w_hi]): fill its
                            // stage (the next one of the ring) from the same interpolation instead of computing everything twice
                            const bool pair = !cu.lo && c + 2 < p.nchunks && p.chunk_map[c + 2] == (p.chunk_map[c] | 0x40) &&
                                              (p.chunk_map[c + 1] & 0x20);
                            int sa2 = sa + 1, pa2 = pa;
                            if (sa2 == p.na) { sa2 = 0; pa2 ^= 1; }
                            if (pair) mbar_wait(a_empty + 8 * sa2, pa2 ^ 1);
                            uint8_t *dst2 = base_ptr + sm.a + sa2 * p.a_stage_bytes;
                            // split precision: prev rows are [hi | lo] (2 Cin0 channels); interpolate hi + lo in fp32 with the fp32
                            // path's formula (lam0 a + lam1 b), emit the high or the low bf16 part of the result. Two items per
                            // thread are in flight: their 8 loads are issued before the first is used (the unit is latency-bound).
                            if (pair && !p.packed) {
                                // full-length frames: a thread owns 8 consecutive output rows x one 16-byte channel vector. Output row
                                // l lies between previous-level rows i0 = (l-1)>>1 and i0 + 1 (align_corners: src = l (Lin-1)/(2 Lin-1)),
                                // so the 8 rows need 6 source rows; they are loaded once (hi and lo halves), summed to fp32, and every
                                // row is interpolated, split into hi / lo and written to both operand stages. ~10x fewer loads and
                                // 3x fewer instructions per element than the per-row path below.
                                const int nruns8 = (p.rows_used + 7) >> 3;
                                const int items8 = nruns8 * nvec;
#pragma unroll 1
                                for (int itx = pt; itx < items8; itx += NPROD) {
                                    const int run = itx / nvec, vec = itx - run * nvec;
                                    const int ch = cu.idx * 64 + vec * 8;
                                    const int lstart = l0 - PAD + 8 * run;                        // even
                                    const int ms = lstart >> 1;
                                    const bool chok = ch < p.Cin0 && b0 < p.B;
                                    const __nv_bfloat16 *pb = p.prev + (size_t)b0 * p.Lin * (2 * p.Cin0) + ch;
                                    float fa[6][8];
#pragma unroll
                                    for (int qq = 0; qq < 6; ++qq) {
                                        int m = ms - 1 + qq;
                                        m = m < 0 ? 0 : (m > p.Lin - 1 ? p.Lin - 1 : m);
                                        uint4 hv = make_uint4(0u, 0u, 0u, 0u), lv = hv;
                                        if (chok) {
                                            hv = __ldg(reinterpret_cast<const uint4 *>(pb + (size_t)m * (2 * p.Cin0)));
                                            lv = __ldg(reinterpret_cast<const uint4 *>(pb + (size_t)m * (2 * p.Cin0) + p.Cin0));
                                        }
                                        const uint32_t hh[4] = {hv.x, hv.y, hv.z, hv.w}, ll[4] = {lv.x, lv.y, lv.z, lv.w};
#pragma unroll
                                        for (int q4 = 0; q4 < 4; ++q4) {
                                            const float2 fh = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&hh[q4]));
                                            const float2 fl = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&ll[q4]));
                                            fa[qq][2 * q4] = fh.x + fl.x; fa[qq][2 * q4 + 1] = fh.y + fl.y;
                                        }
                                    }
                                    const float lf0 = (float)lstart, mf0 = (float)(ms - 1);
#pragma unroll
                                    for (int j = 0; j < 8; ++j) {
                                        const int l = lstart + j, row = 8 * run + j;
                                        const int qa = (j >> 1) + (j & 1);
                                        const float lam1 = fmaf(p.up_scale, lf0 + (float)j, -(mf0 + (float)qa));
                                        const float lam0 = 1.f - lam1;
                                        const bool keep = chok && (unsigned)l < (unsigned)p.L;      // zero rows = Conv1d padding
                                        uint32_t rh[4], rl[4];
#pragma unroll
                                        for (int q4 = 0; q4 < 4; ++q4) {
                                            const float vx = keep ? lam0 * fa[qa][2 * q4] + lam1 * fa[qa + 1][2 * q4] : 0.f;
                                            const float vy = keep ? lam0 * fa[qa][2 * q4 + 1] + lam1 * fa[qa + 1][2 * q4 + 1] : 0.f;
                                            const float hx = __bfloat162float(__float2bfloat16_rn(vx)), hy = __bfloat162float(__float2bfloat16_rn(vy));
                                            rh[q4] = pack_bf16(vx, vy);
                                            rl[q4] = pack_bf16(vx - hx, vy - hy);
                                        }
                                        if (row < p.rows_used) {
                                            const uint32_t off = (uint32_t)(row * 128 + ((vec ^ (row & 7)) << 4));
                                            *reinterpret_cast<uint4 *>(dst + off) = make_uint4(rh[0], rh[1], rh[2], rh[3]);
                                            *reinterpret_cast<uint4 *>(dst2 + off) = make_uint4(rl[0], rl[1], rl[2], rl[3]);
                                        }
                                    }
                                }
                            } else {
                            constexpr int U = 2;
#pragma unroll 1
                            for (int itb = pt; itb < items; itb += U * NPROD) {
                                uint4 h0[U], l0v[U], h1[U], l1v[U];
                                float lam1[U];
                                bool ok[U];
#pragma unroll
                                for (int u = 0; u < U; ++u) {
                                    const int itx = itb + u * NPROD;
                                    const int row = itx / nvec, vec = itx - row * nvec;
                                    int bb = b0, l = l0 - PAD + row;
                                    if (p.packed) { const int f = row / p.S; bb = b0 + f; l = row - f * p.S - PAD; }
                                    const int ch = cu.idx * 64 + vec * 8;
                                    ok[u] = itx < items && bb < p.B && l >= 0 && l < p.L && ch < p.Cin0;
                                    h0[u] = l0v[u] = h1[u] = l1v[u] = make_uint4(0u, 0u, 0u, 0u);
                                    lam1[u] = 0.f;
                                    if (ok[u]) {
                                        const float s = p.up_scale * (float)l;
                                        const int i0 = (int)s;
                                        const int i1 = i0 + (i0 < p.Lin - 1 ? 1 : 0);
                                        lam1[u] = s - (float)i0;
                                        const __nv_bfloat16 *r0 = p.prev + ((size_t)bb * p.Lin + i0) * (2 * p.Cin0) + ch;
                                        const __nv_bfloat16 *r1 = p.prev + ((size_t)bb * p.Lin + i1) * (2 * p.Cin0) + ch;
                                        h0[u] = __ldg(reinterpret_cast<const uint4 *>(r0)); l0v[u] = __ldg(reinterpret_cast<const uint4 *>(r0 + p.Cin0));
                                        h1[u] = __ldg(reinterpret_cast<const uint4 *>(r1)); l1v[u] = __ldg(reinterpret_cast<const uint4 *>(r1 + p.Cin0));
                                    }
                                }
#pragma unroll
                                for (int u = 0; u < U; ++u) {
                                    const int itx = itb + u * NPROD;
                                    if (itx >= items) break;
                                    const int row = itx / nvec, vec = itx - row * nvec;
                                    const float lam0 = 1.f - lam1[u];
                                    const uint32_t ah[4] = {h0[u].x, h0[u].y, h0[u].z, h0[u].w}, al[4] = {l0v[u].x, l0v[u].y, l0v[u].z, l0v[u].w};
                                    const uint32_t bh[4] = {h1[u].x, h1[u].y, h1[u].z, h1[u].w}, bl[4] = {l1v[u].x, l1v[u].y, l1v[u].z, l1v[u].w};
                                    uint32_t r[4], r2[4];
#pragma unroll
                                    for (int q4 = 0; q4 < 4; ++q4) {
                                        const float2 fah = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&ah[q4]));
                                        const float2 fal = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&al[q4]));
                                        const float2 fbh = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&bh[q4]));
                                        const float2 fbl = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&bl[q4]));
                                        const float vx = lam0 * (fah.x + fal.x) + lam1[u] * (fbh.x + fbl.x);
                                        const float vy = lam0 * (fah.y + fal.y) + lam1[u] * (fbh.y + fbl.y);
                                        const float hx = __bfloat162float(__float2bfloat16_rn(vx)), hy = __bfloat162float(__float2bfloat16_rn(vy));
                                        r[q4] = cu.lo ? pack_bf16(vx - hx, vy - hy) : pack_bf16(vx, vy);
                                        r2[q4] = pack_bf16(vx - hx, vy - hy);
                                    }
                                    *reinterpret_cast<uint4 *>(dst + row * 128 + ((vec ^ (row & 7)) << 4)) =
                                        ok[u] ? make_uint4(r[0], r[1], r[2], r[3]) : make_uint4(0u, 0u, 0u, 0u);
                                    if (pair)
                                        *reinterpret_cast<uint4 *>(dst2 + row * 128 + ((vec ^ (row & 7)) << 4)) =
                                            ok[u] ? make_uint4(r2[0], r2[1], r2[2], r2[3]) : make_uint4(0u, 0u, 0u, 0u);
                                }
                            }
                            }
                            if (pair) {
                                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                                __syncwarp();
                                if (lane == 0) mbar_arrive(a_full + 8 * sa2);
                                lo_done = true;
                            }
                        } else
                        for (int itx = pt; itx < items; itx += NPROD) {
                            const int row = itx / nvec, vec = itx - row * nvec;
                            int bb = b0, l = l0 - PAD + row;
                            if (p.packed) { const int f = row / p.S; bb = b0 + f; l = row - f * p.S - PAD; }
                            const int ch = cu.idx * 64 + vec * 8;
                            uint4 o = make_uint4(0u, 0u, 0u, 0u);
                            if (bb < p.B && l >= 0 && l < p.L && ch < p.Cin0) {
                                const float s = p.up_scale * (float)l;
                                const int i0 = (int)s;
                                const int i1 = i0 + (i0 < p.Lin - 1 ? 1 : 0);
                                const float lam1 = s - (float)i0, lam0 = 1.f - lam1;
                                const uint4 u0 = __ldg(reinterpret_cast<const uint4 *>(p.prev + ((size_t)bb * p.Lin + i0) * p.Cin0 + ch));
                                const uint4 u1 = __ldg(reinterpret_cast<const uint4 *>(p.prev + ((size_t)bb * p.Lin + i1) * p.Cin0 + ch));
                                const uint32_t a0[4] = {u0.x, u0.y, u0.z, u0.w}, a1[4] = {u1.x, u1.y, u1.z, u1.w};
                                uint32_t r[4];
#pragma unroll
                                for (int q4 = 0; q4 < 4; ++q4) {
                                    const float2 f0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&a0[q4]));
                                    const float2 f1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&a1[q4]));
                                    r[q4] = pack_bf16(lam0 * f0.x + lam1 * f1.x, lam0 * f0.y + lam1 * f1.y);
                                }
                                o = make_uint4(r[0], r[1], r[2], r[3]);
                            }
                            *reinterpret_cast<uint4 *>(dst + row * 128 + ((vec ^ (row & 7)) << 4)) = o;
                        }
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> tensor core reads
                }
                __syncwarp();
                if (pt == 0) TRACE(4, tr4);
                if (lane == 0) mbar_arrive(a_full + 8 * sa);
                if (++sa == p.na) { sa = 0; pa ^= 1; }
                // (The producers arrive on EVERY chunk's barrier, also on TMA chunks they do not write: an mbarrier wait only tells the
                // current phase from the previous one, and a role that skipped the barriers of several consecutive TMA chunks would
                // lose track of the ring's phases - tried in round 2: dead-lock on the blocks with more skip chunks than stages.)
                if (emitted_fast && !p.pf_late) {
                    // next upsampled unit of this CTA (K-loop order): prefetch its first-round item. Issued AFTER the hand-off:
                    // fence.proxy.async compiles to MEMBAR.ALL.CTA, which would otherwise hold the arrive back until these
                    // loads have returned (trace: ~1900 cycles per unit).
                    int nt = tile, nc = c + 1;
                    for (int hop = 0; hop < p.nchunks; ++hop) {
                        if (nc >= p.nchunks) { nc = 0; nt += gridDim.x; }
                        if (chunk_info<UPCAT, MG, SP>(p, nc).up) break;
                        ++nc;
                    }
                    if (nt < total_tiles && unit_fast(nc)) {
                        int nb0, nl0, nn0;
                        tile_coords(nt, nb0, nl0, nn0);
                        fetch(nb0, nl0, nc, pt);
                        pref = true;
                    }
                }
            }
        }
    }
}

// -------------------------------------------------------------------------------------------------
// bottom of the U (frames of at most 16 samples): the block as ONE dense GEMM over frames
// -------------------------------------------------------------------------------------------------
// With L <= 16 the implicit GEMM over positions wastes most of its MMA rows on per-frame halos and cannot fill the SMs.
// Here the frames are the GEMM rows: the channels-last activations ARE the matrix [B][L*C],
//     Y[b][(l, co)] = sum_(l', ci) X[b][(l', ci)] * W'[(l, co)][(l', ci)],
// with Toeplitz-expanded weights W'[(l,co)][(l',ci)] = w[co][ci][l'-l+pad] (zero outside the taps; built once per weight
// update by expand_gemm_weights_kernel). An encoder's decimation is the tensor map's row stride; a decoder's linear
// interpolation is folded into the expanded weights of its upsampled input (W * U, in fp32, then bf16), so both of its sources
// are plain TMA operands and there are no producer warps. One CTA = 128 frames x Nh output columns (two consumer warpgroups of
// 64 frames each, accumulators in registers); K runs over 64-channel chunks of the input positions that reach the CTA's output
// positions (the band), several chunks per pipeline stage.
struct GemmParams {
    int B, N, Nh;                  // rows (frames), output columns (= L * Cout), columns per CTA (<= kAccColsLarge)
    int cout;                      // channels per output position (the folded BatchNorm vector repeats with this period)
    int L;                         // output positions
    // two sources: chunk list = [source 0 positions x 64-channel chunks | source 1 positions x chunks]; weight K slot = global index
    int npos[2], cpp[2];           // input positions, 64-channel chunks per position
    int reach_lo[2], reach_hi[2];  // input positions [l_lo + reach_lo, l_hi + reach_hi] reach output positions [l_lo, l_hi]; for a
    int halve[2];                  // half-resolution source (decoder: previous block) the output range is halved first
    int nstages, cps;              // ring depth, K chunks per stage
    uint32_t a_bytes, w_bytes;
    const float2 *ss;              // [cout] folded BatchNorm (scale, shift)
    __nv_bfloat16 *out;            // [B][N]
};
constexpr int kGemmThreads = 32 * (kEpiWarpsLarge + 1);   // two consumer warpgroups + the TMA warp

__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tm0, const __grid_constant__ CUtensorMap tm1, const __grid_constant__ CUtensorMap tmW,
               const GemmParams p)
{
    constexpr int NWG = kEpiWarpsLarge / 4;
    constexpr int NB = kAccColsLarge / 16;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    // a stage holds `cps` consecutive K chunks: [A: cps x 16 KB (128 frames x 64 channels each) | W: cps x w_bytes]
    const uint32_t stage_bytes = (uint32_t)p.cps * (16384u + p.w_bytes);
    const uint32_t bars = base + (uint32_t)p.nstages * stage_bytes;                 // full[8] empty[8]
    const uint32_t full = bars, empty = bars + 64;
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n0 = blockIdx.x * p.Nh, b0 = blockIdx.y * 128;
    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tm0)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmW)) : "memory");
        for (int s = 0; s < 8; ++s) { mbar_init(full + 8 * s, 1); mbar_init(empty + 8 * s, NWG); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    asm volatile("griddepcontrol.wait;" ::: "memory");

    // the band: input positions of each source that reach this CTA's output positions
    const int l_lo = n0 / p.cout, l_hi = min(p.N - 1, n0 + p.Nh - 1) / p.cout;
    int plo[2], cnt[2], nch = 0;
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        const int a = p.halve[s] ? (l_lo >> 1) : l_lo, b = p.halve[s] ? (l_hi >> 1) : l_hi;
        plo[s] = max(0, a + p.reach_lo[s]);
        const int phi = min(p.npos[s] - 1, b + p.reach_hi[s]);
        cnt[s] = p.npos[s] > 0 ? (phi - plo[s] + 1) * p.cpp[s] : 0;
        nch += cnt[s];
    }
    const int nst = (nch + p.cps - 1) / p.cps;                   // stages of this CTA's K loop
    const int n_this = min(p.Nh, p.N - n0);
    if (warp == kEpiWarpsLarge) {
        // ======================= TMA producer =======================
        if (lane == 0) {
            for (int it = 0; it < nst; ++it) {
                const uint32_t st = (uint32_t)it % (uint32_t)p.nstages, ph = ((uint32_t)it / (uint32_t)p.nstages) & 1u;
                const int k0 = it * p.cps, kn = min(p.cps, nch - k0);
                mbar_wait(empty + 8 * st, ph ^ 1);
                mbar_expect_tx(full + 8 * st, (uint32_t)kn * (16384u + (uint32_t)p.Nh * 128u));
                const uint32_t dst = base + st * stage_bytes;
                for (int j = 0; j < kn; ++j) {
                    int k = k0 + j, s = 0;
                    if (k >= cnt[0]) { k -= cnt[0]; s = 1; }
                    const int pos = plo[s] + k / p.cpp[s], cc = k % p.cpp[s];
                    const int kslot = (s == 0 ? 0 : p.npos[0] * p.cpp[0]) + pos * p.cpp[s] + cc;
                    tma_load_3d(dst + (uint32_t)j * 16384u, s == 0 ? &tm0 : &tm1, full + 8 * st, cc * 64, pos, b0);
                    tma_load_3d(dst + (uint32_t)p.cps * 16384u + (uint32_t)j * p.w_bytes, &tmW, full + 8 * st, kslot * 64, n0, 0);
                }
            }
        }
    } else {
        // ======================= consumer warpgroups: wgmma over 64 frames each + epilogue =======================
        const int wg = warp >> 2, wq = warp & 3;
        const int nt = n_this >> 4;
        const uint32_t hi = (uint32_t)(1024 >> 4) | (1u << 30);
        float acc[1][8 * NB];
#pragma unroll
        for (int j = 0; j < 8 * NB; ++j) acc[0][j] = 0.f;
        for (int it = 0; it < nst; ++it) {
            const uint32_t st = (uint32_t)it % (uint32_t)p.nstages, ph = ((uint32_t)it / (uint32_t)p.nstages) & 1u;
            const int kn = min(p.cps, nch - it * p.cps);
            mbar_wait(full + 8 * st, ph);
            const uint32_t a0 = (((base + st * stage_bytes) >> 4) & 0x3FFFu) | (1u << 16);
            const uint32_t w0 = (((base + st * stage_bytes + (uint32_t)p.cps * 16384u) >> 4) & 0x3FFFu) | (1u << 16);
            // one wgmma group per K chunk: 4 K16 steps, each one m64n(n_this)k16
#pragma unroll 1
            for (int j = 0; j < kn; ++j)
                wgmma_group(nt, 4, acc, a0 + (uint32_t)j * 1024u + (uint32_t)wg * 512u, w0 + (uint32_t)j * (p.w_bytes >> 4), hi);
            wgmma_wait0();
            if ((threadIdx.x & 127) == 0) mbar_arrive(empty + 8 * st);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int b = b0 + wg * 64 + 16 * wq + (lane >> 2) + 8 * h;
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) {
                if (nb >= nt) break;
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = n0 + nb * 16 + 8 * e + 2 * (lane & 3);
                    const float2 s0 = __ldg(p.ss + n % p.cout), s1 = __ldg(p.ss + (n + 1) % p.cout);
                    const uint32_t o = pack_bf16(lrelu(fmaf(acc[0][8 * nb + 4 * e + 2 * h], s0.x, s0.y)),
                                                 lrelu(fmaf(acc[0][8 * nb + 4 * e + 2 * h + 1], s1.x, s1.y)));
                    if (b < p.B) *reinterpret_cast<uint32_t *>(p.out + (size_t)b * p.N + n) = o;
                }
            }
        }
    }
}

// Toeplitz expansion of a block's weights for gemm_tc_kernel: wx[n = l * Cout + co][k], K slots of 64 channels:
//   encoder / middle (dec = 0): slot (l' * cpp0 + cc) holds channels cc*64.. of input position l', value w[co][ci][l' - l + pad]
//   decoder (dec = 1): source 0 = previous block at half resolution (position m), value sum_l' w[co][ci][l'-l+pad] U[l'][m] with
//     U = F.interpolate(scale_factor=2, linear, align_corners=True) (fp32 index math as ATen: i0 = int(l' s), lam = l' s - i0);
//     source 1 = skip at position l', channels offset by Cin0 in w.
__global__ void expand_gemm_weights_kernel(const float *__restrict__ w, __nv_bfloat16 *__restrict__ wx, int Cout, int Cin0, int Cin1, int K,
                                           int L, int dec, int npos0, int cpp0, int npos1, int cpp1, float up_scale)
{
    const int Ktot = (npos0 * cpp0 + npos1 * cpp1) * 64;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)L * Cout * Ktot) return;
    const int k = (int)(i % Ktot);
    const int n = (int)(i / Ktot);
    const int l = n / Cout, co = n - l * Cout;
    const int pad = (K - 1) / 2, Cin = Cin0 + Cin1;
    int slot = k >> 6;
    const int j = k & 63;
    float v = 0.f;
    if (slot < npos0 * cpp0) {
        const int pos = slot / cpp0, ci = (slot - pos * cpp0) * 64 + j;
        if (ci < Cin0) {
            if (!dec) {
                const int t = pos - l + pad;
                if (t >= 0 && t < K) v = w[((size_t)co * Cin + ci) * K + t];
            } else {
                const int Lin = npos0;
                for (int t = 0; t < K; ++t) {
                    const int lp = l + t - pad;
                    if (lp < 0 || lp >= L) continue;
                    const float s = up_scale * (float)lp;
                    const int i0 = (int)s;
                    const int i1 = i0 + (i0 < Lin - 1 ? 1 : 0);
                    const float lam1 = s - (float)i0, lam0 = 1.f - lam1;
                    const float wv = w[((size_t)co * Cin + ci) * K + t];
                    if (i0 == pos) v = fmaf(wv, lam0, v);
                    if (i1 == pos) v = fmaf(wv, lam1, v);
                }
            }
        }
    } else {
        slot -= npos0 * cpp0;
        const int pos = slot / cpp1, ci = (slot - pos * cpp1) * 64 + j;
        const int t = pos - l + pad;
        if (ci < Cin1 && t >= 0 && t < K) v = w[((size_t)co * Cin + Cin0 + ci) * K + t];
    }
    wx[i] = __float2bfloat16_rn(v);
}

// -------------------------------------------------------------------------------------------------
// enc0: Conv1d(1 -> C, k=15) + BN + LeakyReLU on CUDA cores (Cin = 1: K = 15, HBM-bound), fp32 in, bf16 NLC out
// -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 4) enc0_kernel(const float *__restrict__ x, const float *__restrict__ w /*[C][1][15]*/,
                                                      const float *__restrict__ scale, const float *__restrict__ shift,
                                                      __nv_bfloat16 *__restrict__ out, int B, int T, int C, int split,
                                                      __nv_bfloat16 *__restrict__ even_out)
{
    // even_out != nullptr (row-pair mode of the next block): the even positions are written a second time, densely, as
    // [B][T/2][C] - the decimated input o[:, :, ::2] of the next encoder block as a contiguous matrix, so that [T/4][2 C] is a view of it.
    // A block owns 1024 consecutive positions of one frame; a thread owns 4 consecutive positions and sweeps the channels
    // 8 at a time (32 accumulators, 15 taps: 480 FFMA per 2x15 broadcast LDS.128 of weights). The bf16 rows are staged in
    // shared memory ([1024][C] is one contiguous range of the channels-last output) and leave with ONE bulk async copy.
    constexpr int KS = 15, PAD = 7, TILE = 1024;
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    extern __shared__ uint8_t smem_raw[];
    float *ws = reinterpret_cast<float *>(smem_raw);          // [15][C]
    float *sc = ws + KS * C, *sh = sc + C;
    float *xs = sh + C + ((4 - ((KS * C + 2 * C) & 3)) & 3);  // keep xs 16-byte aligned
    uint8_t *stage = reinterpret_cast<uint8_t *>(xs + TILE + 16);   // [TILE][C] bf16 ([TILE][2 C] = [hi | lo] in split-precision mode)
    const int RC = split ? 2 * C : C;                                // channels per stored row
    const int b = blockIdx.y;
    const int l0 = blockIdx.x * TILE;
    for (int i = threadIdx.x; i < KS * C; i += 256) { const int k = i / C, c = i - k * C; ws[i] = w[c * KS + k]; }
    for (int i = threadIdx.x; i < C; i += 256) { sc[i] = scale[i]; sh[i] = shift[i]; }
    // the previous forward's last kernel may still be reading this workspace: wait before the first dependent access
    asm volatile("griddepcontrol.wait;" ::: "memory");
    for (int i = threadIdx.x; i < TILE + 16; i += 256) {
        const int l = l0 - PAD + i - 1;                       // xs[i] = x[l0 - 8 + i] so that a thread's window starts 16-byte aligned
        xs[i] = (l >= 0 && l < T) ? x[(size_t)b * T + l] : 0.f;
    }
    __syncthreads();
    // window: positions 4*tid .. 4*tid+3 need x[l-7 .. l+3+7] = xs[4*tid + 1 .. 4*tid + 18]; load xs[4*tid .. 4*tid+19]
    float xw[20];
#pragma unroll
    for (int q = 0; q < 5; ++q) {
        const float4 v = *reinterpret_cast<const float4 *>(&xs[4 * threadIdx.x + 4 * q]);
        xw[4 * q] = v.x; xw[4 * q + 1] = v.y; xw[4 * q + 2] = v.z; xw[4 * q + 3] = v.w;
    }
    for (int c0 = 0; c0 < C; c0 += 8) {
        float acc[4][8];
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int m = 0; m < 8; ++m) acc[j][m] = 0.f;
#pragma unroll
        for (int k = 0; k < KS; ++k) {
            const float4 w0 = *reinterpret_cast<const float4 *>(&ws[k * C + c0]);
            const float4 w1 = *reinterpret_cast<const float4 *>(&ws[k * C + c0 + 4]);
            const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int m = 0; m < 8; ++m) acc[j][m] = fmaf(wv[m], xw[j + k + 1], acc[j][m]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float f[8];
#pragma unroll
            for (int m = 0; m < 8; ++m) f[m] = lrelu(fmaf(acc[j][m], sc[c0 + m], sh[c0 + m]));
            uint8_t *srow = stage + (size_t)(4 * threadIdx.x + j) * (RC * 2) + c0 * 2;
            *reinterpret_cast<uint4 *>(srow) =
                make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
            if (even_out != nullptr && (j & 1) == 0 && l0 + 4 * (int)threadIdx.x + j < T)
                *reinterpret_cast<uint4 *>(even_out + ((size_t)b * (T >> 1) + ((l0 + 4 * threadIdx.x + j) >> 1)) * C + c0) =
                    make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
            if (split) {
                float g[8];
#pragma unroll
                for (int m = 0; m < 8; ++m) g[m] = f[m] - __bfloat162float(__float2bfloat16_rn(f[m]));
                *reinterpret_cast<uint4 *>(srow + C * 2) =
                    make_uint4(pack_bf16(g[0], g[1]), pack_bf16(g[2], g[3]), pack_bf16(g[4], g[5]), pack_bf16(g[6], g[7]));
            }
        }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (threadIdx.x == 0) {
        const int rows = min(TILE, T - l0);
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                     ::"l"(out + ((size_t)b * T + l0) * RC), "r"(smem_u32(stage)), "r"((uint32_t)(rows * RC * 2)) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

// enc0, persistent form (round 2, last session): the same arithmetic in the same order (bit-identical output), but a block loops over
// tiles: the weights are loaded once, the samples of the NEXT tile stream into shared memory by cp.async while this tile is
// computed, and the bulk store of a tile's rows drains while the next tile's first channel pass is computed (the one-shot
// kernel above spends ~35 % of its time in the un-overlapped load -> compute -> store -> drain phases of its 4 resident blocks).
__global__ void __launch_bounds__(256, 4) enc0_kernel_v2(const float *__restrict__ x, const float *__restrict__ w /*[C][1][15]*/,
                                                         const float *__restrict__ scale, const float *__restrict__ shift,
                                                         __nv_bfloat16 *__restrict__ out, int B, int T, int C, int split,
                                                         __nv_bfloat16 *__restrict__ even_out)
{
    constexpr int KS = 15, PAD = 7, TILE = 1024;
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    extern __shared__ uint8_t smem_raw[];
    float *ws = reinterpret_cast<float *>(smem_raw);          // [15][C]
    float *sc = ws + KS * C, *sh = sc + C;
    float *xs = sh + C + ((4 - ((KS * C + 2 * C) & 3)) & 3);  // 16-byte aligned: xs[i] = x[l0 - 8 + i], i < TILE + 16
    uint8_t *stage = reinterpret_cast<uint8_t *>(xs + TILE + 16);
    const int RC = split ? 2 * C : C;
    const int tpf = (T + TILE - 1) / TILE;                    // tiles per frame
    const int total = B * tpf;
    for (int i = threadIdx.x; i < KS * C; i += 256) { const int k = i / C, c = i - k * C; ws[i] = w[c * KS + k]; }
    for (int i = threadIdx.x; i < C; i += 256) { sc[i] = scale[i]; sh[i] = shift[i]; }
    asm volatile("griddepcontrol.wait;" ::: "memory");
    // samples of a tile -> xs by 4-byte cp.async (zero fill outside the frame = Conv1d padding)
    auto prefetch = [&](int tile) {
        const int b = tile / tpf, l0 = (tile - b * tpf) * TILE;
        for (int i = threadIdx.x; i < TILE + 16; i += 256) {
            const int l = l0 - PAD + i - 1;
            const bool ok = l >= 0 && l < T;
            const float *src = x + (size_t)b * T + (ok ? l : 0);
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(xs + i)), "l"(src), "r"(ok ? 4 : 0) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    int tile = blockIdx.x;
    if (tile < total) prefetch(tile);
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();
    for (; tile < total; tile += gridDim.x) {
        const int b = tile / tpf, l0 = (tile - b * tpf) * TILE;
        float xw[20];
#pragma unroll
        for (int q = 0; q < 5; ++q) {
            const float4 v = *reinterpret_cast<const float4 *>(&xs[4 * threadIdx.x + 4 * q]);
            xw[4 * q] = v.x; xw[4 * q + 1] = v.y; xw[4 * q + 2] = v.z; xw[4 * q + 3] = v.w;
        }
        __syncthreads();                                      // every thread has its window: xs may be overwritten
        if (tile + (int)gridDim.x < total) prefetch(tile + gridDim.x);
        for (int c0 = 0; c0 < C; c0 += 8) {
            float acc[4][8];
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int m = 0; m < 8; ++m) acc[j][m] = 0.f;
#pragma unroll
            for (int k = 0; k < KS; ++k) {
                const float4 w0 = *reinterpret_cast<const float4 *>(&ws[k * C + c0]);
                const float4 w1 = *reinterpret_cast<const float4 *>(&ws[k * C + c0 + 4]);
                const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int m = 0; m < 8; ++m) acc[j][m] = fmaf(wv[m], xw[j + k + 1], acc[j][m]);
            }
            if (c0 == 0) {
                // the previous tile's bulk store must have read the staging rows before they are overwritten
                if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                __syncthreads();
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float f[8];
#pragma unroll
                for (int m = 0; m < 8; ++m) f[m] = lrelu(fmaf(acc[j][m], sc[c0 + m], sh[c0 + m]));
                uint8_t *srow = stage + (size_t)(4 * threadIdx.x + j) * (RC * 2) + c0 * 2;
                const uint4 o = make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
                *reinterpret_cast<uint4 *>(srow) = o;
                if (even_out != nullptr && (j & 1) == 0 && l0 + 4 * (int)threadIdx.x + j < T)
                    *reinterpret_cast<uint4 *>(even_out + ((size_t)b * (T >> 1) + ((l0 + 4 * threadIdx.x + j) >> 1)) * C + c0) = o;
                if (split) {
                    float g[8];
#pragma unroll
                    for (int m = 0; m < 8; ++m) g[m] = f[m] - __bfloat162float(__float2bfloat16_rn(f[m]));
                    *reinterpret_cast<uint4 *>(srow + C * 2) =
                        make_uint4(pack_bf16(g[0], g[1]), pack_bf16(g[2], g[3]), pack_bf16(g[4], g[5]), pack_bf16(g[6], g[7]));
                }
            }
        }
        asm volatile("cp.async.wait_all;" ::: "memory");           // the next tile's samples have landed (this thread's copies)
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();                                          // staging rows complete, xs of the next tile visible to all
        if (threadIdx.x == 0) {
            const int rows = min(TILE, T - l0);
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                         ::"l"(out + ((size_t)b * T + l0) * RC), "r"(smem_u32(stage)), "r"((uint32_t)(rows * RC * 2)) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
    }
    if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// -------------------------------------------------------------------------------------------------
// row-pair mode: a K-tap conv block over positions as a K'-tap block over PAIRS of positions
// -------------------------------------------------------------------------------------------------
// Row m of the pair block = positions 2m (q = 0) and 2m + 1 (q = 1); output column r * Cout + co = position 2m + r. With
// P = (K-1)/2 and P' = (P+1)/2 the pair block has K' = 2P'+1 taps dm = -P' .. P' and
//     W'[dm + P'][r Cout + co][v] = w[co][c(v)][2 dm + q(v) - r + P]      (zero where that tap index is outside 0 .. K-1)
// v = virtual input channel: segment 0 (2 C0 channels) then segment 1 (2 C1 channels). Segment 1 and an encoder's segment 0
// are the contiguous view [L/2][2 C] of a channels-last tensor: v = q C + c. A decoder's segment 0 is written by the
// producer warps 32 real channels per 64-wide chunk, [q0: range | q1: the same range]: chunk k = v / 64 holds real channels
// 32 k .. 32 k + w - 1 (w = min(32, C0 - 32 k)), q = (v % 64) / w. Same function on the host (wunet_debug_pair_weights, tests).
__host__ __device__ inline int pair_taps(int K) { return 2 * ((((K - 1) / 2) + 1) / 2) + 1; }
__host__ __device__ inline float pair_weight(const float *w, int Cout, int C0, int C1, int K, int dec, int cov, int v, int tv)
{
    const int P = (K - 1) / 2, Pp = (P + 1) / 2;
    const int r = cov / Cout, co = cov - r * Cout;
    int q, c;
    if (v < 2 * C0) {
        if (dec) {
            const int k = v >> 6, j = v & 63, lo = 32 * k;
            const int wd = (C0 - lo) < 32 ? (C0 - lo) : 32;
            q = j / wd; c = lo + (j - q * wd);
            if (q > 1) return 0.f;
        } else { q = v / C0; c = v - q * C0; }
    } else {
        const int u = v - 2 * C0;
        if (u >= 2 * C1) return 0.f;
        q = u / C1; c = C0 + (u - q * C1);
    }
    const int t = 2 * (tv - Pp) + q - r + P;
    if (r > 1 || t < 0 || t >= K) return 0.f;
    return w[((size_t)co * (C0 + C1) + c) * K + t];
}
// wv[2 Cout][2 (C0 + C1)][K'] fp32 (the layout pack_tc_kernel reads), scale / shift replicated for both halves of the columns
__global__ void expand_pair_weights_kernel(const float *__restrict__ w, const float *__restrict__ scale, const float *__restrict__ shift,
                                           float *__restrict__ wv, float *__restrict__ scale_v, float *__restrict__ shift_v, int Cout,
                                           int C0, int C1, int K, int dec)
{
    const int Kp = pair_taps(K), Cv = 2 * (C0 + C1);
    const long long n = (long long)2 * Cout * Cv * Kp;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const int tv = (int)(i % Kp);
        const int v = (int)((i / Kp) % Cv);
        const int cov = (int)(i / ((long long)Kp * Cv));
        wv[i] = pair_weight(w, Cout, C0, C1, K, dec, cov, v, tv);
    }
    if (i < 2 * Cout) { scale_v[i] = scale[i % Cout]; shift_v[i] = shift[i % Cout]; }
}

// -------------------------------------------------------------------------------------------------
// block 0 (Conv1d(1 -> C, k = 15)) on the tensor cores: groups of 8 samples
// -------------------------------------------------------------------------------------------------
// The raw input [T] IS the matrix [T/8][8]; row m = samples 8m .. 8m+7 (virtual input channels q = 0..7, one K16 step with the
// upper half zero-filled by TMA), output row m = the 8 x C results of those samples = [T/8][8 C], the same memory as the
// channels-last [T][C]. The 15 taps become 3 taps over rows (dm = -1, 0, 1):
//     W'[dm + 1][r C + co][q] = w[co][8 dm + q - r + 7]      (zero where that index is outside 0 .. 14)
// so the block is 3 MMAs of N = 8 C per 128 rows = 1024 samples, and its cost is its epilogue and its HBM traffic - it runs as a
// plain 3-tap encoder block of conv_tc_kernel. The input is needed in bf16 for that (x_to_bf16_kernel): the products then carry
// bf16-rounded samples and weights like those of every other block of this path.
__host__ __device__ inline float group8_weight(const float *w, int Cout, int K, int cov, int q, int tv)
{
    const int r = cov / Cout, co = cov - r * Cout;
    const int t = 8 * (tv - 1) + q - r + (K - 1) / 2;
    if (r > 7 || q > 7 || t < 0 || t >= K) return 0.f;
    return w[(size_t)co * K + t];
}
__global__ void expand_group8_weights_kernel(const float *__restrict__ w, const float *__restrict__ scale, const float *__restrict__ shift,
                                             float *__restrict__ wv, float *__restrict__ scale_v, float *__restrict__ shift_v, int Cout, int K)
{
    const int n = 8 * Cout * 8 * 3;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const int tv = i % 3, q = (i / 3) % 8, cov = i / 24;
        wv[i] = group8_weight(w, Cout, K, cov, q, tv);
    }
    if (i < 8 * Cout) { scale_v[i] = scale[i % Cout]; shift_v[i] = shift[i % Cout]; }
}
__global__ void x_to_bf16_kernel(const float *__restrict__ x, __nv_bfloat16 *__restrict__ xb, long long n4)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const float4 v = __ldg(reinterpret_cast<const float4 *>(x) + i);
    reinterpret_cast<uint2 *>(xb)[i] = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
}

// weights [Cout][Cin][K] fp32 -> [K][Npad][Ktot] bf16, K axis = [seg0 padded to 64 | seg1 padded to 64], zero padded
__global__ void pack_tc_kernel(const float *__restrict__ w, const float *__restrict__ scale, const float *__restrict__ shift,
                               __nv_bfloat16 *__restrict__ wp, float2 *__restrict__ ss, int Cout, int Cin0, int Cin1, int K,
                               int Npad, int Ktot)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n = (long long)K * Npad * Ktot;
    if (i < n) {
        const int ks = (int)(i % Ktot);
        const int co = (int)((i / Ktot) % Npad);
        const int t = (int)(i / ((long long)Ktot * Npad));
        const int seg1_base = (Cin0 + 63) / 64 * 64;
        int ci = -1;
        if (ks < seg1_base) { if (ks < Cin0) ci = ks; }
        else { if (ks - seg1_base < Cin1) ci = Cin0 + (ks - seg1_base); }
        float v = 0.f;
        if (co < Cout && ci >= 0) v = w[((size_t)co * (Cin0 + Cin1) + ci) * K + t];
        wp[i] = __float2bfloat16(v);
    }
    if (i < Npad) ss[i] = (i < Cout) ? make_float2(scale[i], shift[i]) : make_float2(0.f, 0.f);
}

// experimental: the extra K slot of a merged tail chunk, [t][co][Ktot - 64 + j]: j < s -> skip tail channel, j < s + u ->
// upsampled tail channel, else 0 (the regular slots are written by pack_tc_kernel, which leaves this one untouched = 0)
__global__ void pack_tc_merged_kernel(const float *__restrict__ w, __nv_bfloat16 *__restrict__ wp, int Cout, int Cin0, int Cin1,
                                      int K, int Npad, int Ktot, int s, int u)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n = (long long)K * Npad * 64;
    if (i >= n) return;
    const int j = (int)(i % 64);
    const int co = (int)((i / 64) % Npad);
    const int t = (int)(i / (64LL * Npad));
    int ci = -1;
    if (j < s) ci = Cin0 + (Cin1 / 64) * 64 + j;
    else if (j < s + u) ci = (Cin0 / 64) * 64 + (j - s);
    float v = 0.f;
    if (co < Cout && ci >= 0) v = w[((size_t)co * (Cin0 + Cin1) + ci) * K + t];
    wp[((size_t)t * Npad + co) * Ktot + (Ktot - 64) + j] = __float2bfloat16(v);
}

// split-precision ("fp32_tc") weights: K-loop position c of a block multiplies the data part (hi / lo) of one 64-channel chunk
// with the high or the low bf16 part of the fp32 weights; SplitTable lists, per position, the first original input channel of
// the chunk, its width and which weight part it takes. wp[t][co][c * 64 + j], zero beyond the chunk's width (the TMA box of a
// chunk narrower than 64 channels reads on into the next channels of the row: they meet zero weights).
struct SplitTable { short base[48]; unsigned char width[48], wlo[48]; int n; };
__global__ void pack_tc_split_kernel(const float *__restrict__ w, __nv_bfloat16 *__restrict__ wp, int Cout, int Cin, int K, int Npad,
                                     const SplitTable tab)
{
    const int Ktot = tab.n * 64;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)K * Npad * Ktot) return;
    const int ks = (int)(i % Ktot);
    const int co = (int)((i / Ktot) % Npad);
    const int t = (int)(i / ((long long)Ktot * Npad));
    const int c = ks >> 6, j = ks & 63;
    float v = 0.f;
    if (co < Cout && j < tab.width[c]) {
        const float wf = w[((size_t)co * Cin + tab.base[c] + j) * K + t];
        const float hi = __bfloat162float(__float2bfloat16_rn(wf));
        v = tab.wlo[c] ? wf - hi : hi;
    }
    wp[i] = __float2bfloat16_rn(v);
}

// [B][L][2C] ([hi | lo] bf16 halves) -> [B][C][L] fp32 (read_level of the split-precision path)
__global__ void nlc_split_to_ncl_f32_kernel(const __nv_bfloat16 *__restrict__ src, float *__restrict__ dst, int B, int L, int C)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n = (long long)B * C * L;
    if (i >= n) return;
    const int l = (int)(i % L);
    const int c = (int)((i / L) % C);
    const int b = (int)(i / ((long long)L * C));
    const __nv_bfloat16 *row = src + ((size_t)b * L + l) * (2 * C);
    dst[i] = __bfloat162float(row[c]) + __bfloat162float(row[C + c]);
}

__global__ void nlc_bf16_to_ncl_f32_kernel(const __nv_bfloat16 *__restrict__ src, float *__restrict__ dst, int B, int L, int C)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;       // index into dst [B][C][L]
    const long long n = (long long)B * C * L;
    if (i >= n) return;
    const int l = (int)(i % L);
    const int c = (int)((i / L) % C);
    const int b = (int)(i / ((long long)L * C));
    dst[i] = __bfloat162float(src[((size_t)b * L + l) * C + c]);
}

// -------------------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct TcLevel {
    int cin0, cin1, cout, k;
    int Npad, Ktot;
    int mg_s = 0, mg_u = 0;            // merged tail chunk: channel tails of the skip / upsampled segment that share
                                       // one extra 64-wide K slot at the end of the packed weights (0 = not merged)
    __nv_bfloat16 *wp = nullptr;
    float2 *ss = nullptr;
    float *w_f32 = nullptr;            // library-owned fp32 copy of the block's weights (source of the expansions made at plan time)
    __nv_bfloat16 *wx = nullptr;       // Toeplitz-expanded weights of the dense bottom-of-U GEMM (gemm_tc_kernel), built for wx_L positions
    int wx_L = 0;
    size_t wx_elems = 0;
    __nv_bfloat16 *wp_sp = nullptr;    // split-precision packing [K][Npad][sp_chunks * 64] (sp_chunk_order lists the K-loop positions)
    int sp_chunks = 0;
    const float *w_src = nullptr;      // enc0 only: fp32 weights (w_own, a library-owned copy) / scale / shift (the context's folded copies)
    float *w_own = nullptr;            // enc0 only: [Cout][1][K] fp32 copy made by tc_set_weights (the caller's tensor is not read afterwards)
    const float *scale = nullptr, *shift = nullptr;
};

static int sp_chunk_order(const TcLevel &lv, bool dec, unsigned char *map, SplitTable *tab);

struct TcPlanLevel {
    TcParams p;
    GemmParams gp;                     // is_gemm: the block runs gemm_tc_kernel (tmA / tmO = its two sources, tmW = expanded weights)
    bool is_gemm = false;
    CUtensorMap tmA, tmW, tmO;
    dim3 grid;
    int threads;
    int per_sm;
    size_t smem;
    bool upcat;
    bool small;                        // two-CTAs-per-SM kernel flavour
    int kind = 0;                      // reported by wunet_debug_plan in the 'small' field: 2 = dense GEMM over frames (gemm_tc_kernel)
    int pair = 0;                      // row-pair mode: 1 = encoder block (conv_tc_kernel<9, false, ...>), 
                                       // 3 = block 0 over groups of 8 samples (<3, false, ...>)
};

// Per-block tiling overrides for tuning sweeps: WUNET_TC_OVR="<block>:key=val,key=val;<block>:..." with keys
// mt, ns (column splits), na, nacc, tg, res (0/1), small (0/1), packed (1: pack L=128 frames). Unset keys keep
// the heuristic's choice.
struct TcOverride { int mt = 0, ns = 0, na = 0, nacc = 0, tg = 0, nb = 0, res = -1, small = -1, packed = -1; bool any = false; };
static void parse_kv(const std::string &seg, TcOverride &ov)
{
    size_t q = 0;
    while (q < seg.size()) {
        size_t qe = seg.find(',', q);
        if (qe == std::string::npos) qe = seg.size();
        const std::string kv = seg.substr(q, qe - q);
        q = qe + 1;
        const size_t eq = kv.find('=');
        if (eq == std::string::npos) continue;
        const std::string k = kv.substr(0, eq);
        const int v = atoi(kv.c_str() + eq + 1);
        if (k == "mt") ov.mt = v; else if (k == "ns") ov.ns = v; else if (k == "na") ov.na = v;
        else if (k == "nacc") ov.nacc = v; else if (k == "tg") ov.tg = v; else if (k == "res") ov.res = v;
        else if (k == "small") ov.small = v; else if (k == "packed") ov.packed = v;
        else if (k == "nb") ov.nb = v;
        ov.any = true;
    }
}
static TcOverride parse_override(const std::string &env, int block)
{
    TcOverride ov;
    size_t pos = 0;
    while (pos < env.size()) {
        size_t end = env.find(';', pos);
        if (end == std::string::npos) end = env.size();
        const std::string seg = env.substr(pos, end - pos);
        pos = end + 1;
        const size_t colon = seg.find(':');
        if (colon == std::string::npos || atoi(seg.substr(0, colon).c_str()) != block) continue;
        parse_kv(seg.substr(colon + 1), ov);
    }
    return ov;
}

struct TcPlan {
    std::vector<TcPlanLevel> lv;       // index 1..2n (0 = enc0 handled separately)
    std::vector<size_t> off;           // workspace offsets of the 2n+1 block outputs (+ the even-row copy of block 0)
    bool even_copy = false;            // block 1 runs in row-pair mode: enc0 also writes its even rows densely (off[2n+1])
    bool enc0_tc = false;              // block 0 runs on the tensor cores (lv[0]; input converted to bf16 at off[2n+2])
};

struct TcState {
    int n = 0, ci = 0;
    std::vector<TcLevel> levels;       // 2n+1
    const float *out_w = nullptr, *out_b = nullptr;
    EncodeTiledFn encode = nullptr;
    bool store_last = false;           // WUNET_TC_STORE_LAST=1: also materialise the last decoder block (tests)
    int enc_l2promo = 256;             // L2 promotion of the encoders' decimated input views (WUNET_TC_L2PROMO = 0 / 64 / 128 / 256)
    bool attr_set = false;
    bool pdl = false;                  // programmatic dependent launch between the blocks (WUNET_TC_PDL=1); measured slower, off
    bool merge = true;                 // merged tail chunks (WUNET_TC_MERGE=0 switches them off for A/B measurements)
    bool pf_late = true;               // see TcParams::pf_late; WUNET_TC_PFLATE=0 switches it off (A/B measurements, tests). Since the
                                       // taps of a stage share one wgmma group, the late prefetch is the faster one (dec4 ... dec10, H100)
    bool gemm = true;                  // dense GEMM over frames for blocks of at most 16 samples (WUNET_TC_GEMM=0 switches it off)
    // row-pair mode (WUNET_TC_PAIR bit 0: first tensor-core encoder block, bit 1: last decoder block + head): virtual blocks with
    // doubled channel counts and Toeplitz-expanded weights (pair_weight), planned on frames of half the length
    int pair_mask = 1;                 // default: block 1 in row-pair mode (enc0 also writes a dense copy of its even rows)
    int enc0_v = 0;                    // WUNET_TC_ENC0V: 2 = persistent form of the CUDA-core enc0 kernel (bit-identical), 1 = one tile per block,
                                       // 0 (default) = persistent for the split-precision path (two blocks per SM there), one
                                       // tile per block for bf16 (four blocks per SM overlap their phases already)
    bool enc0_tc = false;              // WUNET_TC_ENC0=1: block 0 on the tensor cores in its group-of-8 form (group8_weight); bf16 mode only
    bool enc0_ok = false;
    TcLevel g8_lv;                     // its virtual block: 8 input channels, 8 C columns, 3 taps
    float *g8_w = nullptr, *g8_scale = nullptr, *g8_shift = nullptr;
    TcLevel pair_lv[2];                // [0] block 1, [1] block 2n (cin0 / cin1 / cout = virtual counts, k = pair taps)
    float *pair_w[2] = {nullptr, nullptr}, *pair_scale[2] = {nullptr, nullptr}, *pair_shift[2] = {nullptr, nullptr};
    bool pair_ok[2] = {false, false};
    int num_sms = 148;                 // SM count the plan and the persistent grids are sized for (WUNET_TC_SMS, else dev_sms)
    int dev_sms = 148;                 // the device's multiprocessor count
    cudaStream_t copy_in = nullptr, copy_out = nullptr;     // host pipeline: H2D / D2H streams
    cudaEvent_t ev_in[8] = {}, ev_out[8] = {};
    long long *trace = nullptr;        // development: WUNET_TC_TRACE builds + WUNET_TC_TRACE_LEVEL=<block>
    int trace_level = -1;
    // plan cache, keyed on (workspace pointer, B, T)
    const void *plan_ws = nullptr;
    int plan_B = 0, plan_T = 0;
    const float *plan_x = nullptr;
    float *plan_y = nullptr;
    std::string plan_ovr;              // WUNET_TC_OVR value the cached plan was built with
    int plan_sms = 0;                  // num_sms the cached plan was built with
    int plan_mode = 0;                 // 0: bf16 plan, 1: split-precision (fp32_tc) plan
    TcPlan plan;
};

const char *tc_error() { return g_tc_err; }

// off[0 .. 2n] = block outputs; off[2n+1] = dense copy of block 0's even rows [B][T/2][ci] (bf16 mode; row-pair mode of block 1);
// off[2n+2] = the raw input in bf16
static void tc_layout(int n, int ci, int B, int T, std::vector<size_t> &off, size_t &total, int mode = 0)
{
    off.resize(2 * n + 3);
    size_t cur = 0;
    for (int i = 0; i < 2 * n + 1; ++i) {
        const int L = (i <= n) ? (T >> i) : (T >> (2 * n - i));
        const int cout = (i < n) ? (i + 1) * ci : (i == n ? n * ci : (2 * n - i + 1) * ci);
        off[i] = cur;
        cur += round_up_sz((size_t)B * L * cout * sizeof(__nv_bfloat16) * (mode ? 2 : 1), 1024);
    }
    off[2 * n + 1] = cur;
    if (mode == 0) cur += round_up_sz((size_t)B * (T / 2) * ci * sizeof(__nv_bfloat16), 1024);
    off[2 * n + 2] = cur;                                 // bf16 copy of the raw input [B][T] (block 0 on the tensor cores)
    if (mode == 0) cur += round_up_sz((size_t)B * T * sizeof(__nv_bfloat16), 1024);
    total = cur + 1024;
}

size_t tc_workspace_bytes(int n, int ci, int B, int T, int mode)
{
    std::vector<size_t> off;
    size_t total;
    tc_layout(n, ci, B, T, off, total, mode);
    return total;
}

// K segments and padded sizes of every block: encoders have one input segment, decoder block i concatenates the previous
// block's (upsampled) output with the skip of encoder 2n - i (model/unet_basic.py:93-95)
static void derive_levels(std::vector<TcLevel> &levels, const TcBlockSrc *blocks, int nblocks, int n, bool merge = true)
{
    for (int i = 0; i < nblocks; ++i) {
        TcLevel &lv = levels[i];
        lv.cout = blocks[i].cout; lv.k = blocks[i].k;
        if (i <= n) { lv.cin0 = blocks[i].cin; lv.cin1 = 0; }
        else { lv.cin0 = levels[i - 1].cout; lv.cin1 = blocks[i].cin - lv.cin0; }
        lv.Npad = round_up(lv.cout, 16);
        lv.Ktot = round_up(lv.cin0, 64) + (lv.cin1 ? round_up(lv.cin1, 64) : 0);
        lv.w_src = blocks[i].w; lv.scale = blocks[i].scale; lv.shift = blocks[i].shift;
        lv.mg_s = lv.mg_u = 0;
        const int u = lv.cin0 % 64, sk = lv.cin1 % 64;
        if (merge && i > n && u > 0 && sk > 0 && u + sk <= 64 && u % 8 == 0 && sk % 8 == 0) {
            lv.mg_s = sk; lv.mg_u = u;
            lv.Ktot += 64;                                  // slot [skip tail | upsampled tail | 0] after the regular slots
        }
    }
}

int tc_set_weights(TcState **pst, int n, int ci, const TcBlockSrc *blocks, int nblocks, const float *out_w,
                   const float *out_b, cudaStream_t stream)
{
    if (nblocks != 2 * n + 1) return tc_fail("bad block count");
    TcState *st = *pst;
    if (!st) {
        st = new TcState();
        st->n = n; st->ci = ci;
        st->levels.resize(nblocks);
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) {
            delete st;
            return tc_fail("cuTensorMapEncodeTiled not available from the driver");
        }
        st->encode = reinterpret_cast<EncodeTiledFn>(fn);
        const char *e = getenv("WUNET_TC_STORE_LAST");
        st->store_last = e && e[0] == '1';
        const char *pe = getenv("WUNET_TC_PDL");
        st->pdl = pe && pe[0] == '1';
        if (const char *xe = getenv("WUNET_TC_MERGE")) st->merge = xe[0] != '0';
        if (const char *xe = getenv("WUNET_TC_PFLATE")) st->pf_late = xe[0] != '0';
        if (const char *xe = getenv("WUNET_TC_GEMM")) st->gemm = xe[0] != '0';
        if (const char *xe = getenv("WUNET_TC_L2PROMO")) st->enc_l2promo = atoi(xe);
        if (const char *xe = getenv("WUNET_TC_PAIR")) st->pair_mask = atoi(xe) & 3;
        if (const char *xe = getenv("WUNET_TC_ENC0")) st->enc0_tc = xe[0] == '1';
        if (const char *xe = getenv("WUNET_TC_ENC0V")) st->enc0_v = atoi(xe) == 2 ? 2 : (atoi(xe) == 1 ? 1 : 0);
#ifdef WUNET_TC_TRACE
        if (const char *tl = getenv("WUNET_TC_TRACE_LEVEL")) {
            st->trace_level = atoi(tl);
            cudaMalloc(&st->trace, 5 * 512 * sizeof(long long));
            cudaMemset(st->trace, 0, 5 * 512 * sizeof(long long));
        }
#endif
        *pst = st;
    }
    st->out_w = out_w; st->out_b = out_b;
    st->plan_ws = nullptr;                               // weights moved: rebuild maps lazily
    derive_levels(st->levels, blocks, nblocks, n, st->merge);
    if (ci % 8 != 0 || ci > 32) return 0;                // tensor-core path unsupported for this plan; forward reports it
    {
        // enc0 runs on CUDA cores from fp32 weights: keep a library-owned copy (include/wunet_b200.h: the caller's tensors are
        // only read during wunet_set_weights)
        TcLevel &l0 = st->levels[0];
        const size_t wn = (size_t)l0.cout * blocks[0].cin * l0.k * sizeof(float);
        if (!l0.w_own && cudaMalloc(&l0.w_own, wn) != cudaSuccess) return tc_fail("cudaMalloc(enc0 weights) failed");
        if (cudaMemcpyAsync(l0.w_own, blocks[0].w, wn, cudaMemcpyDeviceToDevice, stream) != cudaSuccess)
            return tc_fail("enc0 weight copy failed");
        l0.w_src = l0.w_own;
    }
    for (int i = 1; i < nblocks; ++i) {                  // enc0 runs on CUDA cores from the fp32 weights
        TcLevel &lv = st->levels[i];
        const size_t nel = (size_t)lv.k * lv.Npad * lv.Ktot;
        if (!lv.wp) {
            if (cudaMalloc(&lv.wp, nel * sizeof(__nv_bfloat16)) != cudaSuccess) return tc_fail("cudaMalloc(wp) failed");
            if (cudaMalloc(&lv.ss, lv.Npad * sizeof(float2)) != cudaSuccess) return tc_fail("cudaMalloc(ss) failed");
        }
        pack_tc_kernel<<<(unsigned)((nel + 255) / 256), 256, 0, stream>>>(blocks[i].w, blocks[i].scale, blocks[i].shift, lv.wp,
                                                                          lv.ss, lv.cout, lv.cin0, lv.cin1, lv.k, lv.Npad, lv.Ktot);
        if (cudaGetLastError() != cudaSuccess) return tc_fail("pack_tc_kernel launch failed");
        {
            const size_t wn = (size_t)lv.cout * (lv.cin0 + lv.cin1) * lv.k;
            if (!lv.w_f32 && cudaMalloc(&lv.w_f32, wn * sizeof(float)) != cudaSuccess) return tc_fail("cudaMalloc(w_f32) failed");
            if (cudaMemcpyAsync(lv.w_f32, blocks[i].w, wn * sizeof(float), cudaMemcpyDeviceToDevice, stream) != cudaSuccess)
                return tc_fail("weight copy failed");
            lv.wx_L = 0;                                   // expansions are rebuilt with the next plan
        }
        {
            // split-precision packing (fp32_tc): [K][Npad][positions * 64] in the split K-loop order
            SplitTable tab;
            lv.sp_chunks = sp_chunk_order(lv, i > n, nullptr, &tab);
            const size_t ns = (size_t)lv.k * lv.Npad * lv.sp_chunks * 64;
            if (!lv.wp_sp && cudaMalloc(&lv.wp_sp, ns * sizeof(__nv_bfloat16)) != cudaSuccess) return tc_fail("cudaMalloc(wp_sp) failed");
            pack_tc_split_kernel<<<(unsigned)((ns + 255) / 256), 256, 0, stream>>>(blocks[i].w, lv.wp_sp, lv.cout, lv.cin0 + lv.cin1, lv.k,
                                                                                  lv.Npad, tab);
            if (cudaGetLastError() != cudaSuccess) return tc_fail("pack_tc_split_kernel launch failed");
        }
        if (lv.mg_s) {
            const size_t nm = (size_t)lv.k * lv.Npad * 64;
            pack_tc_merged_kernel<<<(unsigned)((nm + 255) / 256), 256, 0, stream>>>(blocks[i].w, lv.wp, lv.cout, lv.cin0, lv.cin1, lv.k,
                                                                                    lv.Npad, lv.Ktot, lv.mg_s, lv.mg_u);
            if (cudaGetLastError() != cudaSuccess) return tc_fail("pack_tc_merged_kernel launch failed");
        }
    }
    // block 0 on the tensor cores: virtual block of 8 input channels x 8 C columns x 3 taps
    st->enc0_ok = false;
    if (st->enc0_tc && st->levels[0].k == 15 && blocks[0].cin == 1 && 8 * st->levels[0].cout <= 256 && st->levels[0].cout % 8 == 0) {
        const TcLevel &rl = st->levels[0];
        TcLevel &pv = st->g8_lv;
        pv.cin0 = 8; pv.cin1 = 0; pv.cout = 8 * rl.cout; pv.k = 3;
        pv.Npad = round_up(pv.cout, 16); pv.Ktot = 64;
        pv.mg_s = pv.mg_u = 0;
        const size_t nv = (size_t)pv.cout * 8 * 3, nel = (size_t)3 * pv.Npad * pv.Ktot;
        if (!st->g8_w) {
            if (cudaMalloc(&st->g8_w, nv * sizeof(float)) != cudaSuccess || cudaMalloc(&st->g8_scale, pv.cout * sizeof(float)) != cudaSuccess ||
                cudaMalloc(&st->g8_shift, pv.cout * sizeof(float)) != cudaSuccess || cudaMalloc(&pv.wp, nel * sizeof(__nv_bfloat16)) != cudaSuccess ||
                cudaMalloc(&pv.ss, pv.Npad * sizeof(float2)) != cudaSuccess)
                return tc_fail("cudaMalloc(block 0 tensor-core weights) failed");
        }
        expand_group8_weights_kernel<<<(unsigned)((nv + 255) / 256), 256, 0, stream>>>(blocks[0].w, blocks[0].scale, blocks[0].shift, st->g8_w,
                                                                                       st->g8_scale, st->g8_shift, rl.cout, rl.k);
        if (cudaGetLastError() != cudaSuccess) return tc_fail("expand_group8_weights_kernel launch failed");
        pack_tc_kernel<<<(unsigned)((nel + 255) / 256), 256, 0, stream>>>(st->g8_w, st->g8_scale, st->g8_shift, pv.wp, pv.ss, pv.cout, 8, 0, 3,
                                                                          pv.Npad, pv.Ktot);
        if (cudaGetLastError() != cudaSuccess) return tc_fail("pack_tc_kernel (block 0) launch failed");
        st->enc0_ok = true;
    }
    // row-pair mode: virtual blocks (doubled channel counts, pair_taps(k) taps) packed like any other block
    for (int s = 0; s < 1; ++s) {
        st->pair_ok[s] = false;
        if (!(st->pair_mask & (1 << s)) || n < 2) continue;
        const int i = s == 0 ? 1 : 2 * n;
        const TcLevel &rl = st->levels[i];
        // block 1: 15 taps -> 9 over pairs, the whole virtual input in one 64-channel chunk; last block: 5 taps -> 3, fused head over
        // two samples per row (Cout a multiple of 8, at most 32), its upsampled input at least one full range of 32 channels
        if (s == 0 && !(rl.k == 15 && rl.cin1 == 0 && rl.cin0 % 8 == 0 && 2 * rl.cin0 <= 64 && 2 * rl.cout <= 256)) continue;
        if (s == 1 && !(rl.k == 5 && rl.cin0 % 8 == 0 && rl.cin1 % 8 == 0 && rl.cin0 >= 32 && rl.cout % 8 == 0 && rl.cout <= 32)) continue;
        TcLevel &pv = st->pair_lv[s];
        const int kp = pair_taps(rl.k);
        pv.cin0 = 2 * rl.cin0; pv.cin1 = 2 * rl.cin1; pv.cout = 2 * rl.cout; pv.k = kp;
        pv.Npad = round_up(pv.cout, 16);
        pv.Ktot = round_up(pv.cin0, 64) + (pv.cin1 ? round_up(pv.cin1, 64) : 0);
        pv.mg_s = pv.mg_u = 0;
        const size_t nv = (size_t)pv.cout * (pv.cin0 + pv.cin1) * kp;
        const size_t nel = (size_t)kp * pv.Npad * pv.Ktot;
        if (!st->pair_w[s]) {
            if (cudaMalloc(&st->pair_w[s], nv * sizeof(float)) != cudaSuccess || cudaMalloc(&st->pair_scale[s], pv.cout * sizeof(float)) != cudaSuccess ||
                cudaMalloc(&st->pair_shift[s], pv.cout * sizeof(float)) != cudaSuccess || cudaMalloc(&pv.wp, nel * sizeof(__nv_bfloat16)) != cudaSuccess ||
                cudaMalloc(&pv.ss, pv.Npad * sizeof(float2)) != cudaSuccess)
                return tc_fail("cudaMalloc(row-pair weights) failed");
        }
        expand_pair_weights_kernel<<<(unsigned)((nv + 255) / 256), 256, 0, stream>>>(blocks[i].w, blocks[i].scale, blocks[i].shift, st->pair_w[s],
                                                                                     st->pair_scale[s], st->pair_shift[s], rl.cout, rl.cin0,
                                                                                     rl.cin1, rl.k, s == 1 ? 1 : 0);
        if (cudaGetLastError() != cudaSuccess) return tc_fail("expand_pair_weights_kernel launch failed");
        pack_tc_kernel<<<(unsigned)((nel + 255) / 256), 256, 0, stream>>>(st->pair_w[s], st->pair_scale[s], st->pair_shift[s], pv.wp, pv.ss,
                                                                          pv.cout, pv.cin0, pv.cin1, kp, pv.Npad, pv.Ktot);
        if (cudaGetLastError() != cudaSuccess) return tc_fail("pack_tc_kernel (row-pair) launch failed");
        st->pair_ok[s] = true;
    }
    return 0;
}

// l2promo: L2 fetch granularity of the map's loads in bytes (0 = none). The decimated views of the encoders (every second row)
// take a smaller one than the dense views: with 256-byte promotion the skipped rows are fetched from DRAM as well.
static int make_map(TcState *st, CUtensorMap *m, const void *base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t s1_bytes,
                    uint64_t s2_bytes, uint32_t b0, uint32_t b1, uint32_t b2, int l2promo = 256)
{
    cuuint64_t gdim[3] = {d0, d1, d2};
    cuuint64_t gstr[2] = {s1_bytes, s2_bytes};
    cuuint32_t box[3] = {b0, b1, b2};
    cuuint32_t estr[3] = {1, 1, 1};
    const CUtensorMapL2promotion promo = l2promo >= 256 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B
                                         : l2promo >= 128 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B
                                         : l2promo >= 64 ? CU_TENSOR_MAP_L2_PROMOTION_L2_64B : CU_TENSOR_MAP_L2_PROMOTION_NONE;
    const CUresult r = st->encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void *>(base), gdim, gstr, box, estr,
                                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, promo,
                                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return tc_fail("cuTensorMapEncodeTiled failed (%d): dims %llu,%llu,%llu strides %llu,%llu box %u,%u,%u", (int)r,
                       (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2, (unsigned long long)s1_bytes,
                       (unsigned long long)s2_bytes, b0, b1, b2);
    return 0;
}

// K-loop order of a block in split-precision mode, built from the single-precision order (encoders: natural; decoders: full
// upsampled chunks, skip chunks, partial upsampled chunk - or the partial one first if it is the only one): per chunk, hi
// data x w_hi, the same operand stage x w_lo, lo data x w_hi. Fills chunk_map bytes (bit 7 upsampled segment, bit 6 low data part, bits 0-5 chunk
// index) and the table the weight packing follows. Returns the number of positions.
static int sp_chunk_order(const TcLevel &lv, bool dec, unsigned char *map, SplitTable *tab)
{
    unsigned char one[16];
    int k = 0;
    const int n0 = (lv.cin0 + 63) / 64, n1 = (lv.cin1 + 63) / 64, nfull0 = lv.cin0 / 64;
    if (!dec) { for (int c = 0; c < n0; ++c) one[k++] = (unsigned char)c; }
    else if (nfull0 == 0) {
        one[k++] = 0x80;
        for (int c = 0; c < n1; ++c) one[k++] = (unsigned char)c;
    } else {
        for (int c = 0; c < nfull0; ++c) one[k++] = (unsigned char)(0x80 | c);
        for (int c = 0; c < n1; ++c) one[k++] = (unsigned char)c;
        if (nfull0 < n0) one[k++] = (unsigned char)(0x80 | nfull0);
    }
    int n = 0;
    auto put = [&](int c, bool lo_data, bool w_lo, bool reuse) {
        const bool up = dec && (one[c] & 0x80);
        const int idx = one[c] & 0x1f;
        if (map) map[n] = (unsigned char)(one[c] | (lo_data ? 0x40 : 0) | (reuse ? 0x20 : 0));
        if (tab) {
            const int seg = (up || !dec) ? lv.cin0 : lv.cin1;
            tab->base[n] = (short)(((up || !dec) ? 0 : lv.cin0) + 64 * idx);
            tab->width[n] = (unsigned char)std::min(64, seg - 64 * idx);
            tab->wlo[n] = (unsigned char)w_lo;
        }
        ++n;
    };
    for (int c = 0; c < k; ++c) {
        put(c, false, false, false);      // hi data x w_hi
        put(c, false, true, true);        // the same operand stage x w_lo
        put(c, true, false, false);       // lo data x w_hi (the next stage: the producers fill it together with the hi stage)
    }
    if (tab) tab->n = n;
    return n;
}

// Tiling decision for conv block i: pure host logic (no CUDA calls), so that tests can exercise it without a GPU
// (wunet_debug_plan). Fills every tiling field of P.p and the launch shape; pointers and tensor maps are added by build_plan.
// hd_mt > 0: the block is the last one and only the network output is wanted (head-only instantiation, see build_plan): M
// sub-tiles per CTA for it, so that the ring of previous-level rows fits next to the input ring (small flavour only).
// pair: row-pair mode - lv is the virtual block (doubled channel counts, pair taps) and the frames are half as long.
static int plan_block(const TcLevel &lv, int i, int n, int B, int T, int num_sms, const std::string &ovr, TcPlanLevel &P, bool sp = false,
                      int hd_mt = 0, bool pair = false, bool group8 = false)
{
    TcParams &p = P.p;
    memset(&p, 0, sizeof(p));
    const bool dec = i > n;
    const int KS = lv.k;
    const int L = ((i <= n) ? (T >> i) : (T >> (2 * n - i))) >> (pair ? 1 : (group8 ? 3 : 0));   // group8: block 0 over groups of 8 samples
    P.pair = pair ? (dec ? 2 : 1) : (group8 ? 3 : 0);
    P.upcat = dec;
    p.B = B; p.L = L; p.Cout = lv.cout; p.T = T;
    p.Cin0 = lv.cin0; p.Cin1 = lv.cin1;
    p.nchunks0 = (lv.cin0 + 63) / 64;
    p.nchunks = p.nchunks0 + (lv.cin1 + 63) / 64;
    p.Npad = lv.Npad;
    {
        // K-loop order. Encoders: natural. Decoders: full upsampled chunks, then the skip chunks (TMA), then the partial
        // upsampled chunk: a TMA chunk is never preceded by a short chunk, so its load latency hides behind MMAs.
        int k = 0;
        if (sp) {
            p.split = 1;
            p.nchunks = sp_chunk_order(lv, dec, p.chunk_map, nullptr);
        } else if (!dec) { for (int c = 0; c < p.nchunks; ++c) p.chunk_map[k++] = (unsigned char)c; }
        else if (pair) {
            // row-pair decoder: all upsampled chunks first (they are produced in one phase into consecutive ring stages), then the skip chunks
            const int n1 = p.nchunks - p.nchunks0;
            for (int c = 0; c < p.nchunks0; ++c) p.chunk_map[k++] = (unsigned char)(0x80 | c);
            for (int c = 0; c < n1; ++c) p.chunk_map[k++] = (unsigned char)c;
        } else if (lv.mg_s && L >= 128) {
            // experimental: [full upsampled chunks][full skip chunks][skip tail | upsampled tail] - one chunk fewer
            const int nfull0 = lv.cin0 / 64, nfull1 = lv.cin1 / 64;
            for (int c = 0; c < nfull0; ++c) p.chunk_map[k++] = (unsigned char)(0x80 | c);
            for (int c = 0; c < nfull1; ++c) p.chunk_map[k++] = (unsigned char)c;
            p.chunk_map[k++] = (unsigned char)0x40;
            p.nchunks = k;
            p.mg = 1;
            p.mg_vo = lv.mg_s / 8; p.mg_nvec = lv.mg_u / 8;
            p.mg_nk = (lv.mg_s + lv.mg_u + 15) / 16;
            p.mg_kslot = lv.Ktot / 64 - 1;
            p.mg_skip_idx = nfull1; p.mg_up_idx = nfull0;
        } else {
            const int nfull0 = lv.cin0 / 64, n1 = p.nchunks - p.nchunks0;
            if (nfull0 == 0) {
                // the only upsampled chunk is partial (e.g. the last decoder: 48 + 24 channels): produce it FIRST, so that its
                // shared-memory stage is released half a tile before the producers need it again
                p.chunk_map[k++] = (unsigned char)0x80;
                for (int c = 0; c < n1; ++c) p.chunk_map[k++] = (unsigned char)c;
            } else {
                for (int c = 0; c < nfull0; ++c) p.chunk_map[k++] = (unsigned char)(0x80 | c);
                for (int c = 0; c < n1; ++c) p.chunk_map[k++] = (unsigned char)c;
                if (nfull0 < p.nchunks0) p.chunk_map[k++] = (unsigned char)(0x80 | nfull0);
            }
        }
        if (p.nchunks > 48) return tc_fail("too many K chunks");
    }
    // ---- tiling ---------------------------------------------------------------------------------
    TcOverride ov = parse_override(ovr, i);
    const bool small = ov.small > 0 && !sp;
    const int smem_limit = small ? kSmemLimitSmall : kSmemLimit;
    P.small = small;
    const bool packed = L < 128 || (ov.packed > 0 && L + KS - 1 <= 256);
    auto geometry = [&](int MT, int nsplit) {
        p.nsplit = nsplit;
        p.Nh = nsplit == 1 ? lv.Npad : round_up((lv.Npad + nsplit - 1) / nsplit, 16);
        p.Nstride = round_up(p.Nh, 32);
        p.MT = MT;
        if (!packed) {
            p.packed = 0;
            p.tiles_per_frame = (L + 128 * MT - 1) / (128 * MT);
            const int rows = 128 * MT + KS - 1;
            p.nops = (rows + 255) / 256;
            p.R1 = round_up((rows + p.nops - 1) / p.nops, 8);
            p.S = 0; p.FR = 1;
            p.rows_used = rows;
            p.a_stage_bytes = (uint32_t)round_up(p.nops * p.R1 * 128, 1024);
            p.a_tx_bytes = p.nops * p.R1 * 128;
            p.m_tiles = B * p.tiles_per_frame;
        } else {
            p.packed = 1;
            p.S = L + KS - 1;
            int FR = (128 * MT - L) / p.S + 1;
            if (FR > B) FR = B;
            if (FR > 256) FR = 256;
            p.FR = FR;
            p.tiles_per_frame = 0;
            p.nops = 1; p.R1 = p.S;
            p.rows_used = FR * p.S;
            const int rows_alloc = round_up(std::max(FR * p.S, 128 * MT + KS - 1), 8);
            p.a_stage_bytes = (uint32_t)round_up(rows_alloc * 128, 1024);
            p.a_tx_bytes = FR * p.S * 128;
            p.m_tiles = (B + FR - 1) / FR;
        }
        p.nacc = 1;
        p.tmem_cols = 0;
    };
    // One 128-row M tile per CTA (MT = 1): the accumulators are registers of the consumer warpgroups, at most kAccColsLarge /
    // kAccColsSmall columns per CTA, so wider blocks are split over CTAs by columns.
    const int nh_max = small ? kAccColsSmall : kAccColsLarge;
    int ns = std::max(ov.ns > 0 ? ov.ns : 1, (lv.Npad + nh_max - 1) / nh_max);
    geometry(1, ns);
    while (p.Nh > nh_max) geometry(1, ++ns);
    if (packed && ov.ns <= 0) {
        // bottom of the U: few tiles, long K loops. As many column splits as still fit in one wave of tiles (each CTA then
        // streams a smaller share of the weights from L2).
        const int m_tiles = p.m_tiles;
        for (int cand : {2, 3, 4, 6}) {
            if (cand <= ns) continue;
            const int nh = round_up((lv.Npad + cand - 1) / cand, 16);
            if (m_tiles * cand <= num_sms && nh >= 48 && (cand - 1) * nh < lv.Npad) ns = cand;
        }
        geometry(1, ns);
    }
    if ((p.nsplit - 1) * p.Nh >= lv.Npad) return tc_fail("level %d: %d column splits of %d leave an empty split", i, p.nsplit, p.Nh);
    // epilogue store mode (needs complete tiles of complete rows per warp)
    p.bulk_store = 0;
    p.n_epi = small ? kEpiWarpsSmall : kEpiWarpsLarge;
    p.resident = 0;
    const int ring_budget = smem_limit - 2048 - p.Npad * 8 - 512;
    if (!packed && p.nsplit == 1 && ov.res != 0) {
        // weights-resident mode: if the block's packed weights fit in shared memory next to the input ring, the persistent
        // CTA loads them once instead of re-streaming them from L2 for every tile (the L2->SM stream, not HBM and not the
        // tensor pipe, is what bounds the shallow blocks otherwise).
        {
            geometry(1, 1);
            const int stage = round_up(p.Nh * 128 * KS, 1024);
            const int wbytes = p.nchunks * stage;
            const int na = ov.na > 0 ? ov.na : ((dec && p.nchunks >= 3) ? 3 : 2);
            if (na * (int)p.a_stage_bytes + wbytes <= ring_budget) {
                p.resident = 1; p.na = na; p.tg = KS; p.ngroups = 1;
                p.b_stage_bytes = (uint32_t)stage;
                p.nb = p.nchunks * p.ngroups;
            }
        }
        if (!p.resident) geometry(1, 1);
    }
    if (!p.resident) {
        // A ring depth: decoders whose K chunks are short (5 taps, few K-steps) need the TMA/producers to run two chunks
        // ahead; everything else double-buffers. Weight stages hold `tg` consecutive taps (one TMA box, one handshake).
        const int na_want = ov.na > 0 ? ov.na : ((dec && !packed && p.nchunks >= 3 && p.MT <= 2) ? 3 : 2);
        bool ok = false;
        for (int na = na_want; na >= 1 && !ok; --na) {
            for (int tg = (ov.tg > 0 ? std::min(KS, ov.tg) : KS); tg >= 1; --tg) {
                // every stage handshake costs a ~400-cycle tensor-pipe bubble (trace, DESIGN.md): prefer the fattest stage
                // (most taps per handshake) that still leaves a 2-deep ring; taps past KS in the last group are zero-filled
                const int stage = round_up(p.Nh * 128 * tg, 1024);
                const int min_stages = 2;
                if (na * (int)p.a_stage_bytes + min_stages * stage > ring_budget) continue;
                p.na = na; p.tg = tg;
                p.ngroups = (KS + tg - 1) / tg;
                p.b_stage_bytes = (uint32_t)stage;
                int nb = (ring_budget - na * (int)p.a_stage_bytes) / stage;
                if (nb > kMaxBStages) nb = kMaxBStages;
                if (ov.nb >= min_stages && nb > ov.nb) nb = ov.nb;
                p.nb = nb;
                ok = true;
                break;
            }
        }
        if (!ok) return tc_fail("level %d does not fit in shared memory", i);
        if (ov.any && p.na < 2) return tc_fail("level %d: override leaves a single input stage", i);
    }
    {
        const int threads = 32 + 32 * (small ? kEpiWarpsSmall + (dec ? kProducerWarpsSmall : 0)
                                             : kEpiWarpsLarge + (dec ? kProducerWarpsLarge : 0));
        const int per_sm = std::max(1, std::min({(int)((228 * 1024) / (smem_total(p) + 1024)), small ? 2 : 1, 2048 / threads}));
        const int total_tiles = p.m_tiles * p.nsplit;
        p.tile_begin = 0; p.tile_end = total_tiles;
        P.per_sm = per_sm;
        P.grid = dim3((unsigned)std::min(total_tiles, num_sms * per_sm), 1, 1);
        P.threads = threads;
    }
    P.smem = smem_total(p);
    if (P.smem > (size_t)kSmemLimit) return tc_fail("level %d: smem %zu too large", i, P.smem);

    const bool last_block = (i == 2 * n);
    if (last_block && lv.cout > (pair ? 64 : 32)) return tc_fail("fused head needs channels_interval <= 32");
    if (dec && pair && p.na < p.nchunks0) return tc_fail("level %d: the row-pair producers fill %d ring stages at once, the ring has %d", i, p.nchunks0, p.na);
    if (last_block && p.packed) return tc_fail("bf16 path needs frames of at least 128 samples (T=%d): the fused head works on full frames", T);
    if (last_block && p.nsplit != 1) return tc_fail("fused head needs the whole channel range in one CTA");
    return 0;
}

// Dense GEMM over frames for a block of at most 16 samples (gemm_tc_kernel). Host logic only: shapes and the launch grid.
static bool plan_block_gemm(const TcLevel &lv, int i, int n, int B, int T, int num_sms, TcPlanLevel &P)
{
    const bool dec = i > n;
    const int L = (i <= n) ? (T >> i) : (T >> (2 * n - i));
    if (i < 1 || L > 16 || L < 1 || lv.cout % 8 != 0 || lv.cin0 % 8 != 0 || lv.cin1 % 8 != 0) return false;
    if (i == 2 * n) return false;                               // the last block carries the fused head
    if (B < 64) return false;                                   // small batches: the expanded weights (up to 65 MB per block) would be
                                                                // streamed for a mostly empty 128-frame row tile (B=3: 0.52 vs 0.46 ms)
    GemmParams &g = P.gp;
    memset(&g, 0, sizeof(g));
    g.B = B; g.L = L; g.cout = lv.cout; g.N = L * lv.cout;
    if (g.N % 16 != 0) return false;
    // columns per CTA: a multiple of 16 that divides N, giving about one CTA per SM (times the 256-frame row tiles)
    const int mtiles = (B + 127) / 128;
    int best = 16;
    for (int nh = 16; nh <= kAccColsLarge; nh += 16)
        if (g.N % nh == 0 && (g.N / nh) * mtiles >= num_sms * 3 / 4) best = nh;
    g.Nh = best;
    const int pad = (lv.k - 1) / 2;
    if (!dec) {
        g.npos[0] = L; g.cpp[0] = (lv.cin0 + 63) / 64; g.reach_lo[0] = -pad; g.reach_hi[0] = pad; g.halve[0] = 0;
        g.npos[1] = 0; g.cpp[1] = 0;
    } else {
        g.npos[0] = L / 2; g.cpp[0] = (lv.cin0 + 63) / 64; g.reach_lo[0] = -2; g.reach_hi[0] = 2; g.halve[0] = 1;
        g.npos[1] = L; g.cpp[1] = (lv.cin1 + 63) / 64; g.reach_lo[1] = -pad; g.reach_hi[1] = pad; g.halve[1] = 0;
        if (g.npos[0] < 1) return false;
    }
    g.a_bytes = 16384; g.w_bytes = (uint32_t)round_up(g.Nh * 128, 1024);
    g.cps = 4;
    int ns = (kSmemLimit - 2048) / (int)(g.cps * (g.a_bytes + g.w_bytes));
    while (ns < 2 && g.cps > 1) { --g.cps; ns = (kSmemLimit - 2048) / (int)(g.cps * (g.a_bytes + g.w_bytes)); }
    g.nstages = std::min(4, std::max(2, ns));
    P.is_gemm = true; P.upcat = dec; P.small = false; P.per_sm = 1; P.threads = kGemmThreads;
    P.kind = 2;
    P.smem = (size_t)g.nstages * g.cps * (g.a_bytes + g.w_bytes) + 8 * 16 + 1024;
    P.grid = dim3((unsigned)(g.N / g.Nh), (unsigned)mtiles, 1);
    TcParams &p = P.p;                                          // mirror what tests / tools read
    memset(&p, 0, sizeof(p));
    p.B = B; p.L = L; p.T = T; p.Cout = lv.cout; p.Cin0 = lv.cin0; p.Cin1 = lv.cin1; p.Npad = lv.Npad; p.Nh = g.Nh; p.nsplit = g.N / g.Nh;
    p.Nstride = g.Nh; p.MT = 1; p.nacc = 1; p.FR = 128; p.packed = 1; p.S = L; p.m_tiles = mtiles; p.nchunks = g.npos[0] * g.cpp[0] + g.npos[1] * g.cpp[1];
    p.na = g.nstages; p.nb = g.nstages; p.tg = 1; p.ngroups = 1; p.a_stage_bytes = g.cps * g.a_bytes; p.b_stage_bytes = g.cps * g.w_bytes;
    p.a_tx_bytes = (int)(g.cps * g.a_bytes); p.rows_used = 128; p.tmem_cols = 0; p.tile_begin = 0; p.tile_end = p.m_tiles * p.nsplit; p.n_epi = kEpiWarpsLarge;
    return true;
}

static int build_plan(TcState *st, const float *x, float *y, int B, int T, void *ws, int mode, cudaStream_t stream)
{
    const int n = st->n;
    TcPlan &pl = st->plan;
    size_t total;
    tc_layout(n, st->ci, B, T, pl.off, total, mode);
    pl.lv.assign(2 * n + 1, TcPlanLevel{});
    const bool sp = mode != 0;
    const uint64_t cm = sp ? 2 : 1;                      // stored channels per logical channel ([hi | lo] halves)
    char *base = static_cast<char *>(ws);
    auto lvl = [&](int i) { return reinterpret_cast<__nv_bfloat16 *>(base + pl.off[i]); };
    pl.even_copy = false;
    pl.enc0_tc = false;
    if (!sp && st->enc0_ok && T % 8 == 0 && T / 8 >= 128) {
        // block 0 on the tensor cores: a 3-tap encoder block over groups of 8 samples, reading the bf16 copy of the input
        TcPlanLevel &P = pl.lv[0];
        const TcLevel &lv = st->g8_lv;
        if (plan_block(lv, 0, n, B, T, st->num_sms, st->plan_ovr, P, false, 0, false, true)) return -1;
        TcParams &p = P.p;
        const int L = p.L;
        p.ss = lv.ss; p.out = lvl(0); p.head = 0;
        p.x = x; p.y = y; p.head_w = st->out_w; p.head_b = st->out_b; p.trace = nullptr;
        __nv_bfloat16 *xb = reinterpret_cast<__nv_bfloat16 *>(base + pl.off[2 * n + 2]);
        if (make_map(st, &P.tmA, xb, 8, L, B, (uint64_t)8 * 2, (uint64_t)L * 8 * 2, 64, (uint32_t)p.R1, 1u)) return -1;
        P.tmO = P.tmA;
        p.hd = 0; p.ps_n = 0; p.ps_rows = p.ps_rows2 = 0; p.ps_bytes = 0; p.ps_tx = p.ps_tx2 = 0;
        if (make_map(st, &P.tmW, lv.wp, (uint64_t)lv.Ktot, lv.Npad, lv.k, (uint64_t)lv.Ktot * 2, (uint64_t)lv.Npad * lv.Ktot * 2, 64, (uint32_t)p.Nh,
                     (uint32_t)p.tg))
            return -1;
        pl.enc0_tc = true;
    }
    for (int i = 1; i < 2 * n + 1; ++i) {
        // row-pair mode (WUNET_TC_PAIR): block 1 and / or the last block run as virtual blocks over pairs of positions
        const int ps = (n >= 2 && i == 1) ? 0 : -1;
        const int Lreal = (i <= n) ? (T >> i) : (T >> (2 * n - i));
        const bool pair = ps >= 0 && !sp && st->pair_ok[ps] && Lreal % 2 == 0 && Lreal / 2 >= 128 &&
                          !pl.enc0_tc;      // the even-row copy comes from the CUDA-core enc0
        const TcLevel &lv = pair ? st->pair_lv[ps] : st->levels[i];
        TcPlanLevel &P = pl.lv[i];
        if (!pair && !sp && st->gemm && parse_override(st->plan_ovr, i).any == false && plan_block_gemm(lv, i, n, B, T, st->num_sms, P)) {
            GemmParams &g = P.gp;
            TcLevel &lw = st->levels[i];
            const bool dec = i > n;
            const int ktot = (g.npos[0] * g.cpp[0] + g.npos[1] * g.cpp[1]) * 64;
            const size_t need = (size_t)g.N * ktot;
            if (lw.wx_L != g.L) {                              // (re)build the Toeplitz expansion for this frame length
                if (lw.wx_elems < need) {
                    cudaFree(lw.wx); lw.wx = nullptr; lw.wx_elems = 0;
                    if (cudaMalloc(&lw.wx, need * sizeof(__nv_bfloat16)) != cudaSuccess) return tc_fail("cudaMalloc(expanded weights) failed");
                    lw.wx_elems = need;
                }
                const float up = (dec && g.L > 1) ? (float)(g.L / 2 - 1) / (float)(g.L - 1) : 0.f;
                expand_gemm_weights_kernel<<<(unsigned)((need + 255) / 256), 256, 0, stream>>>(lw.w_f32, lw.wx, lv.cout, lv.cin0, lv.cin1, lv.k, g.L,
                                                                                               dec ? 1 : 0, g.npos[0], g.cpp[0], g.npos[1], g.cpp[1], up);
                if (cudaGetLastError() != cudaSuccess) return tc_fail("expand_gemm_weights_kernel launch failed");
                lw.wx_L = g.L;
            }
            g.ss = lv.ss; g.out = lvl(i);
            if (!dec) {
                const int Cp = lv.cin0, Lp = 2 * g.L;           // decimated view of the previous block's output
                if (make_map(st, &P.tmA, lvl(i - 1), Cp, g.L, B, (uint64_t)2 * Cp * 2, (uint64_t)Lp * Cp * 2, 64, 1, 128)) return -1;
                P.tmO = P.tmA;
            } else {
                const int e = 2 * n - i, Cs = lv.cin1, Cq = lv.cin0;
                if (make_map(st, &P.tmA, lvl(i - 1), Cq, g.L / 2, B, (uint64_t)Cq * 2, (uint64_t)(g.L / 2) * Cq * 2, 64, 1, 128)) return -1;
                if (make_map(st, &P.tmO, lvl(e), Cs, g.L, B, (uint64_t)Cs * 2, (uint64_t)g.L * Cs * 2, 64, 1, 128)) return -1;
            }
            if (make_map(st, &P.tmW, lw.wx, (uint64_t)ktot, (uint64_t)g.N, 1, (uint64_t)ktot * 2, (uint64_t)g.N * ktot * 2, 64, (uint32_t)g.Nh, 1))
                return -1;
            continue;
        }
        if (plan_block(lv, i, n, B, T, st->num_sms, st->plan_ovr, P, sp, 0, pair)) return -1;
        TcParams &p = P.p;
        const bool dec = i > n;
        const int L = p.L;
        p.ss = lv.ss;
        const bool last = (i == 2 * n);
        p.out = (last && !st->store_last) ? nullptr : lvl(i);
        p.head = last ? 1 : 0;
        p.x = x; p.y = y; p.head_w = st->out_w; p.head_b = st->out_b;
        p.trace = (st->trace && st->trace_level == i) ? st->trace : nullptr;
        // operand maps
        if (!dec && pair) {
            // row-pair mode: the dense copy of the previous block's even rows [B][2L][Cp/2] seen as [B][L][Cp] (two positions per row)
            const int Cp = lv.cin0;
            __nv_bfloat16 *even = reinterpret_cast<__nv_bfloat16 *>(base + pl.off[2 * n + 1]);
            if (make_map(st, &P.tmA, even, Cp, L, B, (uint64_t)Cp * 2, (uint64_t)L * Cp * 2, 64, (uint32_t)p.R1, 1u)) return -1;
            pl.even_copy = true;
        } else if (!dec) {
            // decimated view of the previous encoder output: element (c, l, b) -> prev[b][2l][c]   (o[:, :, ::2])
            const int Cp = lv.cin0, Lp = 2 * L;
            const uint32_t b1 = p.packed ? (uint32_t)p.S : (uint32_t)p.R1, b2 = p.packed ? (uint32_t)p.FR : 1u;
            if (make_map(st, &P.tmA, lvl(i - 1), cm * Cp, L, B, (uint64_t)2 * cm * Cp * 2, (uint64_t)Lp * cm * Cp * 2, 64, b1, b2, st->enc_l2promo)) return -1;
        } else {
            const int e = 2 * n - i;                        // skip = encoder e's full-resolution output
            const int Cs = lv.cin1;
            const uint32_t b1 = p.packed ? (uint32_t)p.S : (uint32_t)p.R1, b2 = p.packed ? (uint32_t)p.FR : 1u;
            if (make_map(st, &P.tmA, lvl(e), cm * Cs, L, B, (uint64_t)cm * Cs * 2, (uint64_t)L * cm * Cs * 2, 64, b1, b2)) return -1;
            p.prev = lvl(i - 1);
            p.Lin = pair ? L : L / 2;                         // row-pair mode: an operand row IS a previous-level row index
            p.up_scale = pair ? (float)(p.Lin - 1) / (float)(2 * L - 1) : ((L > 1) ? (float)(p.Lin - 1) / (float)(L - 1) : 0.f);
        }
        P.tmO = P.tmA;
        p.hd = 0; p.ps_n = 0; p.ps_rows = p.ps_rows2 = 0; p.ps_bytes = 0; p.ps_tx = p.ps_tx2 = 0;
        const uint64_t ktot = sp ? (uint64_t)lv.sp_chunks * 64 : (uint64_t)lv.Ktot;
        if (make_map(st, &P.tmW, sp ? lv.wp_sp : lv.wp, ktot, lv.Npad, lv.k, ktot * 2, (uint64_t)lv.Npad * ktot * 2, 64,
                     (uint32_t)p.Nh, (uint32_t)p.tg))
            return -1;
    }
    if (getenv("WUNET_TC_DEBUG")) {
        for (int i = pl.enc0_tc ? 0 : 1; i < 2 * n + 1; ++i) {
            const TcParams &p = pl.lv[i].p;
            if (pl.lv[i].is_gemm) {
                const GemmParams &g = pl.lv[i].gp;
                fprintf(stderr, "[wunet gemm] blk %2d L=%2d N=%5d Nh=%3d K chunks=%d+%d stages=%d x %d chunks grid=%ux%u smem=%zu\n", i, g.L, g.N, g.Nh,
                        g.npos[0] * g.cpp[0], g.npos[1] * g.cpp[1], g.nstages, g.cps, pl.lv[i].grid.x, pl.lv[i].grid.y, pl.lv[i].smem);
                continue;
            }
            fprintf(stderr, "[wunet tc] blk %2d L=%5d Cin=%3d+%3d Cout=%3d Nh=%3d x%d MT=%d nacc=%d packed=%d FR=%d res=%d bulk=%d na=%d nb=%d tg=%d smem=%zu tmem=%u tiles=%d grid=%u small=%d per_sm=%d hd=%d ring=%d\n",
                    i, p.L, p.Cin0, p.Cin1, p.Cout, p.Nh, p.nsplit, p.MT, p.nacc, p.packed, p.FR, p.resident, p.bulk_store, p.na, p.nb, p.tg, pl.lv[i].smem, p.tmem_cols,
                    p.m_tiles * p.nsplit, pl.lv[i].grid.x, (int)pl.lv[i].small, pl.lv[i].per_sm, p.hd, p.ps_n);
        }
    }
    st->plan_ws = ws; st->plan_B = B; st->plan_T = T; st->plan_x = x; st->plan_y = y; st->plan_mode = mode;
    return 0;
}

int tc_debug_plan(int n, int ci, const TcBlockSrc *blocks, int nblocks, int B, int T, int block, int num_sms, int *f, int cap, int mode)
{
    const char *e0 = getenv("WUNET_TC_ENC0");
    const bool g8 = !mode && block == 0 && e0 && e0[0] == '1';    // block 0 has a tensor-core plan only in its group-of-8 form (bf16)
    if (nblocks != 2 * n + 1 || (block < 1 && !g8) || block >= nblocks) return tc_fail("block %d out of range (1..%d)", block, 2 * n);
    if (ci % 8 != 0 || ci > 32) return tc_fail("bf16 tensor-core path needs channels_interval %% 8 == 0 and <= 32 (got %d)", ci);
    if (cap < 32 || !f) return tc_fail("need room for 32 fields");
    if (g8) {
        if (blocks[0].k != 15 || blocks[0].cin != 1 || 8 * blocks[0].cout > 256 || T % 8 != 0 || T / 8 < 128) return tc_fail("block 0 has no group-of-8 plan for this shape");
        TcLevel pv;
        pv.cin0 = 8; pv.cin1 = 0; pv.cout = 8 * blocks[0].cout; pv.k = 3; pv.Npad = round_up(pv.cout, 16); pv.Ktot = 64;
        TcPlanLevel P{};
        const char *ovr = getenv("WUNET_TC_OVR");
        if (plan_block(pv, 0, n, B, T, num_sms, ovr ? ovr : "", P, false, 0, false, true)) return -1;
        const TcParams &p = P.p;
        const int v[32] = {p.L, p.Cin0, p.Cin1, p.Cout, p.Npad, p.Nh, p.nsplit, p.Nstride, p.MT, p.nacc, p.packed, p.FR, p.S, p.m_tiles,
                           p.nchunks, p.resident, p.bulk_store, p.na, p.nb, p.tg, p.ngroups, (int)p.a_stage_bytes, (int)p.b_stage_bytes,
                           p.a_tx_bytes, p.rows_used, (int)p.tmem_cols, (int)P.smem, P.threads, P.per_sm, (int)P.grid.x, (int)P.small,
                           p.tiles_per_frame};
        for (int k = 0; k < 32; ++k) f[k] = v[k];
        return 0;
    }
    std::vector<TcLevel> levels(nblocks);
    const char *mge = getenv("WUNET_TC_MERGE");
    derive_levels(levels, blocks, nblocks, n, !(mge && mge[0] == '0'));
    const char *ovr = getenv("WUNET_TC_OVR");
    TcPlanLevel P{};
    const std::string ovr_s = ovr ? ovr : "";
    const char *ge = getenv("WUNET_TC_GEMM");
    bool planned = false;
    if (mode) {
        // split precision (fp32_tc): every block on conv_tc_kernel in split form, no row-pair form, no dense GEMM (build_plan)
        if (plan_block(levels[block], block, n, B, T, num_sms, ovr_s, P, true, 0)) return -1;
        planned = true;
    } else {
        // row-pair mode of block 1 (WUNET_TC_PAIR bit 0), planned like build_plan does
        const char *pe = getenv("WUNET_TC_PAIR");
        const int pmask = pe ? atoi(pe) & 1 : 1;
        const int ps = (n >= 2 && block == 1) ? 0 : -1;
        const int Lreal = (block <= n) ? (T >> block) : (T >> (2 * n - block));
        if (ps >= 0 && (pmask & (1 << ps)) && Lreal % 2 == 0 && Lreal / 2 >= 128) {
            const TcLevel &rl = levels[block];
            const bool ok = rl.k == 15 && rl.cin1 == 0 && rl.cin0 % 8 == 0 && 2 * rl.cin0 <= 64 && 2 * rl.cout <= 256;
            if (ok) {
                TcLevel pv = rl;
                pv.cin0 = 2 * rl.cin0; pv.cin1 = 2 * rl.cin1; pv.cout = 2 * rl.cout; pv.k = pair_taps(rl.k);
                pv.Npad = round_up(pv.cout, 16);
                pv.Ktot = round_up(pv.cin0, 64) + (pv.cin1 ? round_up(pv.cin1, 64) : 0);
                pv.mg_s = pv.mg_u = 0;
                if (plan_block(pv, block, n, B, T, num_sms, ovr_s, P, false, 0, true)) return -1;
                planned = true;
            }
        }
    }
    if (!planned && !(!(ge && ge[0] == '0') && parse_override(ovr_s, block).any == false &&
                      plan_block_gemm(levels[block], block, n, B, T, num_sms, P)) &&
        plan_block(levels[block], block, n, B, T, num_sms, ovr_s, P, false, 0))
        return -1;
    const TcParams &p = P.p;
    const int v[32] = {p.L, p.Cin0, p.Cin1, p.Cout, p.Npad, p.Nh, p.nsplit, p.Nstride, p.MT, p.nacc, p.packed, p.FR, p.S, p.m_tiles,
                       p.nchunks, p.resident, p.bulk_store, p.na, p.nb, p.tg, p.ngroups, (int)p.a_stage_bytes, (int)p.b_stage_bytes,
                       p.a_tx_bytes, p.rows_used, (int)p.tmem_cols, (int)P.smem, P.threads, P.per_sm, (int)P.grid.x, P.kind == 2 ? 2 : (int)P.small,
                       p.tiles_per_frame};
    for (int k = 0; k < 32; ++k) f[k] = v[k];
    return 0;
}

static int tc_prepare(TcState *st, const float *x, float *y, int B, int T, void *ws, int mode, cudaStream_t stream)
{
    if (!st) return tc_fail("tensor-core state missing");
    const int ci = st->ci;
    if (ci % 8 != 0 || ci > 32) return tc_fail("bf16 tensor-core path needs channels_interval %% 8 == 0 and <= 32 (got %d)", ci);
    if (!st->attr_set) {
        cudaFuncSetAttribute(conv_tc_kernel<15, false, kEpiWarpsLarge, 0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
        cudaFuncSetAttribute(conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
        cudaFuncSetAttribute(conv_tc_kernel<15, false, kEpiWarpsSmall, 0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
        cudaFuncSetAttribute(conv_tc_kernel<5, true, kEpiWarpsSmall, kProducerWarpsSmall, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
        cudaFuncSetAttribute(conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
        cudaFuncSetAttribute(conv_tc_kernel<5, true, kEpiWarpsSmall, kProducerWarpsSmall, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
        cudaFuncSetAttribute(conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 0, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
        cudaFuncSetAttribute(conv_tc_kernel<15, false, kEpiWarpsLarge, 0, 0, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
        cudaFuncSetAttribute(conv_tc_kernel<3, false, kEpiWarpsLarge, 0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
        cudaFuncSetAttribute(conv_tc_kernel<3, false, kEpiWarpsSmall, 0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
        cudaFuncSetAttribute(conv_tc_kernel<9, false, kEpiWarpsLarge, 0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
        cudaFuncSetAttribute(conv_tc_kernel<9, false, kEpiWarpsSmall, 0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
        cudaFuncSetAttribute(gemm_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
        cudaFuncSetAttribute(enc0_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
        cudaFuncSetAttribute(enc0_kernel_v2, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
        int dev = 0, sms = 0;
        if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && sms > 0)
            st->dev_sms = sms;
        st->attr_set = true;
    }
    (void)x; (void)y;
    // WUNET_TC_SMS=<n> (test hook): plan and size the persistent grids as on a device with n SMs. A grid smaller than the device
    // is always legal, so one GPU can run the plan of any other SM count (n = 1: one CTA, two in the small flavour, per block).
    int sms = st->dev_sms;
    if (const char *se = getenv("WUNET_TC_SMS")) {
        sms = atoi(se);
        if (sms < 1) return tc_fail("WUNET_TC_SMS must be a positive SM count (got \"%s\")", se);
    }
    st->num_sms = sms;
    const char *ovr = getenv("WUNET_TC_OVR");
    const std::string ovr_s = ovr ? ovr : "";
    if (st->plan_ws != ws || st->plan_B != B || st->plan_T != T || st->plan_ovr != ovr_s || st->plan_sms != sms || st->plan_mode != mode) {
        st->plan_ovr = ovr_s;
        st->plan_sms = sms;
        st->plan_ws = nullptr;
        if (build_plan(st, nullptr, nullptr, B, T, ws, mode, stream)) return -1;
    }
    return 0;
}

static int launch_block(TcState *st, int i, int t0, int t1, cudaStream_t stream, const float *x = nullptr, float *y = nullptr);

// enc0 over frames [f0, f0 + nf); *launches receives the number of kernels enqueued
static int launch_enc0(TcState *st, const float *x, int f0, int nf, int T, void *ws, cudaStream_t stream, int *launches = nullptr)
{
    if (launches) *launches = 1;
    if (st->plan.enc0_tc) {
        // tensor-core form: bf16 copy of the frames' samples, then block 0 as a 3-tap block over groups of 8 samples
        __nv_bfloat16 *xb = reinterpret_cast<__nv_bfloat16 *>(static_cast<char *>(ws) + st->plan.off[2 * st->n + 2]) + (size_t)f0 * T;
        const long long n4 = (long long)nf * T / 4;
        x_to_bf16_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(x + (size_t)f0 * T, xb, n4);
        if (cudaGetLastError() != cudaSuccess) return tc_fail("x_to_bf16_kernel launch failed");
        const int tpf = st->plan.lv[0].p.tiles_per_frame * st->plan.lv[0].p.nsplit;    // tiles of one frame, all column splits
        if (launches) *launches = 2;
        return launch_block(st, 0, f0 * tpf, (f0 + nf) * tpf, stream, nullptr, nullptr);
    }
    const TcLevel &lv = st->levels[0];
    const int C = lv.cout;
    const int split = st->plan_mode != 0 ? 1 : 0;
    const int RC = split ? 2 * C : C;
    const size_t smem = (size_t)(15 * C + 2 * C + 4 + 1024 + 16) * sizeof(float) + (size_t)1024 * RC * 2 + 16;
    dim3 grid((unsigned)((T + 1023) / 1024), (unsigned)nf, 1);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = st->pdl ? 1 : 0;
    cfg.attrs = attr; cfg.numAttrs = 1;
    __nv_bfloat16 *out0 = reinterpret_cast<__nv_bfloat16 *>(static_cast<char *>(ws) + st->plan.off[0]);
    __nv_bfloat16 *even = (st->plan.even_copy && !split)
                              ? reinterpret_cast<__nv_bfloat16 *>(static_cast<char *>(ws) + st->plan.off[2 * st->n + 1]) + (size_t)f0 * (T / 2) * C
                              : nullptr;
    if (st->enc0_v == 2 || (st->enc0_v == 0 && split)) {
        const int total = nf * ((T + 1023) / 1024);
        cfg.gridDim = dim3((unsigned)std::min(total, st->num_sms * 4), 1, 1);
        cudaLaunchKernelEx(&cfg, enc0_kernel_v2, x + (size_t)f0 * T, lv.w_src, lv.scale, lv.shift, out0 + (size_t)f0 * T * RC, nf, T, C, split, even);
    } else
    cudaLaunchKernelEx(&cfg, enc0_kernel, x + (size_t)f0 * T, lv.w_src, lv.scale, lv.shift, out0 + (size_t)f0 * T * RC, nf, T, C, split, even);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return tc_fail("enc0 launch failed: %s", cudaGetErrorString(e));
    return 0;
}

// conv block i over the tile range [t0, t1) (t1 < 0: all tiles)
static int launch_block(TcState *st, int i, int t0, int t1, cudaStream_t stream, const float *x, float *y)
{
    TcPlanLevel &P = st->plan.lv[i];
    if (P.is_gemm) {
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = P.grid; cfg.blockDim = dim3(P.threads); cfg.dynamicSmemBytes = P.smem; cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = st->pdl ? 1 : 0;
        cfg.attrs = attr; cfg.numAttrs = 1;
        cudaLaunchKernelEx(&cfg, gemm_tc_kernel, P.tmA, P.tmO, P.tmW, P.gp);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return tc_fail("gemm_tc level %d launch failed: %s", i, cudaGetErrorString(e));
        return 0;
    }
    TcParams p = P.p;
    p.x = x; p.y = y;                                    // only the fused head (last block) reads x / writes y
    p.pf_late = st->pf_late ? 1 : 0;
    if (t1 >= 0) { p.tile_begin = t0; p.tile_end = t1; }
    const int ntiles = p.tile_end - p.tile_begin;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)std::min(ntiles, st->num_sms * P.per_sm), 1, 1);
    cfg.blockDim = dim3(P.threads); cfg.dynamicSmemBytes = P.smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = st->pdl ? 1 : 0;
    cfg.attrs = attr; cfg.numAttrs = 1;
    if (P.pair == 3) {
        // block 0 over groups of 8 samples: a 3-tap encoder block
        if (!P.small) cudaLaunchKernelEx(&cfg, conv_tc_kernel<3, false, kEpiWarpsLarge, 0, 0>, P.tmA, P.tmW, P.tmO, p);
        else cudaLaunchKernelEx(&cfg, conv_tc_kernel<3, false, kEpiWarpsSmall, 0, 0>, P.tmA, P.tmW, P.tmO, p);
    } else if (P.pair == 1) {
        // row-pair mode of the first tensor-core encoder block: a 9-tap block over pairs of positions
        if (!P.small) cudaLaunchKernelEx(&cfg, conv_tc_kernel<9, false, kEpiWarpsLarge, 0, 0>, P.tmA, P.tmW, P.tmO, p);
        else cudaLaunchKernelEx(&cfg, conv_tc_kernel<9, false, kEpiWarpsSmall, 0, 0>, P.tmA, P.tmW, P.tmO, p);
    } else if (p.split) {
        if (P.upcat) cudaLaunchKernelEx(&cfg, conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 0, 1>, P.tmA, P.tmW, P.tmO, p);
        else cudaLaunchKernelEx(&cfg, conv_tc_kernel<15, false, kEpiWarpsLarge, 0, 0, 1>, P.tmA, P.tmW, P.tmO, p);
    } else if (P.upcat && p.mg) {
        if (!P.small) cudaLaunchKernelEx(&cfg, conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 1>, P.tmA, P.tmW, P.tmO, p);
        else cudaLaunchKernelEx(&cfg, conv_tc_kernel<5, true, kEpiWarpsSmall, kProducerWarpsSmall, 1>, P.tmA, P.tmW, P.tmO, p);
    } else if (P.upcat && !P.small) cudaLaunchKernelEx(&cfg, conv_tc_kernel<5, true, kEpiWarpsLarge, kProducerWarpsLarge, 0>, P.tmA, P.tmW, P.tmO, p);
    else if (P.upcat) cudaLaunchKernelEx(&cfg, conv_tc_kernel<5, true, kEpiWarpsSmall, kProducerWarpsSmall, 0>, P.tmA, P.tmW, P.tmO, p);
    else if (!P.small) cudaLaunchKernelEx(&cfg, conv_tc_kernel<15, false, kEpiWarpsLarge, 0, 0>, P.tmA, P.tmW, P.tmO, p);
    else cudaLaunchKernelEx(&cfg, conv_tc_kernel<15, false, kEpiWarpsSmall, 0, 0>, P.tmA, P.tmW, P.tmO, p);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return tc_fail("conv_tc level %d launch failed: %s", i, cudaGetErrorString(e));
    return 0;
}

int tc_forward(TcState *st, const float *x, float *y, int B, int T, void *ws, cudaStream_t stream, int *launches,
               cudaEvent_t *ev, int mode)
{
    if (tc_prepare(st, x, y, B, T, ws, mode, stream)) return -1;
    const int n = st->n;
    int nl = 0;
    if (ev) cudaEventRecord(ev[0], stream);
    int l0n = 1;
    if (launch_enc0(st, x, 0, B, T, ws, stream, &l0n)) return -1;
    nl += l0n;
    if (ev) cudaEventRecord(ev[1], stream);
    for (int i = 1; i < 2 * n + 1; ++i) {
        if (launch_block(st, i, 0, -1, stream, x, y)) return -1;
        ++nl;
        if (ev) cudaEventRecord(ev[i + 1], stream);
    }
    if (ev) cudaEventRecord(ev[2 * n + 2], stream);     // head is fused: zero-length segment
    if (launches) *launches = nl;
    return 0;
}

// Host-buffer pipeline (enhancement.py:64-66 form): the first kernel (enc0) and the last (decoder + fused head) run per
// batch chunk, so the H2D copy of chunk c+1 overlaps enc0 of chunk c and the D2H copy of chunk c overlaps the head of c+1.
int tc_forward_host(TcState *st, const float *x_host, float *y_host, float *x_dev, float *y_dev, int B, int T, void *ws,
                    cudaStream_t stream, int *launches, int mode)
{
    if (tc_prepare(st, x_dev, y_dev, B, T, ws, mode, stream)) return -1;
    const int n = st->n;
    const TcParams &pl = st->plan.lv[2 * n].p;
    int nc = 1;
    if (!pl.packed && pl.nsplit == 1) { if (B % 4 == 0 && B >= 32) nc = 4; else if (B % 2 == 0 && B >= 8) nc = 2; }
    if (!st->copy_in) {
        if (cudaStreamCreateWithFlags(&st->copy_in, cudaStreamNonBlocking) != cudaSuccess ||
            cudaStreamCreateWithFlags(&st->copy_out, cudaStreamNonBlocking) != cudaSuccess)
            return tc_fail("cudaStreamCreate failed");
        for (int i = 0; i < 8; ++i) {
            cudaEventCreateWithFlags(&st->ev_in[i], cudaEventDisableTiming);
            cudaEventCreateWithFlags(&st->ev_out[i], cudaEventDisableTiming);
        }
    }
    const int bc = B / nc;
    const size_t chunk = (size_t)bc * T;
    int nl = 0;
    // the compute stream may still own x_dev/y_dev from an earlier call: order the copies after it
    cudaEventRecord(st->ev_out[7], stream);
    cudaStreamWaitEvent(st->copy_in, st->ev_out[7], 0);
    for (int c = 0; c < nc; ++c) {
        cudaMemcpyAsync(x_dev + c * chunk, x_host + c * chunk, chunk * sizeof(float), cudaMemcpyHostToDevice, st->copy_in);
        cudaEventRecord(st->ev_in[c], st->copy_in);
        cudaStreamWaitEvent(stream, st->ev_in[c], 0);
        int l0n = 1;
        if (launch_enc0(st, x_dev, c * bc, bc, T, ws, stream, &l0n)) return -1;
        nl += l0n;
    }
    for (int i = 1; i < 2 * n; ++i) {
        if (launch_block(st, i, 0, -1, stream)) return -1;
        ++nl;
    }
    const int tiles_per_chunk = (pl.m_tiles * pl.nsplit) / nc;      // non-packed: m_tiles = B * tiles_per_frame
    for (int c = 0; c < nc; ++c) {
        if (nc == 1) { if (launch_block(st, 2 * n, 0, -1, stream, x_dev, y_dev)) return -1; }
        else if (launch_block(st, 2 * n, c * tiles_per_chunk, (c + 1) * tiles_per_chunk, stream, x_dev, y_dev)) return -1;
        ++nl;
        cudaEventRecord(st->ev_out[c], stream);
        cudaStreamWaitEvent(st->copy_out, st->ev_out[c], 0);
        cudaMemcpyAsync(y_host + c * chunk, y_dev + c * chunk, chunk * sizeof(float), cudaMemcpyDeviceToHost, st->copy_out);
    }
    if (cudaStreamSynchronize(st->copy_out) != cudaSuccess) return tc_fail("host pipeline failed: %s", cudaGetErrorString(cudaGetLastError()));
    if (launches) *launches = nl;
    return 0;
}

int tc_read_level(TcState *st, int block, const void *ws, int B, int T, float *out_ncl, cudaStream_t stream, int mode)
{
    if (!st) return tc_fail("tensor-core state missing");
    const int n = st->n;
    if (block == 2 * n && !st->store_last)
        return tc_fail("the last decoder block is fused with the head and not materialised (set WUNET_TC_STORE_LAST=1)");
    std::vector<size_t> off;
    size_t total;
    tc_layout(n, st->ci, B, T, off, total, mode);
    const int L = (block <= n) ? (T >> block) : (T >> (2 * n - block));
    const int C = st->levels[block].cout;
    const long long nel = (long long)B * C * L;
    const __nv_bfloat16 *src = reinterpret_cast<const __nv_bfloat16 *>(static_cast<const char *>(ws) + off[block]);
    if (mode) nlc_split_to_ncl_f32_kernel<<<(unsigned)((nel + 255) / 256), 256, 0, stream>>>(src, out_ncl, B, L, C);
    else nlc_bf16_to_ncl_f32_kernel<<<(unsigned)((nel + 255) / 256), 256, 0, stream>>>(src, out_ncl, B, L, C);
    return cudaGetLastError() == cudaSuccess ? 0 : tc_fail("read_level launch failed");
}

// host-only: the row-pair expansion of one block's weights (pair_weight), as expand_pair_weights_kernel writes it
int tc_debug_pair_weights(const float *w, int Cout, int C0, int C1, int K, int dec, float *out)
{
    if (!w || !out || Cout < 1 || C0 < 1 || C1 < 0 || K < 1 || (K & 1) == 0) return tc_fail("bad row-pair weight query");
    if (dec == 2) {                                       // block 0 over groups of 8 samples: out[8 Cout][8][3]
        if (C0 != 1 || C1 != 0 || K > 15) return tc_fail("the group-of-8 form is for Conv1d(1 -> C, k <= 15)");
        for (int cov = 0; cov < 8 * Cout; ++cov)
            for (int q = 0; q < 8; ++q)
                for (int tv = 0; tv < 3; ++tv) out[((size_t)cov * 8 + q) * 3 + tv] = group8_weight(w, Cout, K, cov, q, tv);
        return 0;
    }
    const int Kp = pair_taps(K), Cv = 2 * (C0 + C1);
    for (int cov = 0; cov < 2 * Cout; ++cov)
        for (int v = 0; v < Cv; ++v)
            for (int tv = 0; tv < Kp; ++tv) out[((size_t)cov * Cv + v) * Kp + tv] = pair_weight(w, Cout, C0, C1, K, dec, cov, v, tv);
    return 0;
}

void tc_destroy(TcState *st)
{
    if (!st) return;
    if (st->copy_in) {
        cudaStreamDestroy(st->copy_in); cudaStreamDestroy(st->copy_out);
        for (int i = 0; i < 8; ++i) { cudaEventDestroy(st->ev_in[i]); cudaEventDestroy(st->ev_out[i]); }
    }
    if (st->trace) {
        std::vector<long long> h(5 * 512);
        cudaDeviceSynchronize();
        cudaMemcpy(h.data(), st->trace, h.size() * sizeof(long long), cudaMemcpyDeviceToHost);
        long long t0 = h[512];
        for (int r = 0; r < 5; ++r) {
            fprintf(stderr, "[trace role %d]", r);
            for (int i = 0; i < 200 && h[r * 512 + i]; ++i) fprintf(stderr, " %lld", h[r * 512 + i] - t0);
            fprintf(stderr, "\n");
        }
        cudaFree(st->trace);
    }
    for (auto &lv : st->levels) { cudaFree(lv.wp); cudaFree(lv.ss); cudaFree(lv.w_own); cudaFree(lv.wp_sp); cudaFree(lv.w_f32); cudaFree(lv.wx); }
    cudaFree(st->g8_lv.wp); cudaFree(st->g8_lv.ss); cudaFree(st->g8_w); cudaFree(st->g8_scale); cudaFree(st->g8_shift);
    for (int s = 0; s < 2; ++s) { cudaFree(st->pair_lv[s].wp); cudaFree(st->pair_lv[s].ss); cudaFree(st->pair_w[s]); cudaFree(st->pair_scale[s]); cudaFree(st->pair_shift[s]); }
    delete st;
}

}  // namespace wunet
