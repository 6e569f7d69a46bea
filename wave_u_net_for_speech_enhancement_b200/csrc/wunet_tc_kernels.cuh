// wunet_tc_kernels.cuh — device code of the tensor-core inference path, written once for both of its 16-bit element types.
//
// Included once per element type, inside that type's namespace, after `TcElem` names its traits (wunet_tc_common.cuh):
//   wunet_tc.cu      namespace wunet        TcElem = TcBf16  (bf16, and the split-precision fp32_tc kernels)
//   wunet_tc_f16.cu  namespace wunet::f16   TcElem = TcF16   (fp16; defines WUNET_TC_FP16)
// The kernels keep their names in both; the namespace tells them apart. Everything the host code shares between the two
// (kernel parameters, shared-memory map, constants) is in wunet_tc_common.cuh. No #include here: the includer has them.

using TcT = TcElem::T;            // activation / weight element
using TcT2 = TcElem::T2;          // two of them (packed HFMA2 arithmetic)
// Element type of the network input read by block 0 and the fused head, and of the output the head writes (IoType): float,
// unless the includer defines WUNET_TC_IO as a 16-bit type (wunet_tc_io.cuh). A sample is widened to fp32 on load and a
// result rounded once on store, so the float forms are the code they were before the I/O type existed.
#ifndef WUNET_TC_IO
#define WUNET_TC_IO float
#endif
using TcIO = WUNET_TC_IO;

namespace {

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
            wgmma_m64nNk16<16 * NT, 0, 0, TcT>(*reinterpret_cast<float (*)[8 * NT]>(&acc[mb][0]), a_lo + (uint32_t)(mb * 512 + 2 * k),
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

// K-loop position c -> (segment, chunk index inside the segment, K16 steps, 64-wide slot in the packed weights)
// SP = 2 (split precision, wide channel plans, wunet_tc_wide.cu): chunk_map lists the 64-channel chunks, not the positions;
// chunk q is positions 3q (hi data x w_hi), 3q + 1 (the same stage x w_lo) and 3q + 2 (lo data x w_hi), the order and flags
// the SP = 1 map spells out per position. A block may then have up to 3 x 48 positions.
struct ChunkInfo { bool up; int idx, nk, kslot; bool merged; int vo, nvec; bool lo, reuse; };
template <bool UPCAT, int MG, int SP = 0>
__device__ __forceinline__ ChunkInfo chunk_info(const TcParams &p, int c)
{
    ChunkInfo ci;
    const int m = SP == 2 ? p.chunk_map[c / 3] | ((c % 3) == 1 ? 0x20 : 0) | ((c % 3) == 2 ? 0x40 : 0) : p.chunk_map[c];
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
                                    __nv_bfloat16 *orow = static_cast<__nv_bfloat16 *>(p.out) + ((size_t)bb * p.L + l) * (2 * p.Cout) + n0 + col;
                                    *reinterpret_cast<uint32_t *>(orow) = pack_bf16(f0, f1);
                                    *reinterpret_cast<uint32_t *>(orow + p.Cout) =
                                        pack_bf16(f0 - __bfloat162float(__float2bfloat16_rn(f0)), f1 - __bfloat162float(__float2bfloat16_rn(f1)));
                                } else {
                                    *reinterpret_cast<uint32_t *>(static_cast<TcT *>(p.out) + ((size_t)bb * p.L + l) * p.Cout + n0 + col) = TcElem::pack(f0, f1);
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
                            const float hacc = fmaf(hw[p.Cout], io_ld(reinterpret_cast<const TcIO *>(p.x) + (size_t)bb * p.T + l),
                                                    hw[p.Cout + 1] + hsum);
                            io_st(reinterpret_cast<TcIO *>(p.y) + (size_t)bb * p.T + l, tanh_fast(hacc));
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
                const TcT *pb = static_cast<const TcT *>(p.prev) + (size_t)ub0 * p.Lin * creal + ch;
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
            const TcT *pb = static_cast<const TcT *>(p.prev) + (size_t)ub0 * p.Lin * p.Cin0 + ch;
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
                        // lam1 = up_scale * l - (m - 1 + qh): the generic instantiation's formula (one fused rounding), packed 16-bit
                        const float lam1 = fmaf(p.up_scale, (float)(2 * m + qh), -(float)(m - 1 + qh));
                        const TcT2 lam = TcElem::to2(lam1);
                        const TcT2 *a2 = reinterpret_cast<const TcT2 *>(&w[j + qh]);
                        const TcT2 *b2 = reinterpret_cast<const TcT2 *>(&w[j + qh + 1]);
                        TcT2 r2[4];
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
                // out = a + lam1 * (b - a) in packed 16-bit arithmetic (HFMA2); lam1 = up_scale * l - (ms - 1 + qa), one fused rounding
                const float lam1 = fmaf(p.up_scale, lf0 + (float)j, -(mf0 + (float)qa));
                const TcT2 lam = TcElem::to2(lam1);
                const TcT2 *a2 = reinterpret_cast<const TcT2 *>(&w[qa]);
                const TcT2 *b2 = reinterpret_cast<const TcT2 *>(&w[qa + 1]);
                TcT2 r2[4];
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
                            const bool pair = SP == 2 ? !cu.lo && c + 2 < p.nchunks
                                                      : !cu.lo && c + 2 < p.nchunks && p.chunk_map[c + 2] == (p.chunk_map[c] | 0x40) &&
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
                                    const __nv_bfloat16 *pb = static_cast<const __nv_bfloat16 *>(p.prev) + (size_t)b0 * p.Lin * (2 * p.Cin0) + ch;
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
                                        const __nv_bfloat16 *r0 = static_cast<const __nv_bfloat16 *>(p.prev) + ((size_t)bb * p.Lin + i0) * (2 * p.Cin0) + ch;
                                        const __nv_bfloat16 *r1 = static_cast<const __nv_bfloat16 *>(p.prev) + ((size_t)bb * p.Lin + i1) * (2 * p.Cin0) + ch;
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
                                const uint4 u0 = __ldg(reinterpret_cast<const uint4 *>(static_cast<const TcT *>(p.prev) + ((size_t)bb * p.Lin + i0) * p.Cin0 + ch));
                                const uint4 u1 = __ldg(reinterpret_cast<const uint4 *>(static_cast<const TcT *>(p.prev) + ((size_t)bb * p.Lin + i1) * p.Cin0 + ch));
                                const uint32_t a0[4] = {u0.x, u0.y, u0.z, u0.w}, a1[4] = {u1.x, u1.y, u1.z, u1.w};
                                uint32_t r[4];
#pragma unroll
                                for (int q4 = 0; q4 < 4; ++q4) {
                                    const float2 f0 = TcElem::f2(a0[q4]);
                                    const float2 f1 = TcElem::f2(a1[q4]);
                                    r[q4] = TcElem::pack(lam0 * f0.x + lam1 * f1.x, lam0 * f0.y + lam1 * f1.y);
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

// WUNET_TC_CONV_ONLY (wunet_tc_wide.cu): the includer instantiates conv_tc_kernel forms of its own and needs none of the
// non-template kernels below, which the other two units already emit.
// WUNET_TC_IO_ONLY (wunet_tc_io.cuh): the forms with a 16-bit network input / output, i.e. conv_tc_kernel (instantiated by the
// includer for the last block), enc0_kernel and x_to_bf16_kernel; none of the other kernels.
#ifndef WUNET_TC_CONV_ONLY
#ifndef WUNET_TC_IO_ONLY
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
                    const uint32_t o = TcElem::pack(lrelu(fmaf(acc[0][8 * nb + 4 * e + 2 * h], s0.x, s0.y)),
                                                 lrelu(fmaf(acc[0][8 * nb + 4 * e + 2 * h + 1], s1.x, s1.y)));
                    if (b < p.B) *reinterpret_cast<uint32_t *>(static_cast<TcT *>(p.out) + (size_t)b * p.N + n) = o;
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
__global__ void expand_gemm_weights_kernel(const float *__restrict__ w, TcT *__restrict__ wx, int Cout, int Cin0, int Cin1, int K,
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
    wx[i] = TcElem::cvt(v);
}

#endif  // WUNET_TC_IO_ONLY

// -------------------------------------------------------------------------------------------------
// enc0: Conv1d(1 -> C, k=15) + BN + LeakyReLU on CUDA cores (Cin = 1: K = 15, HBM-bound), IO in (widened to fp32), 16-bit NLC out
// -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 4) enc0_kernel(const TcIO *__restrict__ x, const float *__restrict__ w /*[C][1][15]*/,
                                                      const float *__restrict__ scale, const float *__restrict__ shift,
                                                      TcT *__restrict__ out, int B, int T, int C, int split,
                                                      TcT *__restrict__ even_out)
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
        xs[i] = (l >= 0 && l < T) ? io_f32(x[(size_t)b * T + l]) : 0.f;
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
                make_uint4(TcElem::pack(f[0], f[1]), TcElem::pack(f[2], f[3]), TcElem::pack(f[4], f[5]), TcElem::pack(f[6], f[7]));
            if (even_out != nullptr && (j & 1) == 0 && l0 + 4 * (int)threadIdx.x + j < T)
                *reinterpret_cast<uint4 *>(even_out + ((size_t)b * (T >> 1) + ((l0 + 4 * threadIdx.x + j) >> 1)) * C + c0) =
                    make_uint4(TcElem::pack(f[0], f[1]), TcElem::pack(f[2], f[3]), TcElem::pack(f[4], f[5]), TcElem::pack(f[6], f[7]));
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

#ifndef WUNET_TC_IO_ONLY
// enc0, persistent form (round 2, last session): the same arithmetic in the same order (bit-identical output), but a block loops over
// tiles: the weights are loaded once, the samples of the NEXT tile stream into shared memory by cp.async while this tile is
// computed, and the bulk store of a tile's rows drains while the next tile's first channel pass is computed (the one-shot
// kernel above spends ~35 % of its time in the un-overlapped load -> compute -> store -> drain phases of its 4 resident blocks).
// float input only: a 16-bit input runs enc0_kernel (same output), since no cp.async form widens 16-bit samples
__global__ void __launch_bounds__(256, 4) enc0_kernel_v2(const float *__restrict__ x, const float *__restrict__ w /*[C][1][15]*/,
                                                         const float *__restrict__ scale, const float *__restrict__ shift,
                                                         TcT *__restrict__ out, int B, int T, int C, int split,
                                                         TcT *__restrict__ even_out)
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
                const uint4 o = make_uint4(TcElem::pack(f[0], f[1]), TcElem::pack(f[2], f[3]), TcElem::pack(f[4], f[5]), TcElem::pack(f[6], f[7]));
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

#endif  // WUNET_TC_IO_ONLY

#ifndef WUNET_TC_FP16
#ifndef WUNET_TC_IO_ONLY
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
// pair_taps, pair_weight: wunet_tc_common.cuh
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
// group8_weight: wunet_tc_common.cuh
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
#endif  // WUNET_TC_IO_ONLY
__global__ void x_to_bf16_kernel(const TcIO *__restrict__ x, __nv_bfloat16 *__restrict__ xb, long long n4)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const float4 v = io_ld4(x + 4 * i);
    reinterpret_cast<uint2 *>(xb)[i] = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
}

#endif

#ifndef WUNET_TC_IO_ONLY
// weights [Cout][Cin][K] fp32 -> [K][Npad][Ktot] 16-bit elements, K axis = [seg0 padded to 64 | seg1 padded to 64], zero padded
__global__ void pack_tc_kernel(const float *__restrict__ w, const float *__restrict__ scale, const float *__restrict__ shift,
                               TcT *__restrict__ wp, float2 *__restrict__ ss, int Cout, int Cin0, int Cin1, int K,
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
        wp[i] = TcElem::cvt(v);
    }
    if (i < Npad) ss[i] = (i < Cout) ? make_float2(scale[i], shift[i]) : make_float2(0.f, 0.f);
}

// experimental: the extra K slot of a merged tail chunk, [t][co][Ktot - 64 + j]: j < s -> skip tail channel, j < s + u ->
// upsampled tail channel, else 0 (the regular slots are written by pack_tc_kernel, which leaves this one untouched = 0)
__global__ void pack_tc_merged_kernel(const float *__restrict__ w, TcT *__restrict__ wp, int Cout, int Cin0, int Cin1,
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
    wp[((size_t)t * Npad + co) * Ktot + (Ktot - 64) + j] = TcElem::cvt(v);
}

#ifndef WUNET_TC_FP16
// split-precision ("fp32_tc") weights: K-loop position c of a block multiplies the data part (hi / lo) of one 64-channel chunk
// with the high or the low bf16 part of the fp32 weights; SplitTable lists, per position, the first original input channel of
// the chunk, its width and which weight part it takes. wp[t][co][c * 64 + j], zero beyond the chunk's width (the TMA box of a
// chunk narrower than 64 channels reads on into the next channels of the row: they meet zero weights).
// SplitTable: wunet_tc_common.cuh
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

#endif

#ifndef WUNET_TC_FP16
__global__ void nlc_bf16_to_ncl_f32_kernel(const __nv_bfloat16 *__restrict__ src, float *__restrict__ dst, int B, int L, int C)
#else
__global__ void nlc_f16_to_ncl_f32_kernel(const __half *__restrict__ src, float *__restrict__ dst, int B, int L, int C)
#endif
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;       // index into dst [B][C][L]
    const long long n = (long long)B * C * L;
    if (i >= n) return;
    const int l = (int)(i % L);
    const int c = (int)((i / L) % C);
    const int b = (int)(i / ((long long)L * C));
    dst[i] = TcElem::to_f32(src[((size_t)b * L + l) * C + c]);
}

#endif  // WUNET_TC_IO_ONLY
#endif  // WUNET_TC_CONV_ONLY
