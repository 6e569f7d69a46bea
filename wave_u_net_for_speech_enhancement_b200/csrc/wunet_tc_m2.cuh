// wunet_tc_m2.cuh — the large flavour of conv_tc_kernel (wunet_tc_kernels.cuh) for the blocks that stream their weights from L2,
// with 256-row work units: each consumer warpgroup holds a whole 128-row tile, so every weight stage brought into shared memory
// serves 256 output rows instead of 128, and the stage hand-off is paid once per 256 rows. Included by wunet_tc_m2.cu after
// wunet_tc_kernels.cuh (its helpers: mbarriers, TMA, wgmma groups, chunk_info), once per element type.
//
// Everything else is conv_tc_kernel's behaviour for such a block (streamed weights, full-length frames, no split precision, no
// fused head, no row-pair form): the TMA lane issues the operand chunks one chunk ahead of the weight ring and slips them in
// between the weight stages; the upsample producers write the upsampled chunks with the same per-item code and register
// prefetch; a weight stage is released after wgmma.wait_group 0 by one arrival per consumer warpgroup.
//
// Work unit: tiles 2u and 2u + 1 of one frame and one column split (units_per_frame = tiles_per_frame / 2). p.tile_begin /
// p.tile_end count units; the CTA walks units first + k gridDim.x. An operand stage holds the unit's 256 + KS - 1 rows: p.nops = 2
// boxes of the plan's R1 rows (tmA is the plan's map). Warpgroup wg computes tile 2u + wg from the stage's rows wg 128 ...: both
// m64 row blocks (MB = 2, the small flavour's fragment shape) x NACC / 16 column blocks. Per accumulator the MMA sequence (chunk,
// tap, K16 step) is conv_tc_kernel's, only grouped into differently sized weight stages, and the epilogue arithmetic per element
// is the same, so the outputs are bit-identical.
//
// TRACE roles (WUNET_TC_TRACE builds, CTA 0): 0 = TMA lane around its operand-stage waits and after each weight-stage wait,
// 1 = consumer thread 0 before / after each weight-stage wait, 2 = consumer thread 0 at the start of each epilogue, 4 = upsample
// producer thread 0 before / after each operand-stage wait and after the hand-off.
template <int KS, bool UPCAT, int MG, int NACC>
__global__ void __launch_bounds__(32 + 32 * (kEpiWarpsLarge + (UPCAT ? kM2ProducerWarps : 0)), 1)
conv_tc_m2_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                  const __grid_constant__ CUtensorMap tmO, const TcParams p)
{
    constexpr int PAD = (KS - 1) / 2;
    constexpr int NPROD = kM2ProducerWarps * 32;
    constexpr int kFirstProducer = kEpiWarpsLarge;
    constexpr int kTmaWarp = kEpiWarpsLarge + (UPCAT ? kM2ProducerWarps : 0);
    (void)tmO;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t *base_ptr = smem_raw + (base - smem_u32(smem_raw));
    const SmemMap sm = smem_map(p);
    const uint32_t bars = base + sm.bars;
    // the barrier slots of conv_tc_kernel: a_full[4] a_empty[4] b_full[8] b_empty[8] | 5 unused | a_tma[4]
    const uint32_t a_full = bars, a_empty = bars + 32, b_full = bars + 64, b_empty = bars + 64 + 8 * kMaxBStages;
    const uint32_t a_tma = bars + 64 + 16 * kMaxBStages + 48;

    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int total_units = p.tile_end;
    const int first_unit = p.tile_begin + (int)blockIdx.x;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmW)) : "memory");
        for (int s = 0; s < 4; ++s) {
            mbar_init(a_full + 8 * s, UPCAT ? 1 + kM2ProducerWarps : 1);
            mbar_init(a_empty + 8 * s, kEpiWarpsLarge / 4);          // one arrival per consumer warpgroup
        }
        for (int s = 0; s < min(p.nb, kMaxBStages); ++s) { mbar_init(b_full + 8 * s, 1); mbar_init(b_empty + 8 * s, kEpiWarpsLarge / 4); }
        if (MG != 0 && p.mg)
            for (int s = 0; s < 4; ++s) mbar_init(a_tma + 8 * s, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    {   // folded BatchNorm scale/shift of all output columns
        float2 *ss = reinterpret_cast<float2 *>(base_ptr + sm.ss);
        for (int i = threadIdx.x; i < p.Npad; i += blockDim.x) ss[i] = p.ss[i];
    }
    __syncthreads();
    asm volatile("griddepcontrol.wait;" ::: "memory");

    // unit -> (frame, first row, first column)
    const int units_per_frame = p.tiles_per_frame >> 1;
    auto unit_coords = [&](int unit, int &b0, int &l0, int &n0) {
        const int mi = unit / p.nsplit;
        n0 = (unit - mi * p.nsplit) * p.Nh;
        b0 = mi / units_per_frame;
        l0 = (mi - b0 * units_per_frame) * 256;
    };

    if (warp == kTmaWarp) {
        // ======================= TMA producer =======================
        if (lane == 0) {
            int sa = 0, pa = 0, sb = 0, pb = 0;
            int tr0 = 0; (void)tr0;
            // operand chunks are issued one chunk ahead of the weight stream (across unit boundaries)
            int a_unit = first_unit, a_c = 0;
            // returns false if the stage is still in use and blocking == false
            auto issue_a = [&](bool blocking) -> bool {
                if (a_unit >= total_units) return true;
                if (!blocking && !mbar_test(a_empty + 8 * sa, pa ^ 1)) return false;
                int b0, l0, n0;
                unit_coords(a_unit, b0, l0, n0);
                const ChunkInfo aci = chunk_info<UPCAT, MG>(p, a_c);
                TRACE(0, tr0);
                mbar_wait(a_empty + 8 * sa, pa ^ 1);
                TRACE(0, tr0);
                if (!aci.up) {
                    mbar_expect_tx(a_full + 8 * sa, p.a_tx_bytes);
                    for (int op = 0; op < p.nops; ++op)
                        tma_load_3d(base + sm.a + sa * p.a_stage_bytes + op * p.R1 * 128, &tmA, a_full + 8 * sa, aci.idx * 64,
                                    l0 - PAD + op * p.R1, b0);
                } else if (MG != 0 && aci.merged) {
                    // skip tail into the leading vectors of the stage (completion on a_tma); the producers add the upsampled
                    // tail once it has landed and complete a_full
                    mbar_expect_tx(a_tma + 8 * sa, p.a_tx_bytes);
                    for (int op = 0; op < p.nops; ++op)
                        tma_load_3d(base + sm.a + sa * p.a_stage_bytes + op * p.R1 * 128, &tmA, a_tma + 8 * sa, p.mg_skip_idx * 64,
                                    l0 - PAD + op * p.R1, b0);
                    mbar_arrive(a_full + 8 * sa);
                } else {
                    mbar_arrive(a_full + 8 * sa);
                }
                if (++sa == p.na) { sa = 0; pa ^= 1; }
                if (++a_c == p.nchunks) { a_c = 0; a_unit += gridDim.x; }
                return true;
            };
            for (int pre = 0; pre < p.na - 1; ++pre) issue_a(true);          // operand chunks run na - 1 chunks ahead of the weights
            if (p.na == 1) issue_a(true);
            for (int unit = first_unit; unit < total_units; unit += gridDim.x) {
                int b0, l0, n0;
                unit_coords(unit, b0, l0, n0);
                for (int c = 0; c < p.nchunks; ++c) {
                    // the weight stages of this chunk go out as soon as their ring slots free up; the operand chunk of the NEXT
                    // K position is slipped in between them the moment its stage is released (it never blocks the weights)
                    bool a_done = false;
                    const int kslot = chunk_info<UPCAT, MG>(p, c).kslot;
                    for (int g = 0; g < p.ngroups; ++g) {
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
    } else if (warp < kEpiWarpsLarge) {
        // ======================= consumer warpgroups: one whole tile of the unit each =======================
        // Fragment of m64nNk16 (f32): thread (warp wq, lane) holds rows 16 wq + lane / 4 (+8) of each m64 block and columns
        // 2 (lane % 4) (+1) of every 8-column group.
        constexpr int MB = 2;
        constexpr int NB = NACC / 16;
        const int wg = warp >> 2, wq = warp & 3;
        const bool wg_leader = (threadIdx.x & 127) == 0;
        const float2 *ss = reinterpret_cast<const float2 *>(base_ptr + sm.ss);
        const uint32_t b_step = ((uint32_t)p.Nh * 128) >> 4;
        // descriptor words: hi = SBO(1024 B) | SWIZZLE_128B, lo = (addr >> 4) | LBO(1)
        const uint32_t hi = (uint32_t)(1024 >> 4) | (1u << 30);
        int sa = 0, pa = 0, sb = 0, pb = 0;
        int tr1 = 0, tr2 = 0; (void)tr1; (void)tr2;
        for (int unit = first_unit; unit < total_units; unit += gridDim.x) {
            int b0, l0, n0;
            unit_coords(unit, b0, l0, n0);
            const int nt = min(p.Nh, p.Npad - n0) >> 4;     // 16-column blocks of this CTA (the last column split may be narrower)
            float acc[MB][8 * NB];
#pragma unroll
            for (int mb = 0; mb < MB; ++mb)
#pragma unroll
                for (int j = 0; j < 8 * NB; ++j) acc[mb][j] = 0.f;
            for (int c = 0; c < p.nchunks; ++c) {
                const ChunkInfo mci = chunk_info<UPCAT, MG>(p, c);
                mbar_wait(a_full + 8 * sa, pa);
                const uint32_t a_base = base + sm.a + sa * p.a_stage_bytes + (uint32_t)(wg * 128 * 128);   // this warpgroup's tile
                const uint32_t a_lo0 = ((a_base >> 4) & 0x3FFFu) | (1u << 16);
                for (int g = 0; g < p.ngroups; ++g) {
                    if (threadIdx.x == 0) TRACE(1, tr1);
                    mbar_wait(b_full + 8 * sb, pb);
                    if (threadIdx.x == 0) TRACE(1, tr1);
                    const uint32_t b_base = base + sm.b + sb * p.b_stage_bytes;
                    const uint32_t b_lo0 = ((b_base >> 4) & 0x3FFFu) | (1u << 16);
                    const int t0 = g * p.tg, t_end = min(KS, (g + 1) * p.tg);
#pragma unroll 1
                    for (int t = t0; t < t_end; t += kMaxGroupTaps)
                        wgmma_group_taps<MB, 8 * NB>(min(kMaxGroupTaps, t_end - t), nt, mci.nk, acc, a_lo0 + (uint32_t)t * 8u,   // tap shift: +128 B
                                                     b_lo0 + (uint32_t)(t - t0) * b_step, hi, b_step);
                    wgmma_wait0();
                    if (wg_leader) mbar_arrive(b_empty + 8 * sb);
                    if (++sb == p.nb) { sb = 0; pb ^= 1; }
                }
                if (wg_leader) mbar_arrive(a_empty + 8 * sa);
                if (++sa == p.na) { sa = 0; pa ^= 1; }
            }
            // epilogue
            if (threadIdx.x == 0) TRACE(2, tr2);
#pragma unroll
            for (int mb = 0; mb < MB; ++mb) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int l = l0 + wg * 128 + mb * 64 + 16 * wq + (lane >> 2) + 8 * h;
                    const bool valid = (b0 < p.B) && (l < p.L);
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
                            if (valid && col_ok)
                                *reinterpret_cast<uint32_t *>(static_cast<TcT *>(p.out) + ((size_t)b0 * p.L + l) * p.Cout + n0 + col) = TcElem::pack(f0, f1);
                        }
                    }
                }
            }
        }
    } else if (UPCAT) {
        // ======================= upsample producers =======================
        // conv_tc_kernel's path for full-length frames: a thread owns 16 consecutive output rows x one 16-byte channel vector and
        // interpolates them from the RPI / 2 + 2 previous-level rows it holds in registers; the first item of a chunk is loaded
        // when the K loop reaches the chunk (before the stage wait), later rounds on demand. A unit's upsampled chunk has
        // rows_used = 256 + KS - 1 rows, 17 runs of 16 rows: a full chunk's 136 items take two rounds of the 96 producer threads,
        // as they would of 128.
        constexpr int RPI = 16, WR = RPI / 2 + 2;
        const int pt = (warp - kFirstProducer) * 32 + lane;
        int sa = 0, pa = 0;
        int tr4 = 0; (void)tr4;
        uint32_t tma_par = 0;                              // merged chunks: phase parity of a_tma[stage], one bit per stage
        uint4 xr[WR];
        bool pref = false;
        const int nruns = (p.rows_used + RPI - 1) / RPI;
        auto fetch = [&](int ub0, int ul0, int c, int item) {
            const ChunkInfo u = chunk_info<UPCAT, MG>(p, c);
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
        auto emit = [&](uint8_t *dst, int l0, int c, int item) {
            const ChunkInfo u = chunk_info<UPCAT, MG>(p, c);
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
                const float lam1 = fmaf(p.up_scale, lf0 + (float)j, -(mf0 + (float)qa));
                const TcT2 lam = TcElem::to2(lam1);
                const TcT2 *a2 = reinterpret_cast<const TcT2 *>(&xr[qa]);
                const TcT2 *b2 = reinterpret_cast<const TcT2 *>(&xr[qa + 1]);
                TcT2 r2[4];
#pragma unroll
                for (int q4 = 0; q4 < 4; ++q4) r2[q4] = __hfma2(lam, __hsub2(b2[q4], a2[q4]), a2[q4]);
                uint4 o = *reinterpret_cast<const uint4 *>(r2);
                const uint32_t keep = (chok && (unsigned)l < (unsigned)p.L) ? 0xffffffffu : 0u;   // zero rows = Conv1d padding
                o.x &= keep; o.y &= keep; o.z &= keep; o.w &= keep;
                st_shared_v4_if(drow + (uint32_t)(j * 128 + ((dvec ^ (j & 7)) << 4)), o, RPI * run + j < p.rows_used);
            }
        };
        for (int unit = first_unit; unit < total_units; unit += gridDim.x) {
            int b0, l0, n0;
            unit_coords(unit, b0, l0, n0);
            for (int c = 0; c < p.nchunks; ++c) {
                const ChunkInfo cu = chunk_info<UPCAT, MG>(p, c);
                if (cu.up && !pref) fetch(b0, l0, c, pt);
                if (pt == 0) TRACE(4, tr4);
                mbar_wait(a_empty + 8 * sa, pa ^ 1);
                if (pt == 0) TRACE(4, tr4);
                if (cu.up) {
                    if (MG != 0 && cu.merged) {                               // the TMA part of this stage must have landed
                        mbar_wait(a_tma + 8 * sa, (tma_par >> sa) & 1u);
                        tma_par ^= 1u << sa;
                    }
                    uint8_t *dst = base_ptr + sm.a + sa * p.a_stage_bytes;
                    const int nitems = nruns * cu.nvec;
#pragma unroll 1
                    for (int itx = pt; itx < nitems; itx += NPROD) {
                        if (itx != pt) fetch(b0, l0, c, itx);                // later rounds load on demand
                        emit(dst, l0, c, itx);
                    }
                    pref = false;
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> tensor core reads
                }
                __syncwarp();
                if (pt == 0) TRACE(4, tr4);
                if (lane == 0) mbar_arrive(a_full + 8 * sa);
                if (++sa == p.na) { sa = 0; pa ^= 1; }
                if (cu.up && !p.pf_late) {
                    // next upsampled chunk of this CTA (K-loop order): prefetch its first-round item after the hand-off
                    int nu = unit, nc = c + 1;
                    for (int hop = 0; hop < p.nchunks; ++hop) {
                        if (nc >= p.nchunks) { nc = 0; nu += gridDim.x; }
                        if (chunk_info<UPCAT, MG>(p, nc).up) break;
                        ++nc;
                    }
                    if (nu < total_units && chunk_info<UPCAT, MG>(p, nc).up) {
                        int nb0, nl0, nn0;
                        unit_coords(nu, nb0, nl0, nn0);
                        fetch(nb0, nl0, nc, pt);
                        pref = true;
                    }
                }
            }
        }
    }
}
