// wunet_tc_pp.cuh — ping-pong form of the large decoder flavour of conv_tc_kernel (wunet_tc_kernels.cuh) for the weight-resident
// blocks: each consumer warpgroup owns whole 128-row tiles, and the two alternate, so that one runs its MMAs while the other runs
// its epilogue. Included by wunet_tc_pp.cu after wunet_tc_kernels.cuh (its helpers: mbarriers, TMA, wgmma groups, chunk_info),
// once per element type.
//
// Everything but the consumer role is conv_tc_kernel's behaviour for such a block (UPCAT, resident weights, one column split,
// full-length frames, no split precision, no head-only or row-pair form): the TMA lane preloads the weights before
// griddepcontrol.wait and then issues the skip chunks in K-loop order; the upsample producers write the upsampled chunks with the
// same register prefetch; the plan's ring (na stages, smem_map) is used as it is.
//
// Consumers: warpgroup w takes the CTA's tiles k = w, w + 2, ... of the sequence first_tile + k gridDim.x. A tile is both m64
// row blocks (MB = 2) x 16 nt columns, the small flavour's fragment shape; the K loop, the tap order and the epilogue arithmetic
// per element are conv_tc_kernel's, so the outputs are bit-identical. The MMA phases of the two warpgroups do not interleave: the
// "MMA turn" passes from tile k's warpgroup to tile k + 1's (named barrier kTurnBar + owner of k + 1) right after tile k's last
// wgmma group is committed, and tile k + 1's warpgroup takes it before its first wgmma. An arrival happens for k + 1 < n and a
// wait for k > 0, with n the CTA's tile count, which both warpgroups compute the same way: every arrival meets exactly one wait,
// and the alternation keeps a second arrival on a barrier from coming before the wait on the first. Since the MMA phases run in
// tile order, the warpgroups consume the operand ring in the global (tile, chunk) order: chunk c of tile k is ring position
// k nchunks + c, and only its owner releases the stage (a_empty expects one arrival).
constexpr int kPpAccCols = 80;         // accumulator columns: 2 x 40 fp32 registers per consumer thread (blocks with Nh <= 80)
constexpr int kTurnBar = 1;            // named barriers kTurnBar + w: the MMA turn passes to warpgroup w (0: __syncthreads)

namespace {
__device__ __forceinline__ void named_bar_sync(int id, int nthreads)
{
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads)
{
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
}  // namespace

template <int MG>
__global__ void __launch_bounds__(32 + 32 * (kEpiWarpsLarge + kProducerWarpsLarge), 1)
conv_tc_pp_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
                  const __grid_constant__ CUtensorMap tmO, const TcParams p)
{
    constexpr int KS = 5, PAD = 2;
    constexpr int NPROD = kProducerWarpsLarge * 32;
    constexpr int kFirstProducer = kEpiWarpsLarge;
    constexpr int kTmaWarp = kEpiWarpsLarge + kProducerWarpsLarge;
    (void)tmO;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t *base_ptr = smem_raw + (base - smem_u32(smem_raw));
    const SmemMap sm = smem_map(p);
    const uint32_t bars = base + sm.bars;
    // the barrier slots of conv_tc_kernel: a_full[4] a_empty[4] b_full[8] b_empty[8] | 5 unused | a_tma[4]
    const uint32_t a_full = bars, a_empty = bars + 32, b_full = bars + 64;
    const uint32_t a_tma = bars + 64 + 16 * kMaxBStages + 48;

    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int total_tiles = p.tile_end;
    const int first_tile = p.tile_begin + (int)blockIdx.x;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmW)) : "memory");
        for (int s = 0; s < 4; ++s) {
            mbar_init(a_full + 8 * s, 1 + kProducerWarpsLarge);
            mbar_init(a_empty + 8 * s, 1);                            // released by the warpgroup that owns the stage's tile
        }
        mbar_init(b_full, 1);
        if (MG != 0 && p.mg)
            for (int s = 0; s < 4; ++s) mbar_init(a_tma + 8 * s, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    {   // folded BatchNorm scale/shift of all output columns, head weights
        float2 *ss = reinterpret_cast<float2 *>(base_ptr + sm.ss);
        for (int i = threadIdx.x; i < p.Npad; i += blockDim.x) ss[i] = p.ss[i];
        if (p.head) {
            float *hw = reinterpret_cast<float *>(base_ptr + sm.ss) + 2 * p.Npad;
            if ((int)threadIdx.x <= p.Cout) hw[threadIdx.x] = p.head_w[threadIdx.x];
            if ((int)threadIdx.x == p.Cout + 1) hw[threadIdx.x] = p.head_b[0];
        }
    }
    __syncthreads();
    if (warp != kTmaWarp) asm volatile("griddepcontrol.wait;" ::: "memory");   // the TMA lane waits after the weight preload

    // tile -> (frame, first row); one column split, full-length frames
    auto tile_coords = [&](int tile, int &b0, int &l0) {
        b0 = tile / p.tiles_per_frame;
        l0 = (tile - b0 * p.tiles_per_frame) * 128;
    };

    if (warp == kTmaWarp) {
        // ======================= TMA producer =======================
        if (lane == 0) {
            int tr0 = 0; (void)tr0;
            // the whole packed weight set of this block (nchunks x KS taps of [Nh x 64]) is loaded once per CTA
            mbar_expect_tx(b_full, (uint32_t)p.nchunks * p.ngroups * p.tg * p.Nh * 128);
            for (int c = 0; c < p.nchunks; ++c) {
                const int kslot = chunk_info<true, MG>(p, c).kslot;
                for (int g = 0; g < p.ngroups; ++g)
                    tma_load_3d(base + sm.b + (uint32_t)(c * p.ngroups + g) * p.b_stage_bytes, &tmW, b_full, kslot * 64, 0, g * p.tg);
            }
            asm volatile("griddepcontrol.wait;" ::: "memory");        // activations of the previous block from here on
            int sa = 0, pa = 0;
            for (int tile = first_tile; tile < total_tiles; tile += gridDim.x) {
                int b0, l0;
                tile_coords(tile, b0, l0);
                for (int c = 0; c < p.nchunks; ++c) {
                    const ChunkInfo aci = chunk_info<true, MG>(p, c);
                    TRACE(0, tr0);
                    mbar_wait(a_empty + 8 * sa, pa ^ 1);
                    TRACE(0, tr0);
                    if (!aci.up) {
                        mbar_expect_tx(a_full + 8 * sa, p.a_tx_bytes);
                        for (int op = 0; op < p.nops; ++op)
                            tma_load_3d(base + sm.a + sa * p.a_stage_bytes + op * p.R1 * 128, &tmA, a_full + 8 * sa, aci.idx * 64,
                                        l0 - PAD + op * p.R1, b0);
                    } else if (MG != 0 && aci.merged) {
                        // skip tail into the leading vectors of the stage (completion on a_tma); the producers add the
                        // upsampled tail once it has landed and complete a_full
                        mbar_expect_tx(a_tma + 8 * sa, p.a_tx_bytes);
                        for (int op = 0; op < p.nops; ++op)
                            tma_load_3d(base + sm.a + sa * p.a_stage_bytes + op * p.R1 * 128, &tmA, a_tma + 8 * sa, p.mg_skip_idx * 64,
                                        l0 - PAD + op * p.R1, b0);
                        mbar_arrive(a_full + 8 * sa);
                    } else {
                        mbar_arrive(a_full + 8 * sa);
                    }
                    if (++sa == p.na) { sa = 0; pa ^= 1; }
                }
            }
        }
    } else if (warp < kEpiWarpsLarge) {
        // ======================= consumer warpgroups: one whole tile each, in turn =======================
        // Fragment of m64nNk16 (f32): thread (warp wq, lane) holds rows 16 wq + lane / 4 (+8) of each m64 block and columns
        // 2 (lane % 4) (+1) of every 8-column group.
        constexpr int MB = 2;
        constexpr int NB = kPpAccCols / 16;
        const int wg = warp >> 2, wq = warp & 3;
        const bool wg_leader = (threadIdx.x & 127) == 0;
        const float2 *ss = reinterpret_cast<const float2 *>(base_ptr + sm.ss);
        const float *hw = reinterpret_cast<const float *>(base_ptr + sm.ss) + 2 * p.Npad;
        const uint32_t b_step = ((uint32_t)p.Nh * 128) >> 4;
        const uint32_t hi = (uint32_t)(1024 >> 4) | (1u << 30);
        const int nt = min(p.Nh, p.Npad) >> 4;
        const int G = (int)gridDim.x;
        const int ntiles = first_tile < total_tiles ? (total_tiles - first_tile + G - 1) / G : 0;
        int tr = 0; (void)tr;
        const bool tracer = (threadIdx.x & 127) == 0;
        mbar_wait(b_full, 0);
        for (int k = wg; k < ntiles; k += 2) {
            int b0, l0;
            tile_coords(first_tile + k * G, b0, l0);
            float acc[MB][8 * NB];
#pragma unroll
            for (int mb = 0; mb < MB; ++mb)
#pragma unroll
                for (int j = 0; j < 8 * NB; ++j) acc[mb][j] = 0.f;
            if (k > 0) named_bar_sync(kTurnBar + wg, 256);          // tile k - 1's MMAs are all issued
            if (tracer) TRACE(1 + 2 * wg, tr);
            const bool pass = k + 1 < ntiles;
            for (int c = 0; c < p.nchunks; ++c) {
                const ChunkInfo mci = chunk_info<true, MG>(p, c);
                const int q = k * p.nchunks + c;                     // ring position
                const int sa = q % p.na, pa = (q / p.na) & 1;
                mbar_wait(a_full + 8 * sa, pa);
                const uint32_t a_base = base + sm.a + sa * p.a_stage_bytes;
                const uint32_t a_lo0 = ((a_base >> 4) & 0x3FFFu) | (1u << 16);
                for (int g = 0; g < p.ngroups; ++g) {
                    const uint32_t b_base = base + sm.b + (uint32_t)(c * p.ngroups + g) * p.b_stage_bytes;
                    const uint32_t b_lo0 = ((b_base >> 4) & 0x3FFFu) | (1u << 16);
                    const int t0 = g * p.tg, t_end = min(KS, (g + 1) * p.tg);
#pragma unroll 1
                    for (int t = t0; t < t_end; t += kMaxGroupTaps)
                        wgmma_group_taps<MB, 8 * NB>(min(kMaxGroupTaps, t_end - t), nt, mci.nk, acc, a_lo0 + (uint32_t)t * 8u,
                                                     b_lo0 + (uint32_t)(t - t0) * b_step, hi, b_step);
                    if (pass && c == p.nchunks - 1 && g == p.ngroups - 1) named_bar_arrive(kTurnBar + (wg ^ 1), 256);
                    wgmma_wait0();
                }
                if (wg_leader) mbar_arrive(a_empty + 8 * sa);
            }
            // epilogue
            if (tracer) TRACE(1 + 2 * wg, tr);
            // the head's raw-input samples of this thread's rows, all loaded up front: one global-load latency per tile instead
            // of one per row pair
            float xin[MB][2];
#pragma unroll
            for (int mb = 0; mb < MB; ++mb)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int l = l0 + mb * 64 + 16 * wq + (lane >> 2) + 8 * h;
                    xin[mb][h] = (p.head && b0 < p.B && l < p.L && (lane & 3) == 0)
                                     ? io_ld(reinterpret_cast<const TcIO *>(p.x) + (size_t)b0 * p.T + l) : 0.f;
                }
#pragma unroll
            for (int mb = 0; mb < MB; ++mb) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = mb * 64 + 16 * wq + (lane >> 2) + 8 * h;
                    const int l = l0 + row;
                    const bool valid = (b0 < p.B) && (l < p.L);
                    float hsum = 0.f;
#pragma unroll
                    for (int nb = 0; nb < NB; ++nb) {
                        if (nb >= nt) break;
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = nb * 16 + 8 * e + 2 * (lane & 3);
                            const float4 s2 = *reinterpret_cast<const float4 *>(&ss[col]);
                            const float f0 = lrelu(fmaf(acc[mb][8 * nb + 4 * e + 2 * h], s2.x, s2.y));
                            const float f1 = lrelu(fmaf(acc[mb][8 * nb + 4 * e + 2 * h + 1], s2.z, s2.w));
                            const bool col_ok = col < p.Cout;                             // Cout is even: both columns or none
                            if (p.out != nullptr && valid && col_ok)
                                *reinterpret_cast<uint32_t *>(static_cast<TcT *>(p.out) + ((size_t)b0 * p.L + l) * p.Cout + col) = TcElem::pack(f0, f1);
                            if (p.head && col_ok) hsum = fmaf(hw[col + 1], f1, fmaf(hw[col], f0, hsum));
                        }
                    }
                    if (p.head) {
                        // cat([o, input], 1) -> Conv1d(C+1 -> 1, k=1) -> Tanh; the four threads of a row hold interleaved column pairs
                        hsum += __shfl_xor_sync(0xffffffffu, hsum, 1);
                        hsum += __shfl_xor_sync(0xffffffffu, hsum, 2);
                        if (valid && (lane & 3) == 0) {
                            const float hacc = fmaf(hw[p.Cout], xin[mb][h], hw[p.Cout + 1] + hsum);
                            io_st(reinterpret_cast<TcIO *>(p.y) + (size_t)b0 * p.T + l, tanh_fast(hacc));
                        }
                    }
                }
            }
            if (tracer) TRACE(1 + 2 * wg, tr);
        }
    } else {
        // ======================= upsample producers =======================
        // conv_tc_kernel's generic decoder path for full-length frames: a thread owns 16 consecutive output rows x one 16-byte
        // channel vector and interpolates them from the RPI / 2 + 2 previous-level rows it holds in registers, loaded one work
        // unit ahead.
        constexpr int RPI = 16, WR = RPI / 2 + 2;
        const int pt = (warp - kFirstProducer) * 32 + lane;
        int sa = 0, pa = 0;
        int tr4 = 0; (void)tr4;
        uint32_t tma_par = 0;                              // merged chunks: phase parity of a_tma[stage], one bit per stage
        uint4 xr[WR];
        bool pref = false;
        const int nruns = (p.rows_used + RPI - 1) / RPI;
        auto fetch = [&](int ub0, int ul0, int c, int item) {
            const ChunkInfo u = chunk_info<true, MG>(p, c);
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
            const ChunkInfo u = chunk_info<true, MG>(p, c);
            const int nvec = u.nvec;
            const int run = item / nvec, vec = item - run * nvec;
            const int ch = u.idx * 64 + vec * 8;
            const int dvec = u.vo + vec;                                       // 16-byte vector inside the stage row
            const int lstart = l0 - PAD + RPI * run;                           // even
            const int ms = lstart >> 1;
            const bool chok = ch < p.Cin0;
            const float lf0 = (float)lstart, mf0 = (float)(ms - 1);
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
        for (int tile = first_tile; tile < total_tiles; tile += gridDim.x) {
            int b0, l0;
            tile_coords(tile, b0, l0);
            for (int c = 0; c < p.nchunks; ++c) {
                const ChunkInfo cu = chunk_info<true, MG>(p, c);
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
                    // next upsampled unit of this CTA (K-loop order): prefetch its first-round item after the hand-off
                    int nt = tile, nc = c + 1;
                    for (int hop = 0; hop < p.nchunks; ++hop) {
                        if (nc >= p.nchunks) { nc = 0; nt += gridDim.x; }
                        if (chunk_info<true, MG>(p, nc).up) break;
                        ++nc;
                    }
                    if (nt < total_tiles && chunk_info<true, MG>(p, nc).up) {
                        int nb0, nl0;
                        tile_coords(nt, nb0, nl0);
                        fetch(nb0, nl0, nc, pt);
                        pref = true;
                    }
                }
            }
        }
    }
}
