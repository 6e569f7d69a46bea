// wunet_tc_wide.cuh — device code that only the wide channel plans (40 <= channels_interval <= 64) of the tensor-core inference
// path use. Included by wunet_tc_wide.cu (and by wunet_tc_io.cuh for the 16-bit I/O forms of enc0_wide_kernel), once per element
// type, after wunet_tc_kernels.cuh (WUNET_TC_CONV_ONLY / WUNET_TC_IO_ONLY) in the same namespace: TcElem, TcT, TcIO and lrelu come
// from there.

// -------------------------------------------------------------------------------------------------
// enc0 with a tile that shrinks with C
// -------------------------------------------------------------------------------------------------
// enc0_kernel stages 1024 positions x RC 16-bit channels (RC = 2 C in split-precision mode) for one bulk store; at C = 40 split
// that is 160 KiB. Here the block's 256 threads are S slices of 256 / S position groups: a tile is 1024 / S positions, and slice s
// sweeps the channel groups c0 = 8 s, 8 (s + S), ... of its 4 positions. Per output value the taps, their order, the fmaf chain,
// the folded BatchNorm, LeakyReLU and the conversions are those of enc0_kernel, so the output is the one it would write with
// enough shared memory. No dense copy of the even rows: the row-pair form of block 1 is off for wide plans.
template <int S>
__global__ void __launch_bounds__(256, 3) enc0_wide_kernel(const TcIO *__restrict__ x, const float *__restrict__ w /*[C][1][15]*/,
                                                           const float *__restrict__ scale, const float *__restrict__ shift,
                                                           TcT *__restrict__ out, int B, int T, int C, int split)
{
    constexpr int KS = 15, PAD = 7, TILE = 1024 / S, NPG = 256 / S;
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    extern __shared__ uint8_t smem_raw[];
    float *ws = reinterpret_cast<float *>(smem_raw);          // [15][C]
    float *sc = ws + KS * C, *sh = sc + C;
    float *xs = sh + C + ((4 - ((KS * C + 2 * C) & 3)) & 3);  // 16-byte aligned: xs[i] = x[l0 - 8 + i], i < TILE + 16
    uint8_t *stage = reinterpret_cast<uint8_t *>(xs + TILE + 16);   // [TILE][RC]
    const int RC = split ? 2 * C : C;
    const int b = blockIdx.y;
    const int l0 = blockIdx.x * TILE;
    const int pg = threadIdx.x % NPG, slice = threadIdx.x / NPG;   // warp-uniform slice (NPG >= 64)
    for (int i = threadIdx.x; i < KS * C; i += 256) { const int k = i / C, c = i - k * C; ws[i] = w[c * KS + k]; }
    for (int i = threadIdx.x; i < C; i += 256) { sc[i] = scale[i]; sh[i] = shift[i]; }
    asm volatile("griddepcontrol.wait;" ::: "memory");
    for (int i = threadIdx.x; i < TILE + 16; i += 256) {
        const int l = l0 - PAD + i - 1;
        xs[i] = (l >= 0 && l < T) ? io_f32(x[(size_t)b * T + l]) : 0.f;
    }
    __syncthreads();
    float xw[20];
#pragma unroll
    for (int q = 0; q < 5; ++q) {
        const float4 v = *reinterpret_cast<const float4 *>(&xs[4 * pg + 4 * q]);
        xw[4 * q] = v.x; xw[4 * q + 1] = v.y; xw[4 * q + 2] = v.z; xw[4 * q + 3] = v.w;
    }
    for (int c0 = 8 * slice; c0 < C; c0 += 8 * S) {
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
            uint8_t *srow = stage + (size_t)(4 * pg + j) * (RC * 2) + c0 * 2;
            *reinterpret_cast<uint4 *>(srow) =
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

#if !defined(WUNET_TC_FP16) && !defined(WUNET_TC_IO_ONLY)
// -------------------------------------------------------------------------------------------------
// split-precision weights of the SP = 2 conv form (chunk_info): per 64-channel chunk q, positions 3q .. 3q + 2
// -------------------------------------------------------------------------------------------------
// tab.base / tab.width list the chunks (first original input channel, width), tab.n the positions. Position c takes the high
// bf16 part of the fp32 weights, or the low part at c % 3 == 1: the values pack_tc_split_kernel writes for the same position.
__global__ void pack_tc_split_wide_kernel(const float *__restrict__ w, __nv_bfloat16 *__restrict__ wp, int Cout, int Cin, int K, int Npad,
                                          const SplitTable tab)
{
    const int Ktot = tab.n * 64;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)K * Npad * Ktot) return;
    const int ks = (int)(i % Ktot);
    const int co = (int)((i / Ktot) % Npad);
    const int t = (int)(i / ((long long)Ktot * Npad));
    const int c = ks >> 6, j = ks & 63, q = c / 3;
    float v = 0.f;
    if (co < Cout && j < tab.width[q]) {
        const float wf = w[((size_t)co * Cin + tab.base[q] + j) * K + t];
        const float hi = __bfloat162float(__float2bfloat16_rn(wf));
        v = (c % 3) == 1 ? wf - hi : hi;
    }
    wp[i] = __float2bfloat16_rn(v);
}
#endif
