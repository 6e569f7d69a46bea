// wunet_tc_common.cuh — what the host code of the tensor-core inference path (wunet_tc.cu) shares with the device code of
// both element types (wunet_tc_kernels.cuh, compiled in wunet_tc.cu for bf16 and in wunet_tc_f16.cu for fp16).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stddef.h>
#include <stdint.h>

#include "wunet_wgmma.cuh"

namespace wunet {

namespace {

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
    const void *prev;          // DEC: previous block output [B][L/2][Cin0] (TcT elements)
    int Lin;
    float up_scale;
    const float2 *ss;          // [Npad] (scale, shift)
    void *out;                 // [B][L][Cout] (TcT elements) or nullptr (fused head without debug store)
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
    void *out;                     // [B][N] (TcT elements)
};
constexpr int kGemmThreads = 32 * (kEpiWarpsLarge + 1);   // two consumer warpgroups + the TMA warp

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

__host__ __device__ inline float group8_weight(const float *w, int Cout, int K, int cov, int q, int tv)
{
    const int r = cov / Cout, co = cov - r * Cout;
    const int t = 8 * (tv - 1) + q - r + (K - 1) / 2;
    if (r > 7 || q > 7 || t < 0 || t >= K) return 0.f;
    return w[(size_t)co * K + t];
}

// split-precision ("fp32_tc") weights: K-loop position c of a block multiplies the data part (hi / lo) of one 64-channel chunk
// with the high or the low bf16 part of the fp32 weights; SplitTable lists, per position, the first original input channel of
// the chunk, its width and which weight part it takes. wp[t][co][c * 64 + j], zero beyond the chunk's width (the TMA box of a
// chunk narrower than 64 channels reads on into the next channels of the row: they meet zero weights).
struct SplitTable { short base[48]; unsigned char width[48], wlo[48]; int n; };

// Element traits of the two 16-bit activation / weight types. Every conversion from fp32 rounds to nearest even.
//   pack(a, b): two values -> one 32-bit word, a in the low half;  cvt(v): one value;  to2(v): v in both halves;
//   f2(u): the word back to two floats;  to_f32(v): one element back to float.
struct TcBf16 {
    using T = __nv_bfloat16;
    using T2 = __nv_bfloat162;
    static __device__ __forceinline__ uint32_t pack(float a, float b) { return pack_bf16(a, b); }
    static __device__ __forceinline__ T cvt(float v) { return __float2bfloat16_rn(v); }
    static __device__ __forceinline__ T2 to2(float v) { return __float2bfloat162_rn(v); }
    static __device__ __forceinline__ float2 f2(uint32_t u) { return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&u)); }
    static __device__ __forceinline__ float to_f32(T v) { return __bfloat162float(v); }
};
// fp16 saturates: every fp32 -> fp16 store goes through cvt.rn.satfinite.f16x2.f32 (one F2FP.SATFINITE.F16.F32.PACK_AB on
// sm_90a), so a value beyond +-65504 is stored as +-65504, never as inf. The one fp16 operation that can still overflow is
// the packed interpolation's b - a (to2 / __hsub2 in the decoder producers) of two adjacent upsampled values more than 65504 apart.
struct TcF16 {
    using T = __half;
    using T2 = __half2;
    static __device__ __forceinline__ uint32_t pack(float a, float b)
    {
        uint32_t r;
        asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));   // first source -> upper half
        return r;
    }
    static __device__ __forceinline__ T cvt(float v) { return __ushort_as_half((unsigned short)(pack(v, 0.f) & 0xffffu)); }
    static __device__ __forceinline__ T2 to2(float v) { return __float2half2_rn(v); }
    static __device__ __forceinline__ float2 f2(uint32_t u) { return __half22float2(*reinterpret_cast<const __half2 *>(&u)); }
    static __device__ __forceinline__ float to_f32(T v) { return __half2float(v); }
};

// The fp16 kernels (wunet_tc_f16.cu): the same forms and arguments as the bf16 ones, launched by the host code of wunet_tc.cu.
namespace f16 {
using ConvKernel = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, TcParams);
using GemmKernel = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, GemmParams);
void set_smem_attributes();
// ks = 15: encoder, 5: decoder (up + concat; mg: its K loop ends in a merged tail chunk), 9: row-pair encoder; small: the
// two-CTAs-per-SM flavour
ConvKernel conv_kernel(int ks, bool small, bool mg);
GemmKernel gemm_kernel();
cudaError_t launch_enc0(const cudaLaunchConfig_t &cfg, bool persistent, const float *x, const float *w, const float *scale,
                        const float *shift, void *out, int B, int T, int C, void *even_out);
cudaError_t pack(const float *w, const float *scale, const float *shift, void *wp, float2 *ss, int Cout, int Cin0, int Cin1, int K,
                 int Npad, int Ktot, cudaStream_t stream);
cudaError_t pack_merged(const float *w, void *wp, int Cout, int Cin0, int Cin1, int K, int Npad, int Ktot, int s, int u,
                        cudaStream_t stream);
cudaError_t expand_gemm_weights(const float *w, void *wx, size_t n, int Cout, int Cin0, int Cin1, int K, int L, int dec, int npos0,
                                int cpp0, int npos1, int cpp1, float up_scale, cudaStream_t stream);
cudaError_t nlc_to_ncl(const void *src, float *dst, int B, int L, int C, cudaStream_t stream);
}  // namespace f16

// The kernels only wide channel plans (40 <= channels_interval <= 64) launch (wunet_tc_wide.cu).
namespace wide {
using ConvKernel = f16::ConvKernel;
void set_smem_attributes();
// block 0 with a tile that shrinks with C; mode 0 = bf16, 1 = split precision, 2 = fp16. Sets cfg's grid, block and shared memory.
// x: B*T samples of the IoType io (16-bit: the io_f16 / io_bf16 form, on the same grid)
cudaError_t launch_enc0(cudaLaunchConfig_t cfg, int mode, const void *x, const float *w, const float *scale, const float *shift, void *out,
                        int B, int T, int C, int io);
// split-precision conv form for blocks of more than 48 K-loop positions (chunk_map lists chunks: chunk_info, SP = 2); large flavour
ConvKernel conv_split_kernel(bool upcat);
// its weights: tab lists the chunks (base, width) and the positions (n = 3 x chunks)
cudaError_t pack_split(const float *w, void *wp, int Cout, int Cin, int K, int Npad, const SplitTable &tab, cudaStream_t stream);
}  // namespace wide

// The ping-pong form of the large decoder flavour (wunet_tc_pp.cu): each consumer warpgroup owns whole tiles, so that one
// warpgroup's epilogue runs under the other's MMAs. bf16 and fp16 (plan mode 2), float I/O.
namespace pp {
using ConvKernel = f16::ConvKernel;
void set_smem_attributes();
ConvKernel conv_kernel(bool fp16, bool mg);
// whether a block of this plan runs the ping-pong form: the last decoder block (fused head), weight-resident, large flavour, one
// column split of at most kPpAccCols columns, full-length frames, no split precision, float I/O (io: IoType of the forward).
// The other resident decoders are bound by their upsample producers, and the form measured no faster there (DESIGN §5.1).
bool selected(const TcParams &p, bool upcat, bool small, int io);
}  // namespace pp

// The 256-row form of the large flavour for the blocks that stream their weights from L2 (wunet_tc_m2.cu): a work unit is two
// tiles of one frame, one per consumer warpgroup, so each weight stage serves 256 output rows. bf16 and fp16 (plan mode 2).
namespace m2 {
using ConvKernel = f16::ConvKernel;
// accumulator columns: 2 x 48 fp32 registers per consumer thread. ptxas sizes the register budget for whole warpgroups: 288
// (encoder) or 384 (decoder) threads per CTA leave 168 registers per thread, 416 only 128. Blocks of 128 columns per CTA keep
// the 128-row tiles: next to 256-row operand stages their weight stages hold 4 taps, and enc4 measured no faster so.
constexpr int kM2AccCols = 96;
constexpr int kM2ProducerWarps = 3;    // upsample producers of the decoder form (conv_tc_kernel: 4, 416 threads per CTA)
void set_smem_attributes();
ConvKernel conv_kernel(bool fp16, bool upcat, bool mg);
// work units (two tiles of one frame and one column split) of a plan; 0 for packed frames or an odd tile count per frame
int units(const TcParams &p);
// the block's parameters in this form, from its plan p (ks taps): operand stages of 256 + ks - 1 rows, the weight ring re-fitted
// next to them (na, tg, ngroups, nb), tile_begin / tile_end counting units; false if it does not fit in shared memory
bool geometry(const TcParams &p, int ks, TcParams &q);
// whether a block of this plan runs the form: bf16 / fp16 (no split precision), not the head, the large flavour and no row-pair
// form (pair == 0), streamed weights, full-length frames with an even tile count, at most kM2AccCols columns per CTA, at
// least num_sms units (small batches keep the 128-row tiles on every SM), and a geometry that fits.
// The host also requires float network I/O.
bool selected(const TcParams &p, int ks, bool upcat, bool small, int pair, int num_sms);
}  // namespace m2

// The forms with a 16-bit network input / output (wunet_tc_io.cuh): io_f16 (__half, wunet_tc_io_f16.cu) and io_bf16
// (__nv_bfloat16, wunet_tc_io_bf16.cu) have the same functions. mode: 0 = bf16, 1 = split precision, 2 = fp16 (tc_* modes).
#define WUNET_TC_IO_DECLS                                                                                                           \
    /* the last block (fused head), large flavour; mg: its K loop ends in a merged tail chunk (bf16 / fp16 modes) */                  \
    ::wunet::f16::ConvKernel head_kernel(int mode, bool mg);                                                                                 \
    void set_smem_attributes(int enc0_wide_max);                                                                                    \
    /* block 0, one tile per CTA (enc0_kernel's grid and shared memory in cfg) */                                                   \
    cudaError_t launch_enc0(const cudaLaunchConfig_t &cfg, int mode, const void *x, const float *w, const float *scale,             \
                            const float *shift, void *out, int B, int T, int C, void *even_out);                                   \
    /* block 0 of the wide plans (enc0_wide_kernel's grid and shared memory in cfg) */                                              \
    cudaError_t launch_enc0_wide(const cudaLaunchConfig_t &cfg, int mode, const void *x, const float *w, const float *scale,        \
                                 const float *shift, void *out, int B, int T, int C);                                              \
    /* the bf16 copy of the input for the group-of-8 block 0 */                                                                     \
    cudaError_t launch_x_to_bf16(const void *x, __nv_bfloat16 *xb, long long n4, cudaStream_t stream);
namespace io_f16 { WUNET_TC_IO_DECLS }
namespace io_bf16 { WUNET_TC_IO_DECLS }
#undef WUNET_TC_IO_DECLS

}  // namespace wunet
