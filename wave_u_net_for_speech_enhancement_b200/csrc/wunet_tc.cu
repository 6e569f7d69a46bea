// wunet_tc.cu — bf16 tensor-core path of the Wave-U-Net forward for sm_90a (wgmma + TMA + mbarrier).
// The kernels below are those of wunet_tc_kernels.cuh (compiled here with bf16 elements, and again with fp16 ones in
// wunet_tc_f16.cu); this file holds their bf16 instantiation and the host code (planner, state, launches) of both.
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
#include "wunet_tc_common.cuh"

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

}  // namespace

// the bf16 kernels (and the split-precision fp32_tc ones); their fp16 twins are compiled in wunet_tc_f16.cu
using TcElem = TcBf16;
#include "wunet_tc_kernels.cuh"

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
    void *wx = nullptr;                // Toeplitz-expanded weights of the dense bottom-of-U GEMM (gemm_tc_kernel), built for wx_L positions
    int wx_L = 0;
    size_t wx_elems = 0;
    void *wp16 = nullptr;              // fp16 packing, wp's layout (packed by the first fp16 forward after the weights were set)
    void *wx16 = nullptr;              // fp16 Toeplitz expansion, wx's layout, built for wx16_L positions
    int wx16_L = 0;
    size_t wx16_elems = 0;
    __nv_bfloat16 *wp_sp = nullptr;    // split-precision packing [K][Npad][sp_chunks * 64] (sp_chunk_order lists the K-loop positions)
    int sp_chunks = 0;
    const float *w_src = nullptr;      // enc0 only: fp32 weights (w_own, a library-owned copy) / scale / shift (the context's folded copies)
    float *w_own = nullptr;            // enc0 only: [Cout][1][K] fp32 copy made by tc_set_weights (the caller's tensor is not read afterwards)
    const float *scale = nullptr, *shift = nullptr;
};

static int sp_chunk_order(const TcLevel &lv, bool dec, unsigned char *map, SplitTable *tab, bool wide = false);

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
    // the 256-row form of a streamed-weight block (wunet_tc_m2.cu; m2::selected): its parameters (operand stages, weight ring,
    // unit range), its weight map (the stage's tap count differs from the plan's), dynamic shared memory. Not part of the plan
    // record (wunet_debug_plan); launched for float network I/O.
    bool m2 = false;
    TcParams m2p;
    CUtensorMap tmW2;
    size_t m2_smem = 0;
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
    bool m2 = true;                    // 256-row form of the streamed-weight blocks where m2::selected (WUNET_TC_M2=0 switches it off)
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
    int plan_mode = 0;                 // 0: bf16 plan, 1: split-precision (fp32_tc) plan, 2: fp16 plan (the bf16 plan on fp16 data)
    bool f16_packed = false;           // the fp16 weight packings (wp16 of the blocks and the row-pair block) match the current weights
    CUtensorMapDataType map_type = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;   // element type of the tensor maps build_plan encodes
    TcPlan plan;
};

const char *tc_error() { return g_tc_err; }

// off[0 .. 2n] = block outputs; off[2n+1] = dense copy of block 0's even rows [B][T/2][ci] (bf16 / fp16 mode; row-pair mode of
// block 1); off[2n+2] = the raw input in bf16. Modes 0 (bf16) and 2 (fp16) have the same layout; mode 1 (split) stores two
// halves per channel and has neither copy.
static void tc_layout(int n, int ci, int B, int T, std::vector<size_t> &off, size_t &total, int mode = 0)
{
    off.resize(2 * n + 3);
    size_t cur = 0;
    for (int i = 0; i < 2 * n + 1; ++i) {
        const int L = (i <= n) ? (T >> i) : (T >> (2 * n - i));
        const int cout = (i < n) ? (i + 1) * ci : (i == n ? n * ci : (2 * n - i + 1) * ci);
        off[i] = cur;
        cur += round_up_sz((size_t)B * L * cout * sizeof(__nv_bfloat16) * (mode == 1 ? 2 : 1), 1024);
    }
    off[2 * n + 1] = cur;
    if (mode != 1) cur += round_up_sz((size_t)B * (T / 2) * ci * sizeof(__nv_bfloat16), 1024);
    off[2 * n + 2] = cur;                                 // bf16 copy of the raw input [B][T] (block 0 on the tensor cores)
    if (mode != 1) cur += round_up_sz((size_t)B * T * sizeof(__nv_bfloat16), 1024);
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
        if (const char *xe = getenv("WUNET_TC_M2")) st->m2 = xe[0] != '0';
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
    st->f16_packed = false;                              // and repack fp16 on the next fp16 forward
    derive_levels(st->levels, blocks, nblocks, n, st->merge && ci <= 32);     // no merged tail chunks in wide plans
    if (ci % 8 != 0 || ci > 64) return 0;                // tensor-core path unsupported for this plan; forward reports it
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
            // (wide plans: more than 48 positions in the chunk form of wunet_tc_wide.cu)
            SplitTable tab;
            lv.sp_chunks = sp_chunk_order(lv, i > n, nullptr, &tab, ci > 32);
            const size_t ns = (size_t)lv.k * lv.Npad * lv.sp_chunks * 64;
            if (!lv.wp_sp && cudaMalloc(&lv.wp_sp, ns * sizeof(__nv_bfloat16)) != cudaSuccess) return tc_fail("cudaMalloc(wp_sp) failed");
            if (lv.sp_chunks > 48) {                        // (more than 3 x 48 positions, or a narrow plan: the planner refuses it)
                if (ci > 32 && lv.sp_chunks <= 3 * 48 && wide::pack_split(blocks[i].w, lv.wp_sp, lv.cout, lv.cin0 + lv.cin1, lv.k, lv.Npad, tab, stream) != cudaSuccess)
                    return tc_fail("pack_tc_split_wide_kernel launch failed");
            } else {
                pack_tc_split_kernel<<<(unsigned)((ns + 255) / 256), 256, 0, stream>>>(blocks[i].w, lv.wp_sp, lv.cout, lv.cin0 + lv.cin1, lv.k,
                                                                                      lv.Npad, tab);
                if (cudaGetLastError() != cudaSuccess) return tc_fail("pack_tc_split_kernel launch failed");
            }
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
    const CUresult r = st->encode(m, st->map_type, 3, const_cast<void *>(base), gdim, gstr, box, estr,
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
// wide (channel plans wider than 32): a block of more than 48 positions gets the chunk form instead, which the SP = 2 kernels
// read (chunk_info): map and table list the chunks, each standing for its three positions in the order above.
static int sp_chunk_order(const TcLevel &lv, bool dec, unsigned char *map, SplitTable *tab, bool wide)
{
    unsigned char one[256];                 // chunks of the block: at most 2 n + 2
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
    if (3 * k > 48) {
        // more positions than chunk_map holds: the chunk form (wide plans), or a count the planner refuses
        if (wide && k <= 48) {
            for (int c = 0; c < k; ++c) {
                const bool up = dec && (one[c] & 0x80);
                const int idx = one[c] & 0x1f;
                if (map) map[c] = one[c];
                if (tab) {
                    const int seg = (up || !dec) ? lv.cin0 : lv.cin1;
                    tab->base[c] = (short)(((up || !dec) ? 0 : lv.cin0) + 64 * idx);
                    tab->width[c] = (unsigned char)std::min(64, seg - 64 * idx);
                    tab->wlo[c] = 0;
                }
            }
        }
        if (tab) tab->n = 3 * k;
        return k <= 48 ? 3 * k : 3 * 48 + 1;
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
// wide: the plan's channels_interval is above 32 (split precision may then take the chunk form, p.split = 2).
static int plan_block(const TcLevel &lv, int i, int n, int B, int T, int num_sms, const std::string &ovr, TcPlanLevel &P, bool sp = false,
                      int hd_mt = 0, bool pair = false, bool group8 = false, bool wide = false)
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
            p.nchunks = sp_chunk_order(lv, dec, p.chunk_map, nullptr, wide);
            p.split = (wide && p.nchunks > 48) ? 2 : 1;  // 2: chunk_map lists chunks (SP = 2 kernels)
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
        if (p.nchunks > (p.split == 2 ? 3 * 48 : 48)) return tc_fail("too many K chunks");
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
    if (last_block && lv.cout > 64) return tc_fail("fused head needs channels_interval <= 64");
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
    const bool sp = mode == 1;
    const bool f16 = mode == 2;                          // the bf16 plan on fp16 data and weights
    st->map_type = f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    const uint64_t cm = sp ? 2 : 1;                      // stored channels per logical channel ([hi | lo] halves)
    char *base = static_cast<char *>(ws);
    auto lvl = [&](int i) { return reinterpret_cast<__nv_bfloat16 *>(base + pl.off[i]); };
    pl.even_copy = false;
    pl.enc0_tc = false;
    if (mode == 0 && st->enc0_ok && T % 8 == 0 && T / 8 >= 128) {
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
            void *&wx = f16 ? lw.wx16 : lw.wx;
            int &wx_L = f16 ? lw.wx16_L : lw.wx_L;
            size_t &wx_elems = f16 ? lw.wx16_elems : lw.wx_elems;
            if (wx_L != g.L) {                                 // (re)build the Toeplitz expansion for this frame length
                if (wx_elems < need) {
                    cudaFree(wx); wx = nullptr; wx_elems = 0;
                    if (cudaMalloc(&wx, need * sizeof(__nv_bfloat16)) != cudaSuccess) return tc_fail("cudaMalloc(expanded weights) failed");
                    wx_elems = need;
                }
                const float up = (dec && g.L > 1) ? (float)(g.L / 2 - 1) / (float)(g.L - 1) : 0.f;
                if (f16) {
                    if (f16::expand_gemm_weights(lw.w_f32, wx, need, lv.cout, lv.cin0, lv.cin1, lv.k, g.L, dec ? 1 : 0, g.npos[0], g.cpp[0],
                                                 g.npos[1], g.cpp[1], up, stream) != cudaSuccess)
                        return tc_fail("expand_gemm_weights_kernel (fp16) launch failed");
                } else {
                    expand_gemm_weights_kernel<<<(unsigned)((need + 255) / 256), 256, 0, stream>>>(lw.w_f32, static_cast<__nv_bfloat16 *>(wx), lv.cout, lv.cin0, lv.cin1, lv.k, g.L,
                                                                                                   dec ? 1 : 0, g.npos[0], g.cpp[0], g.npos[1], g.cpp[1], up);
                    if (cudaGetLastError() != cudaSuccess) return tc_fail("expand_gemm_weights_kernel launch failed");
                }
                wx_L = g.L;
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
            if (make_map(st, &P.tmW, wx, (uint64_t)ktot, (uint64_t)g.N, 1, (uint64_t)ktot * 2, (uint64_t)g.N * ktot * 2, 64, (uint32_t)g.Nh, 1))
                return -1;
            continue;
        }
        if (plan_block(lv, i, n, B, T, st->num_sms, st->plan_ovr, P, sp, 0, pair, false, st->ci > 32)) return -1;
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
        if (make_map(st, &P.tmW, sp ? lv.wp_sp : (f16 ? lv.wp16 : lv.wp), ktot, lv.Npad, lv.k, ktot * 2, (uint64_t)lv.Npad * ktot * 2, 64,
                     (uint32_t)p.Nh, (uint32_t)p.tg))
            return -1;
        P.m2 = false;
        if (st->m2 && m2::selected(p, lv.k, dec, P.small, P.pair, st->num_sms)) {
            // 256-row units: the same operands and maps, weight stages of m2p.tg taps
            m2::geometry(p, lv.k, P.m2p);
            if (make_map(st, &P.tmW2, f16 ? lv.wp16 : lv.wp, ktot, lv.Npad, lv.k, ktot * 2, (uint64_t)lv.Npad * ktot * 2, 64, (uint32_t)p.Nh,
                         (uint32_t)P.m2p.tg))
                return -1;
            P.m2_smem = smem_total(P.m2p);
            P.m2 = true;
        }
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
            if (pl.lv[i].m2) {
                const TcParams &q = pl.lv[i].m2p;
                fprintf(stderr, "[wunet tc]        256-row units=%d na=%d nb=%d tg=%d smem=%zu grid=%d\n", q.tile_end, q.na, q.nb, q.tg,
                        pl.lv[i].m2_smem, std::min(q.tile_end, st->num_sms));
            }
        }
    }
    st->plan_ws = ws; st->plan_B = B; st->plan_T = T; st->plan_x = x; st->plan_y = y; st->plan_mode = mode;
    return 0;
}

// the plan build_plan makes for `block` (host-only, see tc_debug_plan); ks receives the block's tap count
static int debug_plan_level(int n, int ci, const TcBlockSrc *blocks, int nblocks, int B, int T, int block, int num_sms, int mode,
                            TcPlanLevel &P, int &ks)
{
    const char *e0 = getenv("WUNET_TC_ENC0");
    const bool g8 = mode == 0 && block == 0 && e0 && e0[0] == '1';    // block 0 has a tensor-core plan only in its group-of-8 form (bf16)
    if (nblocks != 2 * n + 1 || (block < 1 && !g8) || block >= nblocks) return tc_fail("block %d out of range (1..%d)", block, 2 * n);
    if (ci % 8 != 0 || ci > 64) return tc_fail("bf16 tensor-core path needs channels_interval %% 8 == 0 and <= 64 (got %d)", ci);
    ks = blocks[block].k;
    if (g8) {
        if (blocks[0].k != 15 || blocks[0].cin != 1 || 8 * blocks[0].cout > 256 || T % 8 != 0 || T / 8 < 128) return tc_fail("block 0 has no group-of-8 plan for this shape");
        TcLevel pv;
        pv.cin0 = 8; pv.cin1 = 0; pv.cout = 8 * blocks[0].cout; pv.k = 3; pv.Npad = round_up(pv.cout, 16); pv.Ktot = 64;
        const char *ovr = getenv("WUNET_TC_OVR");
        ks = pv.k;
        return plan_block(pv, 0, n, B, T, num_sms, ovr ? ovr : "", P, false, 0, false, true);
    }
    std::vector<TcLevel> levels(nblocks);
    const char *mge = getenv("WUNET_TC_MERGE");
    derive_levels(levels, blocks, nblocks, n, !(mge && mge[0] == '0') && ci <= 32);
    const char *ovr = getenv("WUNET_TC_OVR");
    const std::string ovr_s = ovr ? ovr : "";
    const char *ge = getenv("WUNET_TC_GEMM");
    bool planned = false;
    if (mode == 1) {
        // split precision (fp32_tc): every block on conv_tc_kernel in split form, no row-pair form, no dense GEMM (build_plan)
        if (plan_block(levels[block], block, n, B, T, num_sms, ovr_s, P, true, 0, false, false, ci > 32)) return -1;
        planned = true;
    } else {
        // bf16 and fp16: row-pair mode of block 1 (WUNET_TC_PAIR bit 0), planned like build_plan does
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
                ks = pv.k;
                planned = true;
            }
        }
    }
    if (!planned && !(!(ge && ge[0] == '0') && parse_override(ovr_s, block).any == false &&
                      plan_block_gemm(levels[block], block, n, B, T, num_sms, P)) &&
        plan_block(levels[block], block, n, B, T, num_sms, ovr_s, P, false, 0))
        return -1;
    return 0;
}

int tc_debug_plan(int n, int ci, const TcBlockSrc *blocks, int nblocks, int B, int T, int block, int num_sms, int *f, int cap, int mode)
{
    if (cap < 32 || !f) return tc_fail("need room for 32 fields");
    TcPlanLevel P{};
    int ks = 0;
    if (debug_plan_level(n, ci, blocks, nblocks, B, T, block, num_sms, mode, P, ks)) return -1;
    const TcParams &p = P.p;
    const int v[32] = {p.L, p.Cin0, p.Cin1, p.Cout, p.Npad, p.Nh, p.nsplit, p.Nstride, p.MT, p.nacc, p.packed, p.FR, p.S, p.m_tiles,
                       p.nchunks, p.resident, p.bulk_store, p.na, p.nb, p.tg, p.ngroups, (int)p.a_stage_bytes, (int)p.b_stage_bytes,
                       p.a_tx_bytes, p.rows_used, (int)p.tmem_cols, (int)P.smem, P.threads, P.per_sm, (int)P.grid.x, P.kind == 2 ? 2 : (int)P.small,
                       p.tiles_per_frame};
    for (int k = 0; k < 32; ++k) f[k] = v[k];
    return 0;
}

int tc_debug_plan_m2(int n, int ci, const TcBlockSrc *blocks, int nblocks, int B, int T, int block, int num_sms, int *f, int cap, int mode)
{
    if (cap < 8 || !f) return tc_fail("need room for 8 fields");
    TcPlanLevel P{};
    int ks = 0;
    if (debug_plan_level(n, ci, blocks, nblocks, B, T, block, num_sms, mode, P, ks)) return -1;
    for (int k = 0; k < 8; ++k) f[k] = 0;
    P.p.head = block == 2 * n ? 1 : 0;                   // as build_plan sets it: the last block carries the fused head
    const char *me = getenv("WUNET_TC_M2");
    if (P.is_gemm || (me && me[0] == '0') || !m2::selected(P.p, ks, P.upcat, P.small, P.pair, num_sms)) return 0;
    TcParams q;
    m2::geometry(P.p, ks, q);
    const int v[8] = {1, q.na, q.nb, q.tg, q.ngroups, (int)smem_total(q), std::min(q.tile_end, num_sms), q.tile_end};
    for (int k = 0; k < 8; ++k) f[k] = v[k];
    return 0;
}

// fp16 weight packings of the blocks (and of the row-pair block), from the library-owned fp32 copies: made by the first fp16
// forward after tc_set_weights, so that a context that never runs fp16 allocates and packs nothing for it
static int pack_f16(TcState *st, cudaStream_t stream)
{
    const int n = st->n;
    for (int i = 1; i < 2 * n + 1; ++i) {
        TcLevel &lv = st->levels[i];
        const size_t nel = (size_t)lv.k * lv.Npad * lv.Ktot;
        if (!lv.wp16 && cudaMalloc(&lv.wp16, nel * sizeof(__half)) != cudaSuccess) return tc_fail("cudaMalloc(fp16 weights) failed");
        if (f16::pack(lv.w_f32, lv.scale, lv.shift, lv.wp16, lv.ss, lv.cout, lv.cin0, lv.cin1, lv.k, lv.Npad, lv.Ktot, stream) != cudaSuccess)
            return tc_fail("pack_tc_kernel (fp16) launch failed");
        if (lv.mg_s && f16::pack_merged(lv.w_f32, lv.wp16, lv.cout, lv.cin0, lv.cin1, lv.k, lv.Npad, lv.Ktot, lv.mg_s, lv.mg_u, stream) != cudaSuccess)
            return tc_fail("pack_tc_merged_kernel (fp16) launch failed");
        lv.wx16_L = 0;                                     // expansions are rebuilt with the next plan
    }
    if (st->pair_ok[0]) {
        TcLevel &pv = st->pair_lv[0];
        const size_t nel = (size_t)pv.k * pv.Npad * pv.Ktot;
        if (!pv.wp16 && cudaMalloc(&pv.wp16, nel * sizeof(__half)) != cudaSuccess) return tc_fail("cudaMalloc(fp16 row-pair weights) failed");
        if (f16::pack(st->pair_w[0], st->pair_scale[0], st->pair_shift[0], pv.wp16, pv.ss, pv.cout, pv.cin0, pv.cin1, pv.k, pv.Npad,
                      pv.Ktot, stream) != cudaSuccess)
            return tc_fail("pack_tc_kernel (fp16 row-pair) launch failed");
    }
    st->f16_packed = true;
    return 0;
}

static int tc_prepare(TcState *st, const float *x, float *y, int B, int T, void *ws, int mode, cudaStream_t stream)
{
    if (!st) return tc_fail("tensor-core state missing");
    const int ci = st->ci;
    if (ci % 8 != 0 || ci > 64) return tc_fail("bf16 tensor-core path needs channels_interval %% 8 == 0 and <= 64 (got %d)", ci);
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
        f16::set_smem_attributes();
        wide::set_smem_attributes();
        pp::set_smem_attributes();
        m2::set_smem_attributes();
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
    if (mode == 2 && !st->f16_packed && pack_f16(st, stream)) return -1;
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

static int launch_block(TcState *st, int i, int t0, int t1, cudaStream_t stream, const void *x = nullptr, void *y = nullptr,
                        int io = IO_F32, void *out = nullptr);

// enc0 over frames [f0, f0 + nf) of x (IoType io samples: the 16-bit forms are those of wunet_tc_io.cuh); *launches receives the
// number of kernels enqueued
static int launch_enc0(TcState *st, const void *x_io, int f0, int nf, int T, void *ws, cudaStream_t stream, int *launches, int io)
{
    if (launches) *launches = 1;
    const void *xf = static_cast<const char *>(x_io) + (size_t)f0 * T * io_bytes(io);     // the frames' first sample
    const float *x = static_cast<const float *>(xf);                                      // io == IO_F32
    if (st->plan.enc0_tc) {
        // tensor-core form: bf16 copy of the frames' samples, then block 0 as a 3-tap block over groups of 8 samples
        __nv_bfloat16 *xb = reinterpret_cast<__nv_bfloat16 *>(static_cast<char *>(ws) + st->plan.off[2 * st->n + 2]) + (size_t)f0 * T;
        const long long n4 = (long long)nf * T / 4;
        if (io == IO_F16) io_f16::launch_x_to_bf16(xf, xb, n4, stream);
        else if (io == IO_BF16) io_bf16::launch_x_to_bf16(xf, xb, n4, stream);
        else x_to_bf16_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(x, xb, n4);
        if (cudaGetLastError() != cudaSuccess) return tc_fail("x_to_bf16_kernel launch failed");
        const int tpf = st->plan.lv[0].p.tiles_per_frame * st->plan.lv[0].p.nsplit;    // tiles of one frame, all column splits
        if (launches) *launches = 2;
        return launch_block(st, 0, f0 * tpf, (f0 + nf) * tpf, stream, nullptr, nullptr);
    }
    const TcLevel &lv = st->levels[0];
    const int C = lv.cout;
    const int split = st->plan_mode == 1 ? 1 : 0;
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
    // the persistent form streams float samples (4-byte cp.async): a 16-bit input takes the one-tile form and its grid
    const bool persistent = io == IO_F32 && (st->enc0_v == 2 || (st->enc0_v == 0 && split));
    if (persistent) {
        const int total = nf * ((T + 1023) / 1024);
        cfg.gridDim = dim3((unsigned)std::min(total, st->num_sms * 4), 1, 1);
    }
    if (st->ci > 32)                                    // wide plans: a tile that shrinks with C (no even-row copy: no row-pair form)
        wide::launch_enc0(cfg, st->plan_mode, xf, lv.w_src, lv.scale, lv.shift, out0 + (size_t)f0 * T * RC, nf, T, C, io);
    else if (io == IO_F16)
        io_f16::launch_enc0(cfg, st->plan_mode, xf, lv.w_src, lv.scale, lv.shift, out0 + (size_t)f0 * T * RC, nf, T, C, even);
    else if (io == IO_BF16)
        io_bf16::launch_enc0(cfg, st->plan_mode, xf, lv.w_src, lv.scale, lv.shift, out0 + (size_t)f0 * T * RC, nf, T, C, even);
    else if (st->plan_mode == 2)                        // fp16: the same kernels with fp16 rows (same size as bf16 ones)
        f16::launch_enc0(cfg, persistent, x, lv.w_src, lv.scale, lv.shift, out0 + (size_t)f0 * T * RC, nf, T, C, even);
    else if (persistent)
        cudaLaunchKernelEx(&cfg, enc0_kernel_v2, x, lv.w_src, lv.scale, lv.shift, out0 + (size_t)f0 * T * RC, nf, T, C, split, even);
    else
        cudaLaunchKernelEx(&cfg, enc0_kernel, x, lv.w_src, lv.scale, lv.shift, out0 + (size_t)f0 * T * RC, nf, T, C, split, even);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return tc_fail("enc0 launch failed: %s", cudaGetErrorString(e));
    return 0;
}

// conv block i over the tile range [t0, t1) (t1 < 0: all tiles); out: null, or where the last block (fused with the head, which
// stores no activation by default) also stores its output, in the layout of the other blocks
static int launch_block(TcState *st, int i, int t0, int t1, cudaStream_t stream, const void *x, void *y, int io, void *out)
{
    TcPlanLevel &P = st->plan.lv[i];
    if (P.is_gemm) {
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = P.grid; cfg.blockDim = dim3(P.threads); cfg.dynamicSmemBytes = P.smem; cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = st->pdl ? 1 : 0;
        cfg.attrs = attr; cfg.numAttrs = 1;
        cudaLaunchKernelEx(&cfg, st->plan_mode == 2 ? f16::gemm_kernel() : gemm_tc_kernel, P.tmA, P.tmO, P.tmW, P.gp);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return tc_fail("gemm_tc level %d launch failed: %s", i, cudaGetErrorString(e));
        return 0;
    }
    TcParams p = P.p;
    p.x = static_cast<const float *>(x); p.y = static_cast<float *>(y);   // only the fused head (last block) reads x / writes y (IO samples)
    p.pf_late = st->pf_late ? 1 : 0;
    if (out) p.out = out;
    if (t1 >= 0) { p.tile_begin = t0; p.tile_end = t1; }
    const int ntiles = p.tile_end - p.tile_begin;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)std::min(ntiles, st->num_sms * P.per_sm), 1, 1);
    cfg.blockDim = dim3(P.threads); cfg.dynamicSmemBytes = P.smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = st->pdl ? 1 : 0;
    cfg.attrs = attr; cfg.numAttrs = 1;
    if (io != IO_F32 && p.head) {
        // 16-bit network input / output: the last block's forms of wunet_tc_io.cuh (large flavour; not the row-pair form)
        if (P.small || P.pair || !P.upcat || p.split == 2) return tc_fail("the last block's tiling has no 16-bit I/O form (small flavour)");
        const int mode = st->plan_mode == 2 ? 2 : (p.split ? 1 : 0);
        cudaLaunchKernelEx(&cfg, io == IO_F16 ? io_f16::head_kernel(mode, p.mg != 0) : io_bf16::head_kernel(mode, p.mg != 0), P.tmA, P.tmW,
                           P.tmO, p);
    } else if (P.m2 && io == IO_F32 && t1 < 0) {
        // streamed-weight block in 256-row units (bf16 / fp16): each weight stage serves both consumer warpgroups' tiles
        TcParams q = P.m2p;
        q.pf_late = p.pf_late;
        cfg.gridDim = dim3((unsigned)std::min(q.tile_end - q.tile_begin, st->num_sms), 1, 1);
        cfg.blockDim = dim3(32 + 32 * (kEpiWarpsLarge + (P.upcat ? m2::kM2ProducerWarps : 0)));
        cfg.dynamicSmemBytes = P.m2_smem;
        q.out = p.out;
        cudaLaunchKernelEx(&cfg, m2::conv_kernel(st->plan_mode == 2, P.upcat, q.mg != 0), P.tmA, P.tmW2, P.tmO, q);
    } else if (pp::selected(p, P.upcat, P.small, io)) {
        // weight-resident last decoder block: the ping-pong form (bf16 / fp16), one epilogue under the other warpgroup's MMAs
        cudaLaunchKernelEx(&cfg, pp::conv_kernel(st->plan_mode == 2, p.mg != 0), P.tmA, P.tmW, P.tmO, p);
    } else if (st->plan_mode == 2) {
        // fp16: the twins of the bf16 forms below (no split-precision form, no block 0 over groups of 8)
        cudaLaunchKernelEx(&cfg, f16::conv_kernel(P.pair == 1 ? 9 : (P.upcat ? 5 : 15), P.small, P.upcat && p.mg), P.tmA, P.tmW, P.tmO, p);
    } else if (P.pair == 3) {
        // block 0 over groups of 8 samples: a 3-tap encoder block
        if (!P.small) cudaLaunchKernelEx(&cfg, conv_tc_kernel<3, false, kEpiWarpsLarge, 0, 0>, P.tmA, P.tmW, P.tmO, p);
        else cudaLaunchKernelEx(&cfg, conv_tc_kernel<3, false, kEpiWarpsSmall, 0, 0>, P.tmA, P.tmW, P.tmO, p);
    } else if (P.pair == 1) {
        // row-pair mode of the first tensor-core encoder block: a 9-tap block over pairs of positions
        if (!P.small) cudaLaunchKernelEx(&cfg, conv_tc_kernel<9, false, kEpiWarpsLarge, 0, 0>, P.tmA, P.tmW, P.tmO, p);
        else cudaLaunchKernelEx(&cfg, conv_tc_kernel<9, false, kEpiWarpsSmall, 0, 0>, P.tmA, P.tmW, P.tmO, p);
    } else if (p.split == 2) {
        // split precision, more than 48 K-loop positions (wide plans): chunk_map lists chunks
        cudaLaunchKernelEx(&cfg, wide::conv_split_kernel(P.upcat), P.tmA, P.tmW, P.tmO, p);
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

int tc_forward(TcState *st, const void *x, void *y, int B, int T, void *ws, cudaStream_t stream, int *launches,
               cudaEvent_t *ev, int mode, int io, bool store_last)
{
    if (tc_prepare(st, nullptr, nullptr, B, T, ws, mode, stream)) return -1;
    const int n = st->n;
    int nl = 0;
    if (ev) cudaEventRecord(ev[0], stream);
    int l0n = 1;
    if (launch_enc0(st, x, 0, B, T, ws, stream, &l0n, io)) return -1;
    nl += l0n;
    if (ev) cudaEventRecord(ev[1], stream);
    for (int i = 1; i < 2 * n + 1; ++i) {
        void *out = (store_last && i == 2 * n) ? static_cast<char *>(ws) + st->plan.off[i] : nullptr;
        if (launch_block(st, i, 0, -1, stream, x, y, io, out)) return -1;
        ++nl;
        if (ev) cudaEventRecord(ev[i + 1], stream);
    }
    if (ev) cudaEventRecord(ev[2 * n + 2], stream);     // head is fused: zero-length segment
    if (launches) *launches = nl;
    return 0;
}

// Host-buffer pipeline (enhancement.py:64-66 form): the first kernel (enc0) and the last (decoder + fused head) run per
// batch chunk, so the H2D copy of chunk c+1 overlaps enc0 of chunk c and the D2H copy of chunk c overlaps the head of c+1.
int tc_forward_host(TcState *st, const void *x_host, void *y_host, void *x_dev, void *y_dev, int B, int T, void *ws,
                    cudaStream_t stream, int *launches, int mode, int io)
{
    if (tc_prepare(st, nullptr, nullptr, B, T, ws, mode, stream)) return -1;
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
    const size_t chunk = (size_t)bc * T * io_bytes(io);           // bytes of one chunk's samples
    const char *xh = static_cast<const char *>(x_host);
    char *yh = static_cast<char *>(y_host), *xd = static_cast<char *>(x_dev), *yd = static_cast<char *>(y_dev);
    int nl = 0;
    // the compute stream may still own x_dev/y_dev from an earlier call: order the copies after it
    cudaEventRecord(st->ev_out[7], stream);
    cudaStreamWaitEvent(st->copy_in, st->ev_out[7], 0);
    for (int c = 0; c < nc; ++c) {
        cudaMemcpyAsync(xd + c * chunk, xh + c * chunk, chunk, cudaMemcpyHostToDevice, st->copy_in);
        cudaEventRecord(st->ev_in[c], st->copy_in);
        cudaStreamWaitEvent(stream, st->ev_in[c], 0);
        int l0n = 1;
        if (launch_enc0(st, x_dev, c * bc, bc, T, ws, stream, &l0n, io)) return -1;
        nl += l0n;
    }
    for (int i = 1; i < 2 * n; ++i) {
        if (launch_block(st, i, 0, -1, stream)) return -1;
        ++nl;
    }
    const int tiles_per_chunk = (pl.m_tiles * pl.nsplit) / nc;      // non-packed: m_tiles = B * tiles_per_frame
    for (int c = 0; c < nc; ++c) {
        if (nc == 1) { if (launch_block(st, 2 * n, 0, -1, stream, x_dev, y_dev, io)) return -1; }
        else if (launch_block(st, 2 * n, c * tiles_per_chunk, (c + 1) * tiles_per_chunk, stream, x_dev, y_dev, io)) return -1;
        ++nl;
        cudaEventRecord(st->ev_out[c], stream);
        cudaStreamWaitEvent(st->copy_out, st->ev_out[c], 0);
        cudaMemcpyAsync(yh + c * chunk, yd + c * chunk, chunk, cudaMemcpyDeviceToHost, st->copy_out);
    }
    if (cudaStreamSynchronize(st->copy_out) != cudaSuccess) return tc_fail("host pipeline failed: %s", cudaGetErrorString(cudaGetLastError()));
    if (launches) *launches = nl;
    return 0;
}

int tc_read_level(TcState *st, int block, const void *ws, int B, int T, float *out_ncl, cudaStream_t stream, int mode)
{
    if (!st) return tc_fail("tensor-core state missing");
    if (block == 2 * st->n && !st->store_last)
        return tc_fail("the last decoder block is fused with the head and not materialised (set WUNET_TC_STORE_LAST=1)");
    return tc_export_level(st, block, ws, B, T, out_ncl, IO_F32, stream, mode);
}

int tc_export_level(TcState *st, int block, const void *ws, int B, int T, void *out_ncl, int io, cudaStream_t stream, int mode)
{
    if (!st) return tc_fail("tensor-core state missing");
    const int n = st->n;
    std::vector<size_t> off;
    size_t total;
    tc_layout(n, st->ci, B, T, off, total, mode);
    const int L = (block <= n) ? (T >> block) : (T >> (2 * n - block));
    const int C = st->levels[block].cout;
    const long long nel = (long long)B * C * L;
    const __nv_bfloat16 *src = reinterpret_cast<const __nv_bfloat16 *>(static_cast<const char *>(ws) + off[block]);
    if (io != IO_F32)      // LevelKind == mode
        return launch_level_export_io(src, mode, out_ncl, io, B, L, C, stream) > 0 ? 0 : tc_fail("level export launch failed");
    float *dst = static_cast<float *>(out_ncl);
    if (mode == 2) return f16::nlc_to_ncl(src, dst, B, L, C, stream) == cudaSuccess ? 0 : tc_fail("read_level launch failed");
    if (mode == 1) nlc_split_to_ncl_f32_kernel<<<(unsigned)((nel + 255) / 256), 256, 0, stream>>>(src, dst, B, L, C);
    else nlc_bf16_to_ncl_f32_kernel<<<(unsigned)((nel + 255) / 256), 256, 0, stream>>>(src, dst, B, L, C);
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
    for (auto &lv : st->levels) { cudaFree(lv.wp); cudaFree(lv.ss); cudaFree(lv.w_own); cudaFree(lv.wp_sp); cudaFree(lv.w_f32); cudaFree(lv.wx); cudaFree(lv.wp16); cudaFree(lv.wx16); }
    cudaFree(st->g8_lv.wp); cudaFree(st->g8_lv.ss); cudaFree(st->g8_w); cudaFree(st->g8_scale); cudaFree(st->g8_shift);
    for (int s = 0; s < 2; ++s) { cudaFree(st->pair_lv[s].wp); cudaFree(st->pair_lv[s].wp16); cudaFree(st->pair_lv[s].ss); cudaFree(st->pair_w[s]); cudaFree(st->pair_scale[s]); cudaFree(st->pair_shift[s]); }
    delete st;
}

}  // namespace wunet
