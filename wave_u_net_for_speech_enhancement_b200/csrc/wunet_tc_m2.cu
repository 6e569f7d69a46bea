// wunet_tc_m2.cu — the 256-row form of the blocks that stream their weights from L2 (wunet_tc_m2.cuh) for bf16 and fp16, for
// sm_90a; the host launches it where m2::selected holds. A unit of its own so that the kernels of wunet_tc.cu, wunet_tc_f16.cu and
// wunet_tc_pp.cu keep their machine code; the host code of wunet_tc.cu reaches these kernels through the functions below.
#include "wunet_common.cuh"
#include "wunet_wgmma.cuh"
#include "wunet_tc_common.cuh"

#include <algorithm>

#define WUNET_TC_CONV_ONLY 1

namespace wunet {
namespace m2 {

namespace bf16 {
using TcElem = TcBf16;
#include "wunet_tc_kernels.cuh"
#include "wunet_tc_m2.cuh"
}  // namespace bf16

namespace f16 {
#define WUNET_TC_FP16 1
using TcElem = TcF16;
#include "wunet_tc_kernels.cuh"
#include "wunet_tc_m2.cuh"
#undef WUNET_TC_FP16
}  // namespace f16

ConvKernel conv_kernel(bool fp16, bool upcat, bool mg)
{
    if (fp16) {
        if (!upcat) return f16::conv_tc_m2_kernel<15, false, 0, kM2AccCols>;
        return mg ? f16::conv_tc_m2_kernel<5, true, 1, kM2AccCols> : f16::conv_tc_m2_kernel<5, true, 0, kM2AccCols>;
    }
    if (!upcat) return bf16::conv_tc_m2_kernel<15, false, 0, kM2AccCols>;
    return mg ? bf16::conv_tc_m2_kernel<5, true, 1, kM2AccCols> : bf16::conv_tc_m2_kernel<5, true, 0, kM2AccCols>;
}

void set_smem_attributes()
{
    for (bool fp16 : {false, true})
        for (int form = 0; form < 3; ++form)
            cudaFuncSetAttribute(conv_kernel(fp16, form > 0, form == 2), cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
}

int units(const TcParams &p)
{
    return p.packed || p.tiles_per_frame % 2 != 0 ? 0 : p.B * (p.tiles_per_frame / 2) * p.nsplit;
}

bool geometry(const TcParams &p, int ks, TcParams &q)
{
    q = p;
    // operand stage: the unit's 256 + ks - 1 rows in two boxes of the plan's R1 >= 128 + ks - 1 rows (the plan's tensor map)
    q.nops = 2;
    q.a_tx_bytes = 2 * p.R1 * 128;
    q.a_stage_bytes = (uint32_t)round_up(q.a_tx_bytes, 1024);
    q.rows_used = 256 + ks - 1;
    // the plan's operand ring depth; weight stages: the fewest per chunk that leave a ring of two next to it, with their taps
    // spread evenly (no zero-filled taps where avoidable), then as many stages as fit (plan_block's ring budget)
    const int budget = kSmemLimit - 2048 - p.Npad * 8 - 512;
    const int room = budget - q.na * (int)q.a_stage_bytes;
    for (int ngroups = 1; ngroups <= ks; ++ngroups) {
        const int tg = (ks + ngroups - 1) / ngroups;
        const int stage = round_up(p.Nh * 128 * tg, 1024);
        if (room < 2 * stage) continue;
        q.tg = tg;
        q.ngroups = (ks + tg - 1) / tg;
        q.b_stage_bytes = (uint32_t)stage;
        q.nb = std::min(kMaxBStages, room / stage);
        q.tile_begin = 0;
        q.tile_end = units(p);
        return smem_total(q) <= (size_t)kSmemLimit;
    }
    return false;
}

bool selected(const TcParams &p, int ks, bool upcat, bool small, int pair, int num_sms)
{
    TcParams q;
    return p.split == 0 && !p.head && p.hd == 0 && pair == 0 && !small && ks == (upcat ? 5 : 15) && p.MT == 1 && !p.resident &&
           !p.packed && p.tiles_per_frame % 2 == 0 && p.Nh <= kM2AccCols && units(p) >= num_sms &&
           geometry(p, ks, q);
}

}  // namespace m2
}  // namespace wunet
