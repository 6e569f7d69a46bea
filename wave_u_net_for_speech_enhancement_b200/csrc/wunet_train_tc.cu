// wunet_train_tc.cu — tensor-core convolutions of the training step, bf16 and tf32 (Model(train_precision="bf16" / "tf32"),
// DESIGN.md §5.4): the instances of the kernels in wunet_train_tc_kernels.cuh at those two operand types, the launch geometry
// of the weight gradient, and the entry points wunet_train.cu calls at every tensor-core precision (the fp16 instances live in
// wunet_train_tc_f16.cu).
#include "wunet_train_tc_kernels.cuh"

#include <algorithm>

namespace wunet {

// CTA = 64 co x 5 taps x 64 ci; the (frame, 64-position chunk) items are split over gridDim.z
WgradGrid wgrad_grid_tc(int B, int L, int Cin, int Cout, int ksize)
{
    const int ntg = ksize / kTapGroup, nco = (Cout + 63) / 64, nci = (Cin + 63) / 64;
    const int items = B * ((L + kWgPos - 1) / kWgPos);
    const int base = nco * ntg * nci;
    const int slices = std::max(1, std::min(items, (2 * 132 + base - 1) / base));           // about two CTAs per SM
    return WgradGrid{dim3((unsigned)(nco * ntg), (unsigned)nci, (unsigned)slices), items, kWgPos};
}

size_t train_tc_packed_bytes(int prec, int cout, int cin, int k)
{
    return prec == TRAIN_TF32 ? packed_bytes<Tf32>(cout, cin, k) : packed_bytes<Bf16>(cout, cin, k);     // fp16: bf16's bytes
}

int train_tc_pack(int prec, const float *w, void *wf, void *wb, int Cout, int Cin, int K, cudaStream_t st)
{
    if (prec == TRAIN_FP16_SCALED) return train_tc_pack_f16(w, wf, wb, Cout, Cin, K, st);
    return prec == TRAIN_TF32 ? pack<Tf32>(w, wf, wb, Cout, Cin, K, st) : pack<Bf16>(w, wf, wb, Cout, Cin, K, st);
}

int launch_train_conv_tc(int prec, const ConvArgs &a, int ksize, int mode, cudaStream_t st)
{
    if (prec == TRAIN_FP16_SCALED) return launch_train_conv_tc_f16(a, ksize, mode, st);
    return prec == TRAIN_TF32 ? launch_conv_op<Tf32>(a, ksize, mode, st) : launch_conv_op<Bf16>(a, ksize, mode, st);
}

int launch_train_wgrad_tc(int prec, const ConvArgs &a, const float *dz, float *dw, int ksize, int mode, cudaStream_t st, bool slices)
{
    if (prec == TRAIN_FP16_SCALED) return launch_train_wgrad_tc_f16(a, dz, dw, ksize, mode, st, slices);
    return prec == TRAIN_TF32 ? launch_wgrad_op<Tf32>(a, dz, dw, ksize, mode, st, slices)
                              : launch_wgrad_op<Bf16>(a, dz, dw, ksize, mode, st, slices);
}

}  // namespace wunet
