// wunet_tc.cuh — interface of the bf16 / wgmma tensor-core path (implemented in wunet_tc.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace wunet {

struct TcState;   // packed bf16 weights, TMA tensor maps, per-shape plans

// One conv block as the tensor-core path sees it: the ORIGINAL fp32 weights [Cout][Cin][K] plus the
// folded eval-BatchNorm scale/shift that the fp32 packer already produced.
struct TcBlockSrc {
    int cin, cout, k;
    const float *w;       // device, [Cout][Cin][K] fp32 (reference layout)
    const float *scale;   // device, [Cout]
    const float *shift;   // device, [Cout]
};

const char *tc_error();
int tc_set_weights(TcState **st, int n_layers, int ci, const TcBlockSrc *blocks, int nblocks, const float *out_w,
                   const float *out_b, cudaStream_t stream);
// mode: 0 = bf16 activations; 1 = split precision (fp32_tc): activations as [hi | lo] bf16 halves, three MMAs per product
size_t tc_workspace_bytes(int n_layers, int ci, int B, int T, int mode = 0);
// events: null, or 2n+3 events: [0] before the first kernel, [i+1] after block i, [2n+2] after the head
int tc_forward(TcState *st, const float *x, float *y, int B, int T, void *ws, cudaStream_t stream, int *launches,
               cudaEvent_t *events, int mode = 0);
// host-buffer form: x_host/y_host (pinned for full rate), x_dev/y_dev = device staging buffers of B*T floats
int tc_forward_host(TcState *st, const float *x_host, float *y_host, float *x_dev, float *y_dev, int B, int T, void *ws,
                    cudaStream_t stream, int *launches, int mode = 0);
int tc_read_level(TcState *st, int block, const void *ws, int B, int T, float *out_ncl, cudaStream_t stream, int mode = 0);
void tc_destroy(TcState *st);
// host-only: the tiling build_plan would choose for `block` (32 ints, see wunet_debug_plan in include/wunet_b200.h)
int tc_debug_plan(int n_layers, int ci, const TcBlockSrc *blocks, int nblocks, int B, int T, int block, int num_sms, int *fields,
                  int capacity);

// host-only: row-pair expansion of [Cout][C0+C1][K] weights to [2 Cout][2 (C0+C1)][K'] (tests of the WUNET_TC_PAIR packing)
int tc_debug_pair_weights(const float *w, int Cout, int C0, int C1, int K, int dec, float *out);

}  // namespace wunet
