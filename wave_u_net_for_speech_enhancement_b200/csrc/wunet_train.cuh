// wunet_train.cuh — interface of the fp32 training step (implemented in wunet_train.cu; SURVEY.md §8f row N1).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>

namespace wunet {

// Parameters of the 2n+1 conv blocks and of the head, in the reference's own layouts, read straight from the torch tensors.
struct TrainParams {
    const float *const *conv_w;   // [2n+1] -> [Cout][Cin][K]
    const float *const *conv_b;   // [2n+1] -> [Cout]
    const float *const *bn_w;     // [2n+1] -> [Cout]   BatchNorm1d.weight
    const float *const *bn_b;     // [2n+1] -> [Cout]   BatchNorm1d.bias
    float *const *bn_mean;        // [2n+1] -> [Cout]   running_mean, UPDATED in place by the forward
    float *const *bn_var;         // [2n+1] -> [Cout]   running_var,  UPDATED in place by the forward
    const float *out_w;           // [1][C+1][1]
    const float *out_b;           // [1]
};
// Gradient buffers, same layouts as the parameters they belong to (fully overwritten).
struct TrainGrads {
    float *const *conv_w, *const *conv_b, *const *bn_w, *const *bn_b;
    float *out_w, *out_b;
};

// Arithmetic of the three convolution-shaped passes. TRAIN_FP32: fp32 FFMA. TRAIN_BF16: bf16 operands (block input, weights,
// dz; round to nearest), fp32 accumulation on the tensor cores (wunet_train_tc.cu); the first block stays fp32. Everything else
// is fp32 at every precision. The workspace of TRAIN_BF16 is the fp32 one plus the bf16 weight packings. TRAIN_TF32: the same
// with tf32 operands (round to nearest, ties away; the same kernels, templated on the operand type), its workspace the fp32
// one plus the tf32 packings. TRAIN_FP16_SCALED: fp16 operands (round to nearest even, overflow to inf), with each block's dz
// scaled by 2^k (dz_scale_exp of its max |dz|, found on the device) for the two passes that read it and their results by 2^-k;
// its workspace is the bf16 one with fp16 packings (the same bytes) plus 2n+1 scale slots (each block's max |dz|).
enum TrainPrec : int { TRAIN_FP32 = 0, TRAIN_BF16 = 1, TRAIN_TF32 = 2, TRAIN_FP16_SCALED = 3 };

// k of a block's dz scaling under TRAIN_FP16_SCALED, from amax = max |dz| over the block: amax 2^k lies in [2^13, 2^14), so the
// scaled dz stays below a quarter of fp16's largest finite value (65504) and keeps 37 binades above its smallest subnormal;
// k = 0 when amax is 0 or not finite (NaN, inf: those propagate unscaled); |k| <= 126, so 2^k and 2^-k are normal fp32 numbers.
__host__ __device__ inline int dz_scale_exp(float amax)
{
    if (!(amax > 0.f && amax <= 3.402823466e38f)) return 0;
    int e;
    frexpf(amax, &e);                                           // amax = m 2^e, m in [0.5, 1): floor(log2 amax) = e - 1
    const int k = 14 - e;
    return k < -126 ? -126 : (k > 126 ? 126 : k);
}
// TRAIN_FROZEN_BN: BatchNorm normalises by the running statistics and never updates them (eval-mode BatchNorm); the forward
// and the backward of one step must agree on it. TRAIN_NO_PARAM_GRADS (backward only): no parameter gradient is computed
// (G may hold null pointers), only the input gradient. TRAIN_DETERMINISTIC: the weight and head gradients combine their
// partial sums in an order fixed by the shapes (slices stored to a scratch region after the workspace layout, then summed in
// index order) instead of with float atomics; the workspace grows by that scratch, and the forward and the backward of one
// step must agree on it.
enum TrainFlags : int { TRAIN_FROZEN_BN = 1, TRAIN_NO_PARAM_GRADS = 2, TRAIN_DETERMINISTIC = 4 };

// BatchNorm statistics synchronised over data-parallel ranks (nn.SyncBatchNorm; wunet_train_set_bn_allreduce): the batch
// statistics and the backward's mean(dy), mean(dy zh) are computed from sums over every rank's frames. `fn` is called on the
// host after the kernels that wrote buf[0 .. count) are enqueued on `stream`, and must leave the element-wise sum over ranks
// there, ordered on `stream`; nonzero = failure. buf holds >= 2 Cout + 1 doubles of the widest block (device memory).
struct BnSync {
    int (*fn)(void *user, double *buf, size_t count, void *stream);
    void *user;
    double *buf;
};

const char *train_error();
size_t train_workspace_bytes(int n_layers, int ci, int B, int T, int prec = TRAIN_FP32, int flags = 0);
// y = model(x) with BatchNorm in training mode (or, with TRAIN_FROZEN_BN, eval mode); keeps every pre-BN output and
// activation in `workspace` for the backward. momentum[2n+1]: each block's running-statistics factor. bn_frozen[2n+1]
// (null = none): nonzero freezes that block's BatchNorm (running statistics, as TRAIN_FROZEN_BN does for all of them).
// sync (batch-statistics blocks only; null = this rank's frames alone): per block, the local sum z and B L, hook, the local
// sum (z - global mean)^2, hook.
int train_forward(int n_layers, int ci, const float *x, float *y, int B, int T, const TrainParams &P, const float *momentum,
                  void *workspace, cudaStream_t stream, int prec = TRAIN_FP32, int flags = 0, const BnSync *sync = nullptr,
                  const unsigned char *bn_frozen = nullptr);
// gradients of every parameter for the upstream gradient dy of the output; `workspace` as left by train_forward.
// part: -1 = the whole backward; 0 = head + decoder blocks (their gradients are complete afterwards: a data-parallel caller
// starts reducing them while part 1 runs); 1 = middle + encoder blocks (must follow part 0 on the same stream).
// dx (optional, [B][1][T], fully overwritten): gradient of the input x; written by part -1 or 1 (block 0 is in part 1).
// sync: must be given iff the forward had it; per batch-statistics block of the part, [sum dy | sum dy zh | B L], hook.
// bn_frozen: as in the forward. A null array or entry in G is a frozen parameter: nothing is computed for it or written.
// early_stop: nothing is issued below the lowest block that needs a gradient (or dx), and that block skips its input
// gradient; dx then also goes to part 0, unwritten, to say that part 1 will ask for it.
// g_act: null, or 2n+1 device pointers (null = none): g_act[i] [B][Cout][L] is added to block i's activation gradient before its
// BatchNorm backward, when block i is processed (its part, at or above the early stop).
int train_backward(int n_layers, int ci, const float *x, const float *y, const float *dy, int B, int T, const TrainParams &P,
                   const TrainGrads &G, void *workspace, cudaStream_t stream, int part = -1, int prec = TRAIN_FP32,
                   float *dx = nullptr, int flags = 0, const BnSync *sync = nullptr, const unsigned char *bn_frozen = nullptr,
                   bool early_stop = false, const float *const *g_act = nullptr);
// One convolution-shaped pass on caller device buffers (test hook): pass 0 = forward conv out[B][Cout][L] = conv(in, w);
// 1 = input gradient out[B][Cin][L] of dz [B][Cout][L] (Conv1d padding, no mode); 2 = weight gradient out[Cout][Cin][K] =
// sum dz * in. `in` is built from src0 / src1 per `mode` as in the forward (ConvArgs). Synchronous.
int train_debug_conv(int pass, int prec, int mode, int ksize, int B, int L, int Cin0, int Cin1, int Cout, const float *src0,
                     const float *src1, const float *w, const float *dz, float *out);
// Host-only: where block `block`'s tensors live in the training workspace and how its weight gradient is launched
// (the fields of wunet_debug_train_layout, include/wunet_b200.h).
constexpr int kTrainLayoutFields = 22;
int train_debug_layout(int n_layers, int ci, int B, int T, int prec, int block, long long *fields, int capacity);

}  // namespace wunet
