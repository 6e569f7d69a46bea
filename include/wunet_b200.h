/*
 * wunet_b200.h — C ABI of the H100-native Wave-U-Net forward path.
 *
 * This is the drop-in boundary for ONE hot path of haoxiangsnr/Wave-U-Net-for-Speech-Enhancement:
 * `Model.forward` (reference model/unet_basic.py:77-100) together with the parameter tree that
 * `Model.__init__` (model/unet_basic.py:33-75) defines.  Every entry point takes plain pointers and
 * sizes; there are no torch types here.  The Python shim
 * (wave_u_net_for_speech_enhancement_b200/unet_basic.py) binds these with ctypes and exposes the
 * reference's `Model(n_layers, channels_interval)` nn.Module surface on top.
 *
 * Conventions
 *   - every function returns 0 on success, a negative WUNET_E* code on failure; the message is
 *     available from wunet_last_error() (thread-local), which the shim turns into RuntimeError
 *     (the reference's error convention is Python exceptions, SURVEY §8b).
 *   - "dev" pointers are device pointers on the context's device; "host" pointers are host memory.
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream). Nothing here
 *     synchronises the device except wunet_forward_host().
 *   - there is NO CPU fallback: without a CUDA device wunet_create() fails.
 */
#ifndef WUNET_B200_H
#define WUNET_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WUNET_OK 0
#define WUNET_EINVAL (-1)   /* bad argument (shape, null pointer, T not a multiple of 2^n_layers ...) */
#define WUNET_ECUDA (-2)    /* a CUDA runtime / driver call failed */
#define WUNET_ESTATE (-3)   /* call order (forward before set_weights ...) */
#define WUNET_ENOMEM (-4)   /* workspace too small / allocation failed */

/* arithmetic of the convolution path */
#define WUNET_PREC_FP32 0   /* fp32 operands, fp32 FFMA accumulate: parity <= 1e-4 vs reference (config 2) */
#define WUNET_PREC_BF16 1   /* bf16 operands/activations, fp32 accumulate on wgmma tensor cores (config 3) */
#define WUNET_PREC_FP32_TC 2 /* fp32-grade on the tensor cores: activations and weights split into bf16 high + low parts, three wgmma
                               MMAs per product (hi*hi + lo*hi + hi*lo, fp32 accumulate): <= 1e-4 vs the reference like WUNET_PREC_FP32 */
#define WUNET_PREC_TF32 3   /* training step only: tf32 operands (round to nearest), fp32 accumulate on wgmma tensor cores; the
                               inference entry points reject it (WUNET_EINVAL) */
#define WUNET_PREC_FP16 4   /* inference only: the bf16 contract with fp16 in place of bf16 — fp16 activations (channels-last) and
                               weights (round to nearest even), fp32 accumulate on wgmma tensor cores, BatchNorm + LeakyReLU in fp32.
                               Every fp16 store saturates: an activation beyond +-65504 is stored as +-65504, never as inf. The one
                               place that can still overflow is the decoder's upsampling on levels of >= 128 samples, which
                               interpolates in packed fp16 and forms b - a of two adjacent values: more than 65504 apart -> inf.
                               Same workspace and tiling plan as WUNET_PREC_BF16; block 0 stays on the CUDA cores (WUNET_TC_ENC0
                               does not apply). The training entry points reject it (WUNET_EINVAL). */
#define WUNET_PREC_FP16_SCALED 5 /* training step only: fp16 operands (round to nearest even, no saturation) with per-block
                               power-of-two scaling of dz, fp32 accumulate on wgmma tensor cores (see the training entry points);
                               the inference entry points reject it (WUNET_EINVAL) */

/* element type of the network input x and output y (the _io entry points) */
#define WUNET_IO_F32 0      /* float32 samples (what every entry point without _io takes) */
#define WUNET_IO_F16 1      /* IEEE binary16 samples: widened to fp32 on load (exact); each output rounded once from the fp32
                               result, to nearest even. Everything in between is the fp32-I/O computation at `precision`, so
                               y = (fp16) forward(fp32(x)) bit for bit. */
#define WUNET_IO_BF16 2     /* bfloat16 samples, the same contract */

typedef struct wunet_ctx wunet_ctx;

/* Version / build info string (static storage). */
const char *wunet_version(void);

/* Last error message of the calling thread (static thread-local storage, never NULL). */
const char *wunet_last_error(void);

/*
 * Replaces: Model.__init__(n_layers=12, channels_interval=24)   model/unet_basic.py:33-75
 * Builds the channel plan (encoder_in/out :38-39, middle :52-57, decoder_in/out :59-62, out :72-75)
 * for `device` (CUDA ordinal). No weights yet.
 */
int wunet_create(int n_layers, int channels_interval, int device, wunet_ctx **out);
void wunet_destroy(wunet_ctx *ctx);

/* Number of conv+BN+LeakyReLU blocks = 2*n_layers+1 (encoder[0..n-1], middle, decoder[0..n-1]). */
int wunet_num_blocks(const wunet_ctx *ctx);
/* Channel plan of block i (forward order): Cin, Cout, kernel size.  (model/unet_basic.py:38-39,59-62) */
int wunet_block_shape(const wunet_ctx *ctx, int block, int *cin, int *cout, int *ksize);

/*
 * Replaces: the parameter reads that nn.Conv1d / nn.BatchNorm1d do inside Model.forward
 * (model/unet_basic.py:10-12, :23-25, :53-55, :73) and load_state_dict (enhancement.py:41,
 * trainer/base_trainer.py:77-79).
 * All arrays have wunet_num_blocks() entries of DEVICE pointers to contiguous fp32 tensors in the
 * reference's shapes: conv_w[i] = [Cout,Cin,K], conv_b/bn_* [Cout]; out_w = [1,ci+1,1], out_b = [1].
 * The library packs them (layout change, eval-BatchNorm folded to scale/shift with eps=1e-5, bf16
 * copies) into its own device buffers on `stream`; the caller's tensors are only read during the
 * call's stream work and may change afterwards (call again to refresh — the shim does so whenever a
 * parameter's version/data_ptr changes, e.g. after optimizer.step(), load_state_dict, .cpu()/.to()).
 */
int wunet_set_weights(wunet_ctx *ctx, const float *const *conv_w, const float *const *conv_b,
                      const float *const *bn_weight, const float *const *bn_bias,
                      const float *const *bn_running_mean, const float *const *bn_running_var,
                      const float *out_w, const float *out_b, void *stream);

/* Bytes of device scratch wunet_forward() needs for a [B,1,T] batch at `precision`. 0 on error. */
size_t wunet_workspace_bytes(const wunet_ctx *ctx, int B, int T, int precision);

/*
 * Replaces: Model.forward(input)   model/unet_basic.py:77-100   (eval-mode BatchNorm)
 *   x_dev [B,1,T] fp32 contiguous  ->  y_dev [B,1,T] fp32 contiguous, values in (-1,1) (16-bit: wunet_forward_io).
 * T must be a multiple of 2^n_layers (the reference raises from torch.cat at :95 otherwise)
 * -> WUNET_EINVAL.  Enqueues kernels on `stream` and returns; `workspace` must stay alive until
 * they finish.  Call sites this serves: trainer/trainer.py:75, enhancement.py:66.
 * The tensor-core precisions (WUNET_PREC_BF16, _FP16, _FP32_TC) need channels_interval % 8 == 0 and <= 64; widths 40 .. 64 run
 * without the forms gated on narrow channels (row-pair block 1, merged decoder tails, the group-of-8 block 0), with a block 0 whose
 * tile shrinks with the width. WUNET_PREC_FP32 takes any channel plan.
 */
int wunet_forward(wunet_ctx *ctx, const float *x_dev, float *y_dev, int B, int T, int precision,
                  void *workspace, size_t workspace_bytes, void *stream);
/*
 * The same with x_dev / y_dev holding B*T samples of `io_dtype` (WUNET_IO_*): a half model's forward, 16-bit in and out. Only
 * the first kernel's input read and the output write change (the kernels that touch x or y are instantiated per I/O type); the
 * workspace is wunet_workspace_bytes()'s, whatever the I/O type. The parameters stay those of wunet_set_weights (fp32: a
 * caller holding 16-bit parameters widens them, which is exact). wunet_forward() is io_dtype = WUNET_IO_F32.
 */
int wunet_forward_io(wunet_ctx *ctx, const void *x_dev, void *y_dev, int B, int T, int precision, int io_dtype,
                     void *workspace, size_t workspace_bytes, void *stream);

/*
 * wunet_forward_io that also writes the outputs of chosen blocks: what forward hooks on the reference's encoder[i], middle and
 * decoder[j] see (model/unet_basic.py:82-96), for the Python module's hooks on those containers.
 *   export_mask[2n+1] (forward order: encoder 0 .. n-1, middle, decoder 0 .. n-1; NULL or all zero = wunet_forward_io, the same
 *     launches and bits): a nonzero entry i writes block i's full-resolution output to level_out[i] (device, caller-owned) as
 *     [B][Cout][L] of io_dtype. The value is the block output the next block reads, widened exactly to fp32 (fp32_tc: hi + lo of
 *     its split halves) and, for 16-bit I/O, rounded once to io_dtype (nearest even); with WUNET_IO_F32 it equals
 *     wunet_read_level's bit for bit.
 *   The last decoder block is fused with the head and stores no output on the tensor-core precisions; when it is marked, the
 *     same kernel runs with its activation store switched on (its launch and y are unchanged, bit for bit).
 *   One conversion launch per marked block after the forward, on `stream`; wunet_last_launch_count() counts the forward only.
 *   The workspace is wunet_workspace_bytes()'s. A marked block without a buffer -> WUNET_EINVAL before anything is enqueued.
 */
int wunet_forward_export(wunet_ctx *ctx, const void *x_dev, void *y_dev, int B, int T, int precision, int io_dtype,
                         const unsigned char *export_mask, void *const *level_out, void *workspace, size_t workspace_bytes,
                         void *stream);

/*
 * Same operator with HOST buffers (the end-to-end form used by enhancement.py:64-66, which does
 * `model(chunk).detach().cpu()`): copies x_host -> device, runs the forward, copies y back and
 * waits for it.  Uses context-owned, grow-only device buffers and a context-owned stream.
 * x_host/y_host should be pinned for full PCIe rate; pageable memory also works.
 */
int wunet_forward_host(wunet_ctx *ctx, const float *x_host, float *y_host, int B, int T, int precision);
/* x_host / y_host of io_dtype (WUNET_IO_*): the copies move 2 bytes per sample for the 16-bit types */
int wunet_forward_host_io(wunet_ctx *ctx, const void *x_host, void *y_host, int B, int T, int precision, int io_dtype);

/*
 * Streaming form of the same operator for MANY batches — what enhancement.py:49-74 / trainer/trainer.py:58-79 do when they
 * push every 16384-sample chunk of every clip through the model. wunet_stream_submit() enqueues batch k and returns at once:
 * the H2D copy (copy stream, one of two device slots), the kernels (compute stream) and the D2H copy (second copy stream)
 * of consecutive batches overlap. wunet_stream_wait(ticket) blocks until that batch's y_host is complete. At most two
 * batches are in flight: submitting a third waits for the first. Host buffers should be pinned and must stay valid until
 * the ticket has been waited for.
 */
int wunet_stream_submit(wunet_ctx *ctx, const float *x_host, float *y_host, int B, int T, int precision, int *ticket);
/* x_host / y_host of io_dtype (WUNET_IO_*); tickets are shared with wunet_stream_submit() */
int wunet_stream_submit_io(wunet_ctx *ctx, const void *x_host, void *y_host, int B, int T, int precision, int io_dtype,
                           int *ticket);
int wunet_stream_wait(wunet_ctx *ctx, int ticket);

/*
 * Host-side data path around the streaming operator (SURVEY §8f row N4) - pure host code, no CUDA call:
 * wunet_frame_clips_*() does for MANY clips what enhancement.py:57-62 does for one (zero-pad the 1-D clip to a multiple of
 * sample_length, split it into chunks): clip i occupies max(1, ceil(lengths[i] / sample_length)) consecutive rows of
 * frames[total_frames][sample_length], clips follow each other in order, the remaining rows are zero-filled (silent frames
 * that keep the batch size constant). The _i16 form takes 16-bit PCM as stored in a wav file and converts it like the
 * reference's loader does (librosa.load / soundfile: sample / 32768), fused into the same pass.
 * wunet_unframe_clips_f32() is the inverse for the model output: concatenate each clip's chunks and drop the padding
 * (enhancement.py:68-71) into caller-allocated clips_out[i][lengths[i]]. `nthreads` host threads share the rows.
 * frames should be the pinned staging buffer handed to wunet_stream_submit().
 */
int wunet_frame_clips_f32(const float *const *clips, const long long *lengths, int nclips, int sample_length, float *frames,
                          long long total_frames, int nthreads);
int wunet_frame_clips_i16(const int16_t *const *clips, const long long *lengths, int nclips, int sample_length, float *frames,
                          long long total_frames, int nthreads);
int wunet_unframe_clips_f32(const float *frames, float *const *clips_out, const long long *lengths, int nclips, int sample_length,
                            long long total_frames, int nthreads);
/* The two framing forms with frames of io_dtype (WUNET_IO_*), the staging buffer of wunet_stream_submit_io(): each sample is
 * computed in fp32 as above (int16 PCM: sample / 32768) and rounded once to io_dtype (nearest even). */
int wunet_frame_clips_f32_io(const float *const *clips, const long long *lengths, int nclips, int sample_length, void *frames,
                             long long total_frames, int nthreads, int io_dtype);
int wunet_frame_clips_i16_io(const int16_t *const *clips, const long long *lengths, int nclips, int sample_length, void *frames,
                             long long total_frames, int nthreads, int io_dtype);

/*
 * Training-side data path (SURVEY §8f row N4) - pure host code, no CUDA call. Replaces, per item of a batch, what
 * dataset/waveform_dataset.py:56-67 does in a DataLoader worker: librosa.load(path, sr=None) of the mixture and the clean file
 * (= soundfile's float32 conversion: integer PCM scaled by 2^-(bits-1), channels averaged) and the aligned random crop
 * util/utils.py:101-113.
 * wunet_wav_info(): header of a RIFF/WAVE file (PCM 8/16/24/32 bit, IEEE float 32/64 bit; any channel count).
 * wunet_wav_read_f32(): frames [first_frame, first_frame + nframes) as mono float32 (so a crop can be read without decoding the
 *   whole file).
 * wunet_crop_pairs(): for item i copy samples [starts[i], starts[i] + sample_length) of mixture[i] and of clean[i] (both
 *   lengths[i] samples long, float32 or - is_i16 != 0 - 16-bit PCM converted by / 32768) into rows i of
 *   mixture_out / clean_out [nitems][sample_length] (the batch tensors [B,1,T]; pinned for the H2D copy), on `nthreads` host
 *   threads. The random starts stay with the caller (the reference draws them from numpy's global generator,
 *   util/utils.py:109). Errors like the reference's asserts: short clips, starts outside the clip -> WUNET_EINVAL.
 */
int wunet_wav_info(const char *path, int *sample_rate, int *channels, long long *frames, int *bits, int *is_float);
int wunet_wav_read_f32(const char *path, long long first_frame, long long nframes, float *out);
int wunet_crop_pairs(const void *const *mixture, const void *const *clean, const long long *lengths, const long long *starts, int nitems,
                     int sample_length, int is_i16, float *mixture_out, float *clean_out, int nthreads);

/*
 * Test/diagnostic hook: copy the full-resolution output of block `block` from the workspace of the
 * LAST wunet_forward() call (same ctx, same workspace, B, T, precision) to out_dev as fp32
 * [B,Cout,L] (the reference's NCL layout) — what a forward hook on encoder[i] / middle /
 * decoder[j] would see.  Used by the per-level parity tests.
 */
int wunet_read_level(wunet_ctx *ctx, int block, const void *workspace, int B, int T, int precision,
                     float *out_dev, void *stream);

/*
 * Measurement hooks (bench.py's per-level roofline): when enabled, wunet_forward() records a CUDA
 * event on the launch stream before the first kernel and after every block (2n+1 conv blocks, then
 * the 1x1+tanh head when it is a separate launch).  wunet_profile_read() waits for the last event
 * and returns the per-block device time in milliseconds: ms[i] = block i, ms[2n+1] = head (0 when the
 * head is fused into the last decoder block).  *count receives the number of entries written.
 */
int wunet_profile_enable(wunet_ctx *ctx, int enable);
int wunet_profile_read(wunet_ctx *ctx, float *ms, int capacity, int *count);

/* Number of kernel launches the last wunet_forward()/wunet_forward_host() enqueued. */
int wunet_last_launch_count(const wunet_ctx *ctx);

/* ---- training step (SURVEY.md §8f row N1; fp32 CUDA-core kernels; the host mirror's default in .train() mode) -----------------
 * Replaces, together, what autograd records and replays for trainer/trainer.py:35-37 (enhanced = model(mixture) in .train()
 * mode; loss.backward()). Parameters are read in the reference's layouts straight from the caller's tensors.
 * wunet_train_forward: y = model(x) with BatchNorm1d (model/unet_basic.py:12,25,55) using batch statistics; updates the
 *   running_mean / running_var buffers in place (momentum, unbiased variance) as torch does; keeps the activations in `workspace`.
 * wunet_train_backward: gradients of all parameters (same layouts, fully overwritten) for the upstream gradient dy [B][1][T];
 *   `workspace` must be the one the matching forward left behind. */
size_t wunet_train_workspace_bytes(const wunet_ctx *ctx, int B, int T);
int wunet_train_forward(wunet_ctx *ctx, const float *x, float *y, int B, int T, const float *const *conv_w,
                        const float *const *conv_b, const float *const *bn_weight, const float *const *bn_bias,
                        float *const *bn_running_mean, float *const *bn_running_var, const float *out_w, const float *out_b,
                        float momentum, void *workspace, size_t workspace_bytes, void *stream);
int wunet_train_backward(wunet_ctx *ctx, const float *x, const float *y, const float *dy, int B, int T,
                         const float *const *conv_w, const float *const *bn_weight, const float *const *bn_bias, const float *out_w,
                         float *const *g_conv_w, float *const *g_conv_b, float *const *g_bn_weight, float *const *g_bn_bias,
                         float *g_out_w, float *g_out_b, void *workspace, size_t workspace_bytes, void *stream);
/* The same backward in two parts, for data-parallel training (SURVEY.md §8e: one process per GPU replaces the nn.DataParallel
 * of trainer/base_trainer.py:26-27): part 0 = head + decoder blocks — their parameter gradients are final when it has run, so
 * the caller starts the all-reduce of that half of the flat gradient bucket on another stream; part 1 = middle + encoder
 * blocks, enqueued after part 0 on the same stream, overlaps that all-reduce. part -1 = both (= wunet_train_backward). */
int wunet_train_backward_part(wunet_ctx *ctx, const float *x, const float *y, const float *dy, int B, int T,
                              const float *const *conv_w, const float *const *bn_weight, const float *const *bn_bias,
                              const float *out_w, float *const *g_conv_w, float *const *g_conv_b, float *const *g_bn_weight,
                              float *const *g_bn_bias, float *g_out_w, float *g_out_b, void *workspace, size_t workspace_bytes,
                              void *stream, int part);
/* The same three entry points with a training precision (the ones above are these with WUNET_PREC_FP32):
 *   WUNET_PREC_FP32  fp32 FFMA in every pass;
 *   WUNET_PREC_BF16  mixed precision: the operands of the three convolution-shaped passes — block input (after decimation, or
 *                    interpolation + concat, computed in fp32 first), weights and dz — are rounded to bf16 and the products
 *                    accumulated in fp32 on the wgmma tensor cores; z, BatchNorm, the head, the decimate / upsample / concat
 *                    adjoints and all gradients stay fp32 (torch.autocast(bfloat16) semantics for Conv1d, except that z is fp32).
 *                    The first block (Cin = 1) stays fp32. Parameters and gradients are fp32 in the reference layouts.
 *   WUNET_PREC_TF32  the same mixed-precision contract with tf32 operands: each is rounded to 11 significant bits (round to
 *                    nearest, ties away from zero: cvt.rna.tf32.f32) and the products are accumulated in fp32 on wgmma
 *                    (m64nNk8.f32.tf32.tf32). This is the arithmetic of cuDNN's Conv1d with torch.backends.cudnn.allow_tf32
 *                    (PyTorch's default), i.e. of the reference's own training step on an H100. The first block stays fp32.
 *   WUNET_PREC_FP16_SCALED  the same mixed-precision contract with fp16 operands (round to nearest even; beyond +-65504 they
 *                    become +-inf and NaN stays NaN: unlike the inference fp16 stores nothing saturates, so a non-finite
 *                    value reaches the gradients, e.g. a GradScaler's found_inf, instead of being hidden) and per-block scaling
 *                    of dz, which fp16's range could not hold unscaled: for each block j the backward finds amax_j = max |dz_j|
 *                    on the device and k_j with amax_j 2^k_j in [2^13, 2^14) (k_j = 0 when amax_j is 0 or not finite; |k_j| <=
 *                    126); the input and weight gradients use fp16(dz 2^k_j) and their results are multiplied by 2^-k_j.
 *                    Powers of two are exact in fp32, so each pass computes exactly sum fp16(dz 2^k) fp16(x) 2^-k, and the
 *                    gradients of loss 2^m are 2^m times those of loss. The forward operands are not scaled. No host sync: the
 *                    step stays graph-capturable and, with WUNET_TRAIN_DETERMINISTIC, bitwise repeatable (max is
 *                    order-independent). Each data-parallel rank picks its own k_j. The first block stays fp32. The workspace
 *                    is the WUNET_PREC_BF16 one (fp16 packings take the bytes of the bf16 ones) plus 2 n_layers + 1 scale slots.
 *   WUNET_PREC_FP32_TC, WUNET_PREC_FP16 -> WUNET_EINVAL (not training precisions).
 * The backward must use the precision and workspace of its forward. Same call sites as above (trainer/trainer.py:35-37). */
size_t wunet_train_workspace_bytes_prec(const wunet_ctx *ctx, int B, int T, int precision);
int wunet_train_forward_prec(wunet_ctx *ctx, const float *x, float *y, int B, int T, const float *const *conv_w,
                             const float *const *conv_b, const float *const *bn_weight, const float *const *bn_bias,
                             float *const *bn_running_mean, float *const *bn_running_var, const float *out_w, const float *out_b,
                             float momentum, void *workspace, size_t workspace_bytes, void *stream, int precision);
int wunet_train_backward_part_prec(wunet_ctx *ctx, const float *x, const float *y, const float *dy, int B, int T,
                                   const float *const *conv_w, const float *const *bn_weight, const float *const *bn_bias,
                                   const float *out_w, float *const *g_conv_w, float *const *g_conv_b, float *const *g_bn_weight,
                                   float *const *g_bn_bias, float *g_out_w, float *g_out_b, void *workspace, size_t workspace_bytes,
                                   void *stream, int part, int precision);

/* The training step with flags and the input gradient (the _prec entry points above are these with flags = 0, dx = NULL).
 * Serves autograd through the model beyond a plain training step: x.grad for whatever sits upstream of the model (a cascade,
 * a learnable front end, an adversarial perturbation), and eval-mode BatchNorm for fine-tuning with frozen statistics. */
#define WUNET_TRAIN_FROZEN_BN      1  /* BatchNorm uses (and never updates) the running statistics: eval-mode BN */
#define WUNET_TRAIN_NO_PARAM_GRADS 2  /* backward: no parameter gradients (g_* may be NULL), only dx */
#define WUNET_TRAIN_DETERMINISTIC 16  /* bitwise repeatable step: no float atomics; the workspace grows (see below) */
/* wunet_train_forward_ex: with WUNET_TRAIN_FROZEN_BN, BatchNorm normalises by bn_running_mean / bn_running_var, which are only
 *   read (momentum is unused): model/unet_basic.py in .eval() mode, with the activations kept for the backward. The forward
 *   ignores WUNET_TRAIN_NO_PARAM_GRADS. The workspace size is wunet_train_workspace_bytes_prec (frozen mode needs nothing extra).
 *   Batch statistics of one value per channel (B = 1 and T = 2^n_layers: L = 1 at the middle block) -> WUNET_EINVAL, where
 *   torch.nn.BatchNorm1d raises in training mode; with WUNET_TRAIN_FROZEN_BN that shape is accepted.
 * wunet_train_backward_ex: dx [B][1][T] (device, or NULL) is fully overwritten with the gradient of x. It belongs to part 1
 *   (block 0 is there): pass it with part -1 or 1; dx with part 0 is WUNET_EINVAL. With WUNET_TRAIN_NO_PARAM_GRADS no weight
 *   gradient, bias or BatchNorm-parameter reduction runs and nothing is written through g_*.
 * WUNET_TRAIN_DETERMINISTIC: the weight gradients and the head's gradients combine their partial sums in an order that depends
 *   only on (n_layers, channels_interval, B, T, precision): each slice of a weight-gradient grid stores its partial dW to a
 *   scratch region after the activations, and one kernel adds the slices in index order (in double); the head's per-CTA
 *   partials are summed likewise. Every other reduction of the step already has a fixed order, so y, the running buffers, all
 *   parameter gradients and dx are bitwise repeatable for the same inputs on the same GPU model, whatever the workspace held
 *   before. The workspace must hold wunet_train_workspace_bytes_ex with this bit. Without it nothing changes. With the
 *   environment variable WUNET_TRAIN_NAIVE=1 (the naive cross-check kernels) a backward with parameter gradients under this
 *   flag is WUNET_ECUDA. Call site: trainer/base_trainer.py:140-143 (torch.backends.cudnn.deterministic = True).
 * The backward must use the precision, the workspace and the WUNET_TRAIN_FROZEN_BN and WUNET_TRAIN_DETERMINISTIC bits of its
 * forward. Bits other than 1, 2 and 16 -> WUNET_EINVAL. Call sites: loss.backward() through model(x) with x.requires_grad in
 * .train() mode, and through model(x) in .eval() mode (trainer/trainer.py:35-37 with model.eval()). */
/* Bytes of training workspace for these flags: wunet_train_workspace_bytes_prec, plus the deterministic scratch when flags has
 * WUNET_TRAIN_DETERMINISTIC. 0 on error (unknown flag bits included). */
size_t wunet_train_workspace_bytes_ex(const wunet_ctx *ctx, int B, int T, int precision, int flags);
int wunet_train_forward_ex(wunet_ctx *ctx, const float *x, float *y, int B, int T, const float *const *conv_w,
                           const float *const *conv_b, const float *const *bn_weight, const float *const *bn_bias,
                           float *const *bn_running_mean, float *const *bn_running_var, const float *out_w, const float *out_b,
                           float momentum, void *workspace, size_t workspace_bytes, void *stream, int precision, int flags);
int wunet_train_backward_ex(wunet_ctx *ctx, const float *x, const float *y, const float *dy, int B, int T,
                            const float *const *conv_w, const float *const *bn_weight, const float *const *bn_bias,
                            const float *out_w, float *const *g_conv_w, float *const *g_conv_b, float *const *g_bn_weight,
                            float *const *g_bn_bias, float *g_out_w, float *g_out_b, void *workspace, size_t workspace_bytes,
                            void *stream, float *dx, int part, int precision, int flags);
/* The same step with per-block BatchNorm modes and momenta and per-parameter gradients: fine-tuning with frozen layers
 * (model.train() with some BatchNorm containers in .eval(), some parameters with requires_grad False).
 * wunet_train_forward_blocks: the arguments of wunet_train_forward_ex, plus
 *   bn_frozen[2n+1] (NULL = none): nonzero = that block's BatchNorm normalises by, and keeps, its running statistics (an
 *     eval-mode container); WUNET_TRAIN_FROZEN_BN in flags freezes every block whatever bn_frozen says;
 *   momenta[2n+1] (NULL = `momentum` for every block): each block's running-statistics factor (ignored for frozen blocks).
 *   The one-value-per-channel check applies only when the middle block has batch statistics; the all-reduce hook (if
 *   installed) is called only for blocks with batch statistics. With both arrays NULL this is wunet_train_forward_ex.
 * wunet_train_backward_blocks: the arguments of wunet_train_backward_ex, plus bn_frozen, which must equal the forward's.
 *   A NULL array among g_conv_w, g_conv_b, g_bn_weight, g_bn_bias, or a NULL entry in one, or a NULL g_out_w / g_out_b,
 *   is a frozen parameter: nothing is computed for it and nothing is written. WUNET_TRAIN_NO_PARAM_GRADS freezes all of them.
 *   Per block, the BatchNorm reduction runs when the block has batch statistics or its weight or bias gets a gradient, the
 *   bias sum when g_conv_b[i] is set and the weight-gradient pass when g_conv_w[i] is set, each with the kernels, grids and
 *   summation order of the full step (bit for bit the same values, deterministic mode included). Early stop: below the
 *   lowest block that gets a gradient (block 0 when dx is requested) nothing is issued, and that block skips its input
 *   gradient; a part with nothing to do returns at once. In a split backward that requests dx, pass dx to part 0 as well:
 *   part 0 writes nothing there but keeps the gradient flowing to the middle block for part 1. Same workspace as the _ex
 *   pair. */
int wunet_train_forward_blocks(wunet_ctx *ctx, const float *x, float *y, int B, int T, const float *const *conv_w,
                               const float *const *conv_b, const float *const *bn_weight, const float *const *bn_bias,
                               float *const *bn_running_mean, float *const *bn_running_var, const float *out_w, const float *out_b,
                               float momentum, void *workspace, size_t workspace_bytes, void *stream, int precision, int flags,
                               const unsigned char *bn_frozen, const float *momenta);
int wunet_train_backward_blocks(wunet_ctx *ctx, const float *x, const float *y, const float *dy, int B, int T,
                                const float *const *conv_w, const float *const *bn_weight, const float *const *bn_bias,
                                const float *out_w, float *const *g_conv_w, float *const *g_conv_b, float *const *g_bn_weight,
                                float *const *g_bn_bias, float *g_out_w, float *g_out_b, void *workspace, size_t workspace_bytes,
                                void *stream, float *dx, int part, int precision, int flags, const unsigned char *bn_frozen);
/* wunet_train_backward_blocks with extra upstream gradients of block outputs: the gradients that flow back into what forward
 * hooks on the reference's encoder[i], middle and decoder[j] captured (feature-matching, deep-supervision or distillation
 * losses on intermediate levels).
 *   g_act[2n+1] (forward order; NULL, or a NULL entry = none): device [B][Cout][L] fp32, the gradient of the loss with respect to
 *     block i's output (its activation after LeakyReLU). It is added, element by element, to the gradient that reaches that
 *     output from the rest of the network (the next block, the decoder's skip, the head), right before block i's BatchNorm
 *     backward, so deterministic mode stays bitwise repeatable and under WUNET_PREC_FP16_SCALED the block's max |dz| includes it.
 *   It is added in the part that processes block i (encoders and middle: part 1, decoders: part 0), and only at or above the
 *     early stop: parameter-gradient and dx requests decide where the backward stops, as in wunet_train_backward_blocks.
 *   With every entry NULL this is wunet_train_backward_blocks: the same launches. */
int wunet_train_backward_inject(wunet_ctx *ctx, const float *x, const float *y, const float *dy, int B, int T,
                                const float *const *conv_w, const float *const *bn_weight, const float *const *bn_bias,
                                const float *out_w, float *const *g_conv_w, float *const *g_conv_b, float *const *g_bn_weight,
                                float *const *g_bn_bias, float *g_out_w, float *g_out_b, void *workspace, size_t workspace_bytes,
                                void *stream, float *dx, int part, int precision, int flags, const unsigned char *bn_frozen,
                                const float *const *g_act);
/* BatchNorm statistics synchronised over data-parallel ranks: what nn.SyncBatchNorm (torch.nn.SyncBatchNorm.
 * convert_sync_batchnorm(model)) computes in a one-process-per-GPU step. With a hook installed, every training forward with
 * batch statistics (not WUNET_TRAIN_FROZEN_BN) on this context, and its backward, compute the BatchNorm reductions from sums
 * over every rank's frames:
 *   forward, per block (C = its Cout, N = sum over ranks of B L): mean = sum z / N and var = sum (z - mean)^2 / N (a second
 *     pass about the GLOBAL mean), both in double and rounded to fp32 as without the hook; the running statistics use var
 *     N / (N - 1) and come out identical on every rank;
 *   backward: mean(dy) and mean(dy zhat) over the N values; the BatchNorm weight / bias gradients stay this rank's sums (the
 *     caller's gradient all-reduce averages them: nn.SyncBatchNorm + DistributedDataParallel arithmetic).
 * `fn` is called on the calling host thread, after the kernels that wrote buf[0 .. count) are enqueued on the call's `stream`;
 * it must leave the element-wise SUM over ranks in buf[0 .. count), ordered on `stream` (an NCCL all-reduce on that stream
 * does this). A nonzero return fails the call with WUNET_ECUDA naming the block; nothing after that point is enqueued.
 * Calls per block, in order:
 *   forward pass 1: buf[0 .. C) = local sum z, buf[C] = local B L                  -> fn(user, buf, C + 1, stream)
 *   forward pass 2: buf[C + 1 .. 2C + 1) = local sum (z - mean)^2                  -> fn(user, buf + C + 1, C, stream)
 *   backward, each block of the part in processing order: [sum dy | sum dy zhat | B L] -> fn(user, buf, 2C + 1, stream)
 * buf: caller-owned device memory of at least 2 * n_layers * channels_interval + 1 doubles (smaller -> WUNET_EINVAL), alive
 * while the hook is installed. fn == NULL uninstalls the hook (the default: per-rank statistics, exactly the launches of a
 * context that never had one). The one-value-per-channel check of wunet_train_forward_ex does not apply to a synchronised
 * forward (nn.SyncBatchNorm raises only without other ranks). A forward and its backward must agree on the hook being
 * installed. No reference counterpart: the reference's nn.DataParallel replicas keep per-replica statistics. */
typedef int (*wunet_bn_allreduce_fn)(void *user, double *buf, size_t count, void *stream);
int wunet_train_set_bn_allreduce(wunet_ctx *ctx, wunet_bn_allreduce_fn fn, void *user, double *buf, size_t capacity);

/* Test hook, synchronous, on caller device buffers (fp32): one convolution-shaped pass of the training step at `precision`
 * (WUNET_PREC_FP32, WUNET_PREC_BF16, WUNET_PREC_TF32 or WUNET_PREC_FP16_SCALED), the kernels the step itself uses (at
 * WUNET_PREC_FP16_SCALED passes 1 and 2 scale dz by 2^k of its max |dz|, as the step does per block). mode: 0 = direct, 1 = decimated (src0 is
 * [B][cin0][2L], every other sample read), 2 = upsample + concat (src0 = [B][cin0][L/2] interpolated 2x linearly,
 * align_corners=True, then src1 = [B][cin1][L]); ksize 15 with modes 0/1, 5 with mode 2 (pass 1 also takes 5 with mode 0).
 * w = [cout][cin0 + cin1][ksize] (Conv1d, no bias).
 *   pass 0: out[B][cout][L] = conv1d(in, w, padding = ksize/2)          (model/unet_basic.py:10,23,53)
 *   pass 1: out[B][cin][L]  = input gradient of that conv for dz [B][cout][L]
 *   pass 2: out[cout][cin][ksize] = weight gradient for dz [B][cout][L]
 * No reference counterpart (autograd computes these inside loss.backward(), trainer/trainer.py:37). */
int wunet_debug_train_conv(int pass, int precision, int mode, int ksize, int B, int L, int cin0, int cin1, int cout,
                           const float *src0, const float *src1, const float *w, const float *dz, float *out);

/* Introspection for tests, host-only (needs no GPU, no context): the training step of an n_layers / channels_interval model at
 * batch B, frame length T and training `precision` (WUNET_PREC_FP32, _BF16, _TF32 or _FP16_SCALED), block `block` (0 .. 2*n_layers,
 * forward order). Writes 22 long longs (capacity >= 22), and a 23rd when capacity >= 23:
 *  [0] z  [1] act  [2] ga  [3] mean  [4] invstd  [5] s1  [6] s2: byte offsets in the training workspace of the block's pre-BatchNorm
 *      output z [B][Cout][L], its activation [B][Cout][L], the activation gradient [B][Cout][L] (which holds dz after the
 *      backward), and the fp32 [Cout] vectors of the BatchNorm mean and 1/sqrt(var + eps) used by the forward and of the
 *      backward's mean(dy) and mean(dy * zhat) (written when that reduction runs)
 *  [7] Cin  [8] Cin0  [9] Cin1 (the skip channels of a decoder)  [10] Cout  [11] L  [12] ksize  [13] input mode (0 = the raw input,
 *      1 = the previous activation decimated, 2 = interpolated previous activation + skip)
 *  [14] weight-gradient kernel (0 = fp32 tiled, 1 = bf16 wgmma, 2 = tf32 wgmma, 3 = fp16 wgmma; block 0 is always 0)  [15] [16] [17] its gridDim x, y, z
 *  [18] (frame, position tile) work items shared by the gridDim.z slices  [19] positions per item  [20] largest number of items
 *      one CTA reduces  [21] wunet_train_workspace_bytes_prec for this B, T and precision
 *  [22] WUNET_PREC_FP16_SCALED: byte offset of the block's dz scale slot (one float: max |dz| of the block, written by the
 *      backward); -1 for other precisions and for block 0.
 * No reference counterpart. */
int wunet_debug_train_layout(int n_layers, int channels_interval, int B, int T, int precision, int block, long long *fields,
                             int capacity);
/* Host-only (needs no GPU): the k of WUNET_PREC_FP16_SCALED's dz scaling for a block whose max |dz| is amax: amax 2^k in
 * [2^13, 2^14); 0 when amax is 0, NaN or infinite; clamped to [-126, 126]. The kernels use the same function. */
int wunet_debug_train_dz_scale(float amax);

/* Introspection for tests and tuning, host-only (needs no GPU, no context): the tiling the bf16 path would use for conv
 * block `block` (1 .. 2*n_layers; block 0 = first encoder runs on CUDA cores) at batch B, frame length T, on a device with
 * num_sms SMs. No reference counterpart. Writes 32 ints:
 *  [0] L  [1] Cin0  [2] Cin1  [3] Cout  [4] Npad  [5] N per CTA  [6] column splits  [7] accumulator column stride  [8] MT (128-row
 *  sub-tiles per tile)  [9] accumulator buffers  [10] packed frames  [11] frames per tile  [12] rows per packed frame
 *  [13] M tiles  [14] K chunks  [15] weights resident  [16] TMA-store epilogue (always 0)  [17] input stages  [18] weight stages
 *  [19] taps per weight stage  [20] weight stages per chunk  [21] input stage bytes  [22] weight stage bytes
 *  [23] TMA bytes per input chunk  [24] input rows used  [25] unused (0)  [26] dynamic shared memory bytes
 *  [27] threads per CTA  [28] CTAs per SM  [29] grid  [30] small (two-CTAs-per-SM) flavour  [31] tiles per frame */
int wunet_debug_plan(int n_layers, int channels_interval, int B, int T, int block, int num_sms, int *fields, int capacity);
/* The same query for a tensor-core precision: WUNET_PREC_BF16 (= wunet_debug_plan), WUNET_PREC_FP16 (the bf16 plan) or
 * WUNET_PREC_FP32_TC (the split-precision plan: no row-pair form, no dense GEMM, block 0 on CUDA cores). WUNET_PREC_FP32 -> WUNET_EINVAL.
 * channels_interval up to 64 (a multiple of 8); [14] counts split-precision K-loop positions (three per 64-channel chunk). */
int wunet_debug_plan_prec(int n_layers, int channels_interval, int B, int T, int block, int num_sms, int *fields, int capacity,
                          int precision);
/* Introspection, host-only: whether conv block `block` runs in 256-row units at that shape and precision (two tiles of one frame
 * per unit, one per consumer warpgroup, so that each weight stage streamed from L2 serves 256 output rows; blocks whose weights
 * are not resident in shared memory, DESIGN.md 5.1), and the geometry of that form. The plan of wunet_debug_plan is the same
 * either way. No reference counterpart. Writes 8 ints, all 0 when the form is not selected:
 *  [0] selected  [1] input stages  [2] weight stages  [3] taps per weight stage  [4] weight stages per chunk
 *  [5] dynamic shared memory bytes  [6] grid  [7] units */
int wunet_debug_plan_m2(int n_layers, int channels_interval, int B, int T, int block, int num_sms, int *fields, int capacity,
                        int precision);

/* Introspection for tests, host-only: the "row-pair" form of one conv block's weights (WUNET_TC_PAIR, DESIGN.md 5.1). A block
 * with `ksize` taps over positions (w = [cout][cin0 + cin1][ksize] fp32, reference layout; model/unet_basic.py:10,23) is the same
 * operator as a block with 2*((ksize-1)/2+1)/2+1 taps over PAIRS of positions: row m = positions 2m and 2m+1, 2*cout output
 * columns, 2*(cin0 + cin1) virtual input channels (decoder != 0: the first segment in the producers' [q0 range | q1 range] order).
 * Writes out[2*cout][2*(cin0+cin1)][taps'] fp32 - what the library packs for the tensor cores. No reference counterpart.
 * decoder == 2: the group-of-8 form of the first block, Conv1d(1 -> cout, k=15) (WUNET_TC_ENC0): row m = samples 8m .. 8m+7 as 8
 * virtual input channels, 8*cout output columns, 3 taps; writes out[8*cout][8][3]. */
int wunet_debug_pair_weights(const float *w, int cout, int cin0, int cin1, int ksize, int decoder, float *out);

#ifdef __cplusplus
}
#endif
#endif /* WUNET_B200_H */
