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
 *   x_dev [B,1,T] fp32 contiguous  ->  y_dev [B,1,T] fp32 contiguous, values in (-1,1).
 * T must be a multiple of 2^n_layers (the reference raises from torch.cat at :95 otherwise)
 * -> WUNET_EINVAL.  Enqueues kernels on `stream` and returns; `workspace` must stay alive until
 * they finish.  Call sites this serves: trainer/trainer.py:75, enhancement.py:66.
 */
int wunet_forward(wunet_ctx *ctx, const float *x_dev, float *y_dev, int B, int T, int precision,
                  void *workspace, size_t workspace_bytes, void *stream);

/*
 * Same operator with HOST buffers (the end-to-end form used by enhancement.py:64-66, which does
 * `model(chunk).detach().cpu()`): copies x_host -> device, runs the forward, copies y back and
 * waits for it.  Uses context-owned, grow-only device buffers and a context-owned stream.
 * x_host/y_host should be pinned for full PCIe rate; pageable memory also works.
 */
int wunet_forward_host(wunet_ctx *ctx, const float *x_host, float *y_host, int B, int T, int precision);

/*
 * Streaming form of the same operator for MANY batches — what enhancement.py:49-74 / trainer/trainer.py:58-79 do when they
 * push every 16384-sample chunk of every clip through the model. wunet_stream_submit() enqueues batch k and returns at once:
 * the H2D copy (copy stream, one of two device slots), the kernels (compute stream) and the D2H copy (second copy stream)
 * of consecutive batches overlap. wunet_stream_wait(ticket) blocks until that batch's y_host is complete. At most two
 * batches are in flight: submitting a third waits for the first. Host buffers should be pinned and must stay valid until
 * the ticket has been waited for.
 */
int wunet_stream_submit(wunet_ctx *ctx, const float *x_host, float *y_host, int B, int T, int precision, int *ticket);
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
