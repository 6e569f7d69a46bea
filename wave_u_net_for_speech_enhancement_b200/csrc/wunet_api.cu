// wunet_api.cu — the C ABI declared in include/wunet_b200.h: context, weight packing, workspace
// carving and the kernel sequence of Model.forward (reference model/unet_basic.py:77-100).
#include <algorithm>
#include <cstring>
#include <thread>
#include <vector>
#include "../../include/wunet_b200.h"
#include "wunet_common.cuh"
#include "wunet_tc.cuh"
#include "wunet_train.cuh"

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <new>
#include <vector>

using namespace wunet;

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

#define CUDA_TRY(expr)                                                                                   \
    do {                                                                                                 \
        cudaError_t e__ = (expr);                                                                        \
        if (e__ != cudaSuccess)                                                                          \
            return fail(WUNET_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
    } while (0)

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct Block {
    int cin, cout, k;
    float *wp = nullptr, *scale = nullptr, *shift = nullptr;   // fp32 packed
};

}  // namespace

struct wunet_ctx {
    int n = 0, ci = 0, device = 0;
    std::vector<Block> blocks;         // 2n+1
    float *out_w = nullptr, *out_b = nullptr;   // device copies [ci+1], [1]
    bool have_weights = false;
    int last_launches = 0;
    TcState *tc = nullptr;             // bf16 / wgmma path state (packed weights, tensor maps)
    bool profile = false;              // record per-block events (wunet_profile_enable)
    std::vector<cudaEvent_t> ev;       // 2n+3 events
    int ev_recorded = 0;
    // forward_host resources (grow-only)
    cudaStream_t hstream = nullptr;
    void *hx = nullptr, *hy = nullptr;
    size_t hx_cap = 0;
    void *hws = nullptr;
    size_t hws_cap = 0;
    // streaming (double-buffered) host pipeline
    cudaStream_t s_in = nullptr, s_out = nullptr;
    void *sx[2] = {nullptr, nullptr}, *sy[2] = {nullptr, nullptr};
    size_t s_cap = 0;
    cudaEvent_t e_in[2] = {}, e_comp[2] = {}, e_done[2] = {};
    bool slot_busy[2] = {false, false};
    int next_ticket = 0;
    // BatchNorm all-reduce hook of the training step (wunet_train_set_bn_allreduce); fn == nullptr: per-rank statistics
    BnSync bn_sync{nullptr, nullptr, nullptr};
};

namespace {

// offsets (bytes) of every block's full-resolution fp32 NCL output inside the fp32 workspace
void fp32_layout(const wunet_ctx *c, int B, int T, std::vector<size_t> &off, size_t &total)
{
    const int n = c->n;
    off.resize(2 * n + 1);
    size_t cur = 0;
    for (int i = 0; i < 2 * n + 1; ++i) {
        const int L = (i <= n) ? (T >> i) : (T >> (2 * n - i));
        off[i] = cur;
        cur += align_up((size_t)B * c->blocks[i].cout * L * sizeof(float), 256);
    }
    total = cur;
}

int level_len(const wunet_ctx *c, int block, int T)
{
    const int n = c->n;
    return (block <= n) ? (T >> block) : (T >> (2 * n - block));
}

int check_shape(const wunet_ctx *c, int B, int T)
{
    if (!c) return fail(WUNET_EINVAL, "null context");
    if (B < 1 || T < 1) return fail(WUNET_EINVAL, "B and T must be positive (B=%d, T=%d)", B, T);
    if (T % (1 << c->n) != 0)
        return fail(WUNET_EINVAL,
                    "input length T=%d is not a multiple of 2^n_layers=%d (the reference raises from torch.cat, "
                    "model/unet_basic.py:95)", T, 1 << c->n);
    if (T % 4 != 0) return fail(WUNET_EINVAL, "T=%d must be a multiple of 4", T);
    return WUNET_OK;
}

cudaEvent_t *prof_events(wunet_ctx *c)
{
    if (!c->profile) return nullptr;
    const size_t need = 2 * (size_t)c->n + 3;
    while (c->ev.size() < need) {
        cudaEvent_t e;
        if (cudaEventCreate(&e) != cudaSuccess) return nullptr;
        c->ev.push_back(e);
    }
    c->ev_recorded = 0;
    return c->ev.data();
}

// x, y: B*T samples of the IoType io; only block 0 (reads x) and the head (reads x, writes y) depend on it
int forward_fp32(wunet_ctx *c, const void *x, void *y, int B, int T, void *ws, cudaStream_t st, int io)
{
    const int n = c->n;
    std::vector<size_t> off;
    size_t total;
    fp32_layout(c, B, T, off, total);
    char *base = static_cast<char *>(ws);
    auto lvl = [&](int i) { return reinterpret_cast<float *>(base + off[i]); };
    int launches = 0;
    cudaEvent_t *ev = prof_events(c);
    if (ev) cudaEventRecord(ev[0], st);
    for (int i = 0; i <= n; ++i) {                       // encoder (model/unet_basic.py:82-86) + middle (:88)
        const Block &bk = c->blocks[i];
        ConvArgs a{};
        a.src0 = (i == 0) ? static_cast<const float *>(x) : lvl(i - 1);
        a.src1 = nullptr;
        a.wp = bk.wp; a.scale = bk.scale; a.shift = bk.shift;
        a.out = lvl(i);
        a.B = B; a.L = T >> i;
        a.Cin = bk.cin; a.Cin0 = bk.cin; a.Cin1 = 0; a.Cout = bk.cout;
        a.up_scale = 0.f;
        const int r = (i == 0 && io != IO_F32) ? launch_conv_fp32_io(a, io, st) : launch_conv_fp32(a, bk.k, i == 0 ? SRC_DIRECT : SRC_DECIM, st);
        if (r < 0) return fail(WUNET_ECUDA, "encoder block %d launch failed: %s", i, cudaGetErrorString(cudaGetLastError()));
        launches += r;
        if (ev) cudaEventRecord(ev[i + 1], st);
    }
    for (int j = 0; j < n; ++j) {                        // decoder (model/unet_basic.py:91-96)
        const Block &bk = c->blocks[n + 1 + j];
        const int e = n - 1 - j;
        ConvArgs a{};
        a.src0 = lvl(n + j);                             // previous block's output (middle for j=0)
        a.src1 = lvl(e);                                 // skip = full-resolution encoder output
        a.wp = bk.wp; a.scale = bk.scale; a.shift = bk.shift;
        a.out = lvl(n + 1 + j);
        a.B = B; a.L = T >> e;
        a.Cin0 = c->blocks[n + j].cout; a.Cin1 = c->blocks[e].cout; a.Cin = a.Cin0 + a.Cin1; a.Cout = bk.cout;
        if (a.Cin != bk.cin) return fail(WUNET_ESTATE, "decoder %d channel plan mismatch", j);
        const int Lin = a.L / 2;
        a.up_scale = (a.L > 1) ? (float)(Lin - 1) / (float)(a.L - 1) : 0.f;
        const int r = launch_conv_fp32(a, bk.k, SRC_UPCAT, st);
        if (r < 0) return fail(WUNET_ECUDA, "decoder block %d launch failed: %s", j, cudaGetErrorString(cudaGetLastError()));
        launches += r;
        if (ev) cudaEventRecord(ev[n + 2 + j], st);
    }
    {                                                    // out (model/unet_basic.py:98-99)
        const int r = io == IO_F32 ? launch_out_fp32(lvl(2 * n), static_cast<const float *>(x), c->out_w, c->out_b, static_cast<float *>(y), B,
                                                     c->ci, T, st)
                                   : launch_out_fp32_io(lvl(2 * n), x, c->out_w, c->out_b, y, B, c->ci, T, io, st);
        if (r < 0) return fail(WUNET_ECUDA, "out launch failed: %s", cudaGetErrorString(cudaGetLastError()));
        launches += r;
        if (ev) { cudaEventRecord(ev[2 * n + 2], st); c->ev_recorded = 2 * n + 3; }
    }
    c->last_launches = launches;
    return WUNET_OK;
}

}  // namespace

extern "C" {

#ifndef WUNET_SRC_HASH
#define WUNET_SRC_HASH "unknown"
#endif
const char *wunet_version(void) { return "wunet_b200 0.3 (sm_90a; fp32 FFMA + bf16 wgmma paths; src " WUNET_SRC_HASH ")"; }

const char *wunet_last_error(void) { return g_err; }

int wunet_create(int n_layers, int channels_interval, int device, wunet_ctx **out)
{
    if (!out) return fail(WUNET_EINVAL, "out is null");
    *out = nullptr;
    if (n_layers < 1 || n_layers > 16 || channels_interval < 1 || channels_interval > 1024)
        return fail(WUNET_EINVAL, "unsupported n_layers=%d / channels_interval=%d", n_layers, channels_interval);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(WUNET_ECUDA, "no CUDA device available (this library has no CPU fallback)");
    }
    if (device < 0 || device >= ndev) return fail(WUNET_EINVAL, "device %d out of range (have %d)", device, ndev);
    wunet_ctx *c = new (std::nothrow) wunet_ctx();
    if (!c) return fail(WUNET_ENOMEM, "out of host memory");
    c->n = n_layers; c->ci = channels_interval; c->device = device;
    const int n = n_layers, ci = channels_interval;
    // channel plan: model/unet_basic.py:38-39 (encoder), :52-57 (middle), :59-62 (decoder)
    for (int i = 0; i < n; ++i) c->blocks.push_back(Block{i == 0 ? 1 : i * ci, (i + 1) * ci, 15});
    c->blocks.push_back(Block{n * ci, n * ci, 15});
    for (int j = 0; j < n; ++j) c->blocks.push_back(Block{j == 0 ? 2 * n * ci : (2 * (n - j) + 1) * ci, (n - j) * ci, 5});
    *out = c;
    return WUNET_OK;
}

void wunet_destroy(wunet_ctx *c)
{
    if (!c) return;
    int prev = 0;
    cudaGetDevice(&prev);
    cudaSetDevice(c->device);
    for (auto &b : c->blocks) { cudaFree(b.wp); cudaFree(b.scale); cudaFree(b.shift); }
    cudaFree(c->out_w); cudaFree(c->out_b);
    tc_destroy(c->tc);
    for (auto e : c->ev) cudaEventDestroy(e);
    if (c->hstream) cudaStreamDestroy(c->hstream);
    cudaFree(c->hx); cudaFree(c->hy); cudaFree(c->hws);
    if (c->s_in) {
        cudaStreamDestroy(c->s_in); cudaStreamDestroy(c->s_out);
        for (int i = 0; i < 2; ++i) { cudaEventDestroy(c->e_in[i]); cudaEventDestroy(c->e_comp[i]); cudaEventDestroy(c->e_done[i]); cudaFree(c->sx[i]); cudaFree(c->sy[i]); }
    }
    cudaSetDevice(prev);
    delete c;
}

int wunet_num_blocks(const wunet_ctx *c) { return c ? (int)c->blocks.size() : fail(WUNET_EINVAL, "null context"); }

int wunet_block_shape(const wunet_ctx *c, int block, int *cin, int *cout, int *ksize)
{
    if (!c || block < 0 || block >= (int)c->blocks.size()) return fail(WUNET_EINVAL, "bad block index %d", block);
    if (cin) *cin = c->blocks[block].cin;
    if (cout) *cout = c->blocks[block].cout;
    if (ksize) *ksize = c->blocks[block].k;
    return WUNET_OK;
}

int wunet_set_weights(wunet_ctx *c, const float *const *conv_w, const float *const *conv_b,
                      const float *const *bn_weight, const float *const *bn_bias,
                      const float *const *bn_running_mean, const float *const *bn_running_var, const float *out_w,
                      const float *out_b, void *stream)
{
    if (!c) return fail(WUNET_EINVAL, "null context");
    if (!conv_w || !conv_b || !bn_weight || !bn_bias || !bn_running_mean || !bn_running_var || !out_w || !out_b)
        return fail(WUNET_EINVAL, "null parameter array");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_TRY(cudaSetDevice(c->device));
    for (size_t i = 0; i < c->blocks.size(); ++i) {
        Block &b = c->blocks[i];
        if (!conv_w[i] || !conv_b[i] || !bn_weight[i] || !bn_bias[i] || !bn_running_mean[i] || !bn_running_var[i])
            return fail(WUNET_EINVAL, "null parameter pointer for block %zu", i);
        const size_t wn = (size_t)b.cout * b.cin * b.k;
        if (!b.wp) {
            CUDA_TRY(cudaMalloc(&b.wp, wn * sizeof(float)));
            CUDA_TRY(cudaMalloc(&b.scale, b.cout * sizeof(float)));
            CUDA_TRY(cudaMalloc(&b.shift, b.cout * sizeof(float)));
        }
        if (launch_pack_fp32(conv_w[i], conv_b[i], bn_weight[i], bn_bias[i], bn_running_mean[i], bn_running_var[i],
                             b.wp, b.scale, b.shift, b.cout, b.cin, b.k, st) < 0)
            return fail(WUNET_ECUDA, "pack kernel launch failed: %s", cudaGetErrorString(cudaGetLastError()));
    }
    if (!c->out_w) {
        CUDA_TRY(cudaMalloc(&c->out_w, (c->ci + 1) * sizeof(float)));
        CUDA_TRY(cudaMalloc(&c->out_b, sizeof(float)));
    }
    CUDA_TRY(cudaMemcpyAsync(c->out_w, out_w, (c->ci + 1) * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(c->out_b, out_b, sizeof(float), cudaMemcpyDeviceToDevice, st));
    // bf16 / wgmma path: repack from the folded fp32 copies
    {
        std::vector<TcBlockSrc> src(c->blocks.size());
        for (size_t i = 0; i < c->blocks.size(); ++i)
            src[i] = TcBlockSrc{c->blocks[i].cin, c->blocks[i].cout, c->blocks[i].k, conv_w[i], c->blocks[i].scale,
                                c->blocks[i].shift};
        const int r = tc_set_weights(&c->tc, c->n, c->ci, src.data(), (int)src.size(), c->out_w, c->out_b, st);
        if (r != 0) return fail(WUNET_ECUDA, "tensor-core weight packing failed: %s", tc_error());
    }
    c->have_weights = true;
    return WUNET_OK;
}

// inference precision -> tc_* mode (0 = bf16, 1 = split precision, 2 = fp16); -1 for the fp32 path and anything else
static int tc_mode(int precision)
{
    return precision == WUNET_PREC_BF16 ? 0 : precision == WUNET_PREC_FP32_TC ? 1 : precision == WUNET_PREC_FP16 ? 2 : -1;
}

size_t wunet_workspace_bytes(const wunet_ctx *c, int B, int T, int precision)
{
    if (check_shape(c, B, T) != WUNET_OK) return 0;
    if (precision == WUNET_PREC_FP32) {
        std::vector<size_t> off;
        size_t total;
        fp32_layout(c, B, T, off, total);
        return total;
    }
    if (tc_mode(precision) >= 0) return tc_workspace_bytes(c->n, c->ci, B, T, tc_mode(precision));
    if (precision == WUNET_PREC_TF32) fail(WUNET_EINVAL, "WUNET_PREC_TF32 is a training precision only (the forward has no tf32 path)");
    else if (precision == WUNET_PREC_FP16_SCALED)
        fail(WUNET_EINVAL, "WUNET_PREC_FP16_SCALED is a training precision only (inference in fp16 is WUNET_PREC_FP16)");
    else fail(WUNET_EINVAL, "unknown precision %d", precision);
    return 0;
}

static int check_io(int io)
{
    if (io != WUNET_IO_F32 && io != WUNET_IO_F16 && io != WUNET_IO_BF16) return fail(WUNET_EINVAL, "unknown I/O dtype %d", io);
    return WUNET_OK;
}

int wunet_forward(wunet_ctx *c, const float *x, float *y, int B, int T, int precision, void *workspace,
                  size_t workspace_bytes, void *stream)
{
    return wunet_forward_io(c, x, y, B, T, precision, WUNET_IO_F32, workspace, workspace_bytes, stream);
}

// wunet_forward_io; store_last: the tensor-core forward also stores the last decoder block (wunet_forward_export)
static int forward_io_impl(wunet_ctx *c, const void *x, void *y, int B, int T, int precision, int io, void *workspace,
                           size_t workspace_bytes, void *stream, bool store_last)
{
    int rc = check_shape(c, B, T);
    if (rc != WUNET_OK) return rc;
    if (check_io(io) != WUNET_OK) return WUNET_EINVAL;
    if (!c->have_weights) return fail(WUNET_ESTATE, "wunet_forward called before wunet_set_weights");
    if (!x || !y || !workspace) return fail(WUNET_EINVAL, "null buffer");
    const size_t need = wunet_workspace_bytes(c, B, T, precision);
    if (need == 0) return WUNET_EINVAL;
    if (workspace_bytes < need) return fail(WUNET_ENOMEM, "workspace too small: %zu < %zu bytes", workspace_bytes, need);
    CUDA_TRY(cudaSetDevice(c->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (precision == WUNET_PREC_FP32) return forward_fp32(c, x, y, B, T, workspace, st, io);
    int launches = 0;
    cudaEvent_t *ev = prof_events(c);
    if (tc_mode(precision) < 0) return fail(WUNET_EINVAL, "unknown precision %d", precision);
    const int r = tc_forward(c->tc, x, y, B, T, workspace, st, &launches, ev, tc_mode(precision), io, store_last);
    if (ev && r == 0) c->ev_recorded = 2 * c->n + 3;
    if (r != 0) return fail(WUNET_ECUDA, "tensor-core forward failed: %s", tc_error());
    c->last_launches = launches;
    return WUNET_OK;
}

int wunet_forward_io(wunet_ctx *c, const void *x, void *y, int B, int T, int precision, int io, void *workspace,
                     size_t workspace_bytes, void *stream)
{
    return forward_io_impl(c, x, y, B, T, precision, io, workspace, workspace_bytes, stream, false);
}

int wunet_forward_export(wunet_ctx *c, const void *x, void *y, int B, int T, int precision, int io,
                         const unsigned char *export_mask, void *const *level_out, void *workspace, size_t workspace_bytes,
                         void *stream)
{
    if (!c) return fail(WUNET_EINVAL, "null context");
    const int nb = 2 * c->n + 1;
    bool any = false;
    for (int i = 0; export_mask && i < nb; ++i) {
        if (!export_mask[i]) continue;
        if (!level_out || !level_out[i]) return fail(WUNET_EINVAL, "block %d is marked for export but has no output buffer", i);
        any = true;
    }
    const bool last = any && export_mask[nb - 1];
    int rc = forward_io_impl(c, x, y, B, T, precision, io, workspace, workspace_bytes, stream, last);
    if (rc != WUNET_OK || !any) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    std::vector<size_t> off;
    size_t total;
    if (precision == WUNET_PREC_FP32) fp32_layout(c, B, T, off, total);
    for (int i = 0; i < nb; ++i) {
        if (!export_mask[i]) continue;
        const int C = c->blocks[i].cout, L = level_len(c, i, T);
        if (precision != WUNET_PREC_FP32) {
            if (tc_export_level(c->tc, i, workspace, B, T, level_out[i], io, st, tc_mode(precision)) != 0)
                return fail(WUNET_ECUDA, "block %d export failed: %s", i, tc_error());
        } else if (io == WUNET_IO_F32) {
            CUDA_TRY(cudaMemcpyAsync(level_out[i], static_cast<const char *>(workspace) + off[i], (size_t)B * C * L * sizeof(float),
                                     cudaMemcpyDeviceToDevice, st));
        } else if (launch_level_export_io(static_cast<const char *>(workspace) + off[i], LEVEL_F32_NCL, level_out[i], io, B, L, C, st) < 0)
            return fail(WUNET_ECUDA, "block %d export launch failed: %s", i, cudaGetErrorString(cudaGetLastError()));
    }
    return WUNET_OK;
}

int wunet_forward_host(wunet_ctx *c, const float *x_host, float *y_host, int B, int T, int precision)
{
    return wunet_forward_host_io(c, x_host, y_host, B, T, precision, WUNET_IO_F32);
}

int wunet_forward_host_io(wunet_ctx *c, const void *x_host, void *y_host, int B, int T, int precision, int io)
{
    int rc = check_shape(c, B, T);
    if (rc != WUNET_OK) return rc;
    if (check_io(io) != WUNET_OK) return WUNET_EINVAL;
    if (!x_host || !y_host) return fail(WUNET_EINVAL, "null host buffer");
    CUDA_TRY(cudaSetDevice(c->device));
    if (!c->hstream) CUDA_TRY(cudaStreamCreateWithFlags(&c->hstream, cudaStreamNonBlocking));
    const size_t nbytes = (size_t)B * T * io_bytes(io);
    if (c->hx_cap < nbytes) {
        cudaFree(c->hx); cudaFree(c->hy);
        c->hx = c->hy = nullptr; c->hx_cap = 0;
        CUDA_TRY(cudaMalloc(&c->hx, nbytes));
        CUDA_TRY(cudaMalloc(&c->hy, nbytes));
        c->hx_cap = nbytes;
    }
    const size_t need = wunet_workspace_bytes(c, B, T, precision);
    if (need == 0) return WUNET_EINVAL;
    if (c->hws_cap < need) {
        cudaFree(c->hws);
        c->hws = nullptr; c->hws_cap = 0;
        CUDA_TRY(cudaMalloc(&c->hws, need));
        c->hws_cap = need;
    }
    if (tc_mode(precision) >= 0) {
        // chunked pipeline: H2D, first/last kernels and D2H overlap per batch chunk (see tc_forward_host)
        if (!c->have_weights) return fail(WUNET_ESTATE, "wunet_forward_host called before wunet_set_weights");
        int launches = 0;
        if (tc_forward_host(c->tc, x_host, y_host, c->hx, c->hy, B, T, c->hws, c->hstream, &launches, tc_mode(precision), io) != 0)
            return fail(WUNET_ECUDA, "tensor-core host pipeline failed: %s", tc_error());
        c->last_launches = launches;
        return WUNET_OK;
    }
    CUDA_TRY(cudaMemcpyAsync(c->hx, x_host, nbytes, cudaMemcpyHostToDevice, c->hstream));
    rc = wunet_forward_io(c, c->hx, c->hy, B, T, precision, io, c->hws, c->hws_cap, c->hstream);
    if (rc != WUNET_OK) return rc;
    CUDA_TRY(cudaMemcpyAsync(y_host, c->hy, nbytes, cudaMemcpyDeviceToHost, c->hstream));
    CUDA_TRY(cudaStreamSynchronize(c->hstream));
    return WUNET_OK;
}

int wunet_stream_submit(wunet_ctx *c, const float *x_host, float *y_host, int B, int T, int precision, int *ticket)
{
    return wunet_stream_submit_io(c, x_host, y_host, B, T, precision, WUNET_IO_F32, ticket);
}

int wunet_stream_submit_io(wunet_ctx *c, const void *x_host, void *y_host, int B, int T, int precision, int io, int *ticket)
{
    int rc = check_shape(c, B, T);
    if (rc != WUNET_OK) return rc;
    if (check_io(io) != WUNET_OK) return WUNET_EINVAL;
    if (!x_host || !y_host || !ticket) return fail(WUNET_EINVAL, "null argument");
    if (!c->have_weights) return fail(WUNET_ESTATE, "wunet_stream_submit called before wunet_set_weights");
    CUDA_TRY(cudaSetDevice(c->device));
    if (!c->hstream) CUDA_TRY(cudaStreamCreateWithFlags(&c->hstream, cudaStreamNonBlocking));
    if (!c->s_in) {
        CUDA_TRY(cudaStreamCreateWithFlags(&c->s_in, cudaStreamNonBlocking));
        CUDA_TRY(cudaStreamCreateWithFlags(&c->s_out, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
            CUDA_TRY(cudaEventCreateWithFlags(&c->e_in[i], cudaEventDisableTiming));
            CUDA_TRY(cudaEventCreateWithFlags(&c->e_comp[i], cudaEventDisableTiming));
            CUDA_TRY(cudaEventCreateWithFlags(&c->e_done[i], cudaEventDisableTiming));
        }
    }
    const size_t nbytes = (size_t)B * T * io_bytes(io);
    const int k = c->next_ticket;
    const int slot = k & 1;
    if (c->slot_busy[slot]) { CUDA_TRY(cudaEventSynchronize(c->e_done[slot])); c->slot_busy[slot] = false; }
    if (c->s_cap < nbytes) {
        for (int i = 0; i < 2; ++i) {
            if (c->slot_busy[i]) { CUDA_TRY(cudaEventSynchronize(c->e_done[i])); c->slot_busy[i] = false; }
            cudaFree(c->sx[i]); cudaFree(c->sy[i]); c->sx[i] = c->sy[i] = nullptr;
        }
        c->s_cap = 0;
        for (int i = 0; i < 2; ++i) { CUDA_TRY(cudaMalloc(&c->sx[i], nbytes)); CUDA_TRY(cudaMalloc(&c->sy[i], nbytes)); }
        c->s_cap = nbytes;
    }
    const size_t need = wunet_workspace_bytes(c, B, T, precision);
    if (need == 0) return WUNET_EINVAL;
    if (c->hws_cap < need) {
        CUDA_TRY(cudaStreamSynchronize(c->hstream));
        cudaFree(c->hws);
        c->hws = nullptr; c->hws_cap = 0;
        CUDA_TRY(cudaMalloc(&c->hws, need));
        c->hws_cap = need;
    }
    // slot reuse: x_dev[slot] was last read by the forward of ticket k-2 (e_comp), y_dev[slot] by its D2H (e_done, waited above)
    if (k >= 2) CUDA_TRY(cudaStreamWaitEvent(c->s_in, c->e_comp[slot], 0));
    CUDA_TRY(cudaMemcpyAsync(c->sx[slot], x_host, nbytes, cudaMemcpyHostToDevice, c->s_in));
    CUDA_TRY(cudaEventRecord(c->e_in[slot], c->s_in));
    CUDA_TRY(cudaStreamWaitEvent(c->hstream, c->e_in[slot], 0));
    rc = wunet_forward_io(c, c->sx[slot], c->sy[slot], B, T, precision, io, c->hws, c->hws_cap, c->hstream);
    if (rc != WUNET_OK) return rc;
    CUDA_TRY(cudaEventRecord(c->e_comp[slot], c->hstream));
    CUDA_TRY(cudaStreamWaitEvent(c->s_out, c->e_comp[slot], 0));
    CUDA_TRY(cudaMemcpyAsync(y_host, c->sy[slot], nbytes, cudaMemcpyDeviceToHost, c->s_out));
    CUDA_TRY(cudaEventRecord(c->e_done[slot], c->s_out));
    c->slot_busy[slot] = true;
    *ticket = k;
    c->next_ticket = k + 1;
    return WUNET_OK;
}

int wunet_stream_wait(wunet_ctx *c, int ticket)
{
    if (!c) return fail(WUNET_EINVAL, "null context");
    if (ticket < 0 || ticket >= c->next_ticket) return fail(WUNET_EINVAL, "unknown ticket %d", ticket);
    if (ticket < c->next_ticket - 2) return WUNET_OK;            // older tickets were completed when their slot was reused
    const int slot = ticket & 1;
    CUDA_TRY(cudaSetDevice(c->device));
    if (c->slot_busy[slot]) { CUDA_TRY(cudaEventSynchronize(c->e_done[slot])); c->slot_busy[slot] = false; }
    return WUNET_OK;
}

int wunet_read_level(wunet_ctx *c, int block, const void *workspace, int B, int T, int precision, float *out_dev,
                     void *stream)
{
    int rc = check_shape(c, B, T);
    if (rc != WUNET_OK) return rc;
    if (block < 0 || block >= (int)c->blocks.size() || !workspace || !out_dev)
        return fail(WUNET_EINVAL, "bad block index / null buffer");
    CUDA_TRY(cudaSetDevice(c->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int L = level_len(c, block, T);
    if (precision == WUNET_PREC_FP32) {
        std::vector<size_t> off;
        size_t total;
        fp32_layout(c, B, T, off, total);
        CUDA_TRY(cudaMemcpyAsync(out_dev, static_cast<const char *>(workspace) + off[block],
                                 (size_t)B * c->blocks[block].cout * L * sizeof(float), cudaMemcpyDeviceToDevice, st));
        return WUNET_OK;
    }
    if (tc_mode(precision) >= 0) {
        const int r = tc_read_level(c->tc, block, workspace, B, T, out_dev, st, tc_mode(precision));
        if (r != 0) return fail(WUNET_ECUDA, "tc_read_level failed: %s", tc_error());
        return WUNET_OK;
    }
    return fail(WUNET_EINVAL, "unknown precision %d", precision);
}

int wunet_last_launch_count(const wunet_ctx *c) { return c ? c->last_launches : 0; }

// training precision -> TrainPrec; -1 (with the error message set) when it is not one
static int train_prec(int precision)
{
    if (precision == WUNET_PREC_FP32) return TRAIN_FP32;
    if (precision == WUNET_PREC_BF16) return TRAIN_BF16;
    if (precision == WUNET_PREC_TF32) return TRAIN_TF32;
    if (precision == WUNET_PREC_FP16_SCALED) return TRAIN_FP16_SCALED;
    if (precision == WUNET_PREC_FP32_TC || precision == WUNET_PREC_FP16)
        fail(WUNET_EINVAL, "training precision %s is not supported: use WUNET_PREC_FP32, WUNET_PREC_BF16, WUNET_PREC_TF32 or "
             "WUNET_PREC_FP16_SCALED",
             precision == WUNET_PREC_FP16 ? "WUNET_PREC_FP16" : "WUNET_PREC_FP32_TC");
    else
        fail(WUNET_EINVAL, "unknown training precision %d", precision);
    return -1;
}

size_t wunet_train_workspace_bytes(const wunet_ctx *c, int B, int T)
{
    return wunet_train_workspace_bytes_prec(c, B, T, WUNET_PREC_FP32);
}

size_t wunet_train_workspace_bytes_prec(const wunet_ctx *c, int B, int T, int precision)
{
    if (check_shape(c, B, T) != WUNET_OK) return 0;
    const int prec = train_prec(precision);
    if (prec < 0) return 0;
    return train_workspace_bytes(c->n, c->ci, B, T, prec);
}

static const int kTrainFlags = WUNET_TRAIN_FROZEN_BN | WUNET_TRAIN_NO_PARAM_GRADS | WUNET_TRAIN_DETERMINISTIC;

// the flags the training kernels act on (TrainFlags) for the public bits
static int train_flags(int flags)
{
    return ((flags & WUNET_TRAIN_FROZEN_BN) ? TRAIN_FROZEN_BN : 0) | ((flags & WUNET_TRAIN_NO_PARAM_GRADS) ? TRAIN_NO_PARAM_GRADS : 0) |
           ((flags & WUNET_TRAIN_DETERMINISTIC) ? TRAIN_DETERMINISTIC : 0);
}

size_t wunet_train_workspace_bytes_ex(const wunet_ctx *c, int B, int T, int precision, int flags)
{
    if (check_shape(c, B, T) != WUNET_OK) return 0;
    const int prec = train_prec(precision);
    if (prec < 0) return 0;
    if (flags & ~kTrainFlags) {
        fail(WUNET_EINVAL, "unknown training flags 0x%x", flags);
        return 0;
    }
    return train_workspace_bytes(c->n, c->ci, B, T, prec, train_flags(flags));
}

int wunet_train_forward(wunet_ctx *c, const float *x, float *y, int B, int T, const float *const *conv_w,
                        const float *const *conv_b, const float *const *bn_weight, const float *const *bn_bias,
                        float *const *bn_running_mean, float *const *bn_running_var, const float *out_w, const float *out_b,
                        float momentum, void *workspace, size_t workspace_bytes, void *stream)
{
    return wunet_train_forward_prec(c, x, y, B, T, conv_w, conv_b, bn_weight, bn_bias, bn_running_mean, bn_running_var, out_w,
                                    out_b, momentum, workspace, workspace_bytes, stream, WUNET_PREC_FP32);
}

int wunet_train_forward_prec(wunet_ctx *c, const float *x, float *y, int B, int T, const float *const *conv_w,
                             const float *const *conv_b, const float *const *bn_weight, const float *const *bn_bias,
                             float *const *bn_running_mean, float *const *bn_running_var, const float *out_w, const float *out_b,
                             float momentum, void *workspace, size_t workspace_bytes, void *stream, int precision)
{
    return wunet_train_forward_ex(c, x, y, B, T, conv_w, conv_b, bn_weight, bn_bias, bn_running_mean, bn_running_var, out_w,
                                  out_b, momentum, workspace, workspace_bytes, stream, precision, 0);
}

// wunet_train_forward_ex and wunet_train_forward_blocks: bn_frozen / momenta null = every block as `flags` and `momentum` say
static int train_forward_impl(wunet_ctx *c, const float *x, float *y, int B, int T, const float *const *conv_w,
                              const float *const *conv_b, const float *const *bn_weight, const float *const *bn_bias,
                              float *const *bn_running_mean, float *const *bn_running_var, const float *out_w, const float *out_b,
                              float momentum, void *workspace, size_t workspace_bytes, void *stream, int precision, int flags,
                              const unsigned char *bn_frozen, const float *momenta)
{
    int rc = check_shape(c, B, T);
    if (rc != WUNET_OK) return rc;
    const int prec = train_prec(precision);
    if (prec < 0) return WUNET_EINVAL;
    if (flags & ~kTrainFlags) return fail(WUNET_EINVAL, "unknown training flags 0x%x", flags);
    const int nb = 2 * c->n + 1;
    const bool all_frozen = flags & WUNET_TRAIN_FROZEN_BN;
    bool any_batch = !all_frozen;
    if (bn_frozen && !all_frozen) {
        any_batch = false;
        for (int i = 0; i < nb; ++i) any_batch = any_batch || !bn_frozen[i];
    }
    // batch statistics of one value per channel (B = 1 and L = 1 at the middle block): torch.nn.BatchNorm1d raises in training
    // mode rather than normalise by a variance of 0. Synchronised statistics count every rank's frames (nn.SyncBatchNorm
    // raises only without other ranks).
    const bool synced = c->bn_sync.fn && any_batch;
    const bool middle_batch = !all_frozen && !(bn_frozen && bn_frozen[c->n]);
    if (middle_batch && !synced && B == 1 && (T >> c->n) == 1)
        return fail(WUNET_EINVAL, "Expected more than 1 value per channel when training (B=1, T=%d: one value per channel at the "
                                  "middle block)", T);
    if (!x || !y || !workspace || !conv_w || !conv_b || !bn_weight || !bn_bias || !bn_running_mean || !bn_running_var || !out_w || !out_b)
        return fail(WUNET_EINVAL, "null argument");
    const int tflags = train_flags(flags & ~WUNET_TRAIN_NO_PARAM_GRADS);               // NO_PARAM_GRADS: nothing to do here
    const size_t need = train_workspace_bytes(c->n, c->ci, B, T, prec, tflags);
    if (workspace_bytes < need) return fail(WUNET_ENOMEM, "training workspace too small: %zu < %zu bytes", workspace_bytes, need);
    CUDA_TRY(cudaSetDevice(c->device));
    const TrainParams P{conv_w, conv_b, bn_weight, bn_bias, bn_running_mean, bn_running_var, out_w, out_b};
    std::vector<float> m(nb, momentum);
    if (momenta) m.assign(momenta, momenta + nb);
    if (train_forward(c->n, c->ci, x, y, B, T, P, m.data(), workspace, static_cast<cudaStream_t>(stream), prec, tflags,
                      synced ? &c->bn_sync : nullptr, bn_frozen))
        return fail(WUNET_ECUDA, "%s", train_error());
    return WUNET_OK;
}

int wunet_train_forward_ex(wunet_ctx *c, const float *x, float *y, int B, int T, const float *const *conv_w,
                           const float *const *conv_b, const float *const *bn_weight, const float *const *bn_bias,
                           float *const *bn_running_mean, float *const *bn_running_var, const float *out_w, const float *out_b,
                           float momentum, void *workspace, size_t workspace_bytes, void *stream, int precision, int flags)
{
    return train_forward_impl(c, x, y, B, T, conv_w, conv_b, bn_weight, bn_bias, bn_running_mean, bn_running_var, out_w, out_b,
                              momentum, workspace, workspace_bytes, stream, precision, flags, nullptr, nullptr);
}

int wunet_train_forward_blocks(wunet_ctx *c, const float *x, float *y, int B, int T, const float *const *conv_w,
                               const float *const *conv_b, const float *const *bn_weight, const float *const *bn_bias,
                               float *const *bn_running_mean, float *const *bn_running_var, const float *out_w, const float *out_b,
                               float momentum, void *workspace, size_t workspace_bytes, void *stream, int precision, int flags,
                               const unsigned char *bn_frozen, const float *momenta)
{
    return train_forward_impl(c, x, y, B, T, conv_w, conv_b, bn_weight, bn_bias, bn_running_mean, bn_running_var, out_w, out_b,
                              momentum, workspace, workspace_bytes, stream, precision, flags, bn_frozen, momenta);
}

int wunet_train_backward(wunet_ctx *c, const float *x, const float *y, const float *dy, int B, int T,
                         const float *const *conv_w, const float *const *bn_weight, const float *const *bn_bias, const float *out_w,
                         float *const *g_conv_w, float *const *g_conv_b, float *const *g_bn_weight, float *const *g_bn_bias,
                         float *g_out_w, float *g_out_b, void *workspace, size_t workspace_bytes, void *stream)
{
    return wunet_train_backward_part_prec(c, x, y, dy, B, T, conv_w, bn_weight, bn_bias, out_w, g_conv_w, g_conv_b, g_bn_weight,
                                          g_bn_bias, g_out_w, g_out_b, workspace, workspace_bytes, stream, -1, WUNET_PREC_FP32);
}

int wunet_train_backward_part(wunet_ctx *c, const float *x, const float *y, const float *dy, int B, int T,
                              const float *const *conv_w, const float *const *bn_weight, const float *const *bn_bias,
                              const float *out_w, float *const *g_conv_w, float *const *g_conv_b, float *const *g_bn_weight,
                              float *const *g_bn_bias, float *g_out_w, float *g_out_b, void *workspace, size_t workspace_bytes,
                              void *stream, int part)
{
    return wunet_train_backward_part_prec(c, x, y, dy, B, T, conv_w, bn_weight, bn_bias, out_w, g_conv_w, g_conv_b, g_bn_weight,
                                          g_bn_bias, g_out_w, g_out_b, workspace, workspace_bytes, stream, part, WUNET_PREC_FP32);
}

int wunet_train_backward_part_prec(wunet_ctx *c, const float *x, const float *y, const float *dy, int B, int T,
                                   const float *const *conv_w, const float *const *bn_weight, const float *const *bn_bias,
                                   const float *out_w, float *const *g_conv_w, float *const *g_conv_b, float *const *g_bn_weight,
                                   float *const *g_bn_bias, float *g_out_w, float *g_out_b, void *workspace, size_t workspace_bytes,
                                   void *stream, int part, int precision)
{
    return wunet_train_backward_ex(c, x, y, dy, B, T, conv_w, bn_weight, bn_bias, out_w, g_conv_w, g_conv_b, g_bn_weight, g_bn_bias,
                                   g_out_w, g_out_b, workspace, workspace_bytes, stream, nullptr, part, precision, 0);
}

// wunet_train_backward_ex (blocks = false: every gradient slot set unless WUNET_TRAIN_NO_PARAM_GRADS, no early stop) and
// wunet_train_backward_blocks (null slots are frozen parameters; bn_frozen as in the forward)
static int train_backward_impl(wunet_ctx *c, const float *x, const float *y, const float *dy, int B, int T,
                               const float *const *conv_w, const float *const *bn_weight, const float *const *bn_bias,
                               const float *out_w, float *const *g_conv_w, float *const *g_conv_b, float *const *g_bn_weight,
                               float *const *g_bn_bias, float *g_out_w, float *g_out_b, void *workspace, size_t workspace_bytes,
                               void *stream, float *dx, int part, int precision, int flags, bool blocks,
                               const unsigned char *bn_frozen, const float *const *g_act = nullptr)
{
    int rc = check_shape(c, B, T);
    if (rc != WUNET_OK) return rc;
    const int prec = train_prec(precision);
    if (prec < 0) return WUNET_EINVAL;
    if (flags & ~kTrainFlags) return fail(WUNET_EINVAL, "unknown training flags 0x%x", flags);
    if (dx && part == 0 && !blocks) return fail(WUNET_EINVAL, "dx belongs to part 1 (block 0): pass it with part -1 or 1, not 0");
    const bool pgrads = !(flags & WUNET_TRAIN_NO_PARAM_GRADS) && !blocks;
    if (!x || !y || !dy || !workspace || !conv_w || !bn_weight || !bn_bias || !out_w ||
        (pgrads && (!g_conv_w || !g_conv_b || !g_bn_weight || !g_bn_bias || !g_out_w || !g_out_b)))
        return fail(WUNET_EINVAL, "null argument");
    const int tflags = train_flags(flags);
    const size_t need = train_workspace_bytes(c->n, c->ci, B, T, prec, tflags);
    if (workspace_bytes < need) return fail(WUNET_ENOMEM, "training workspace too small: %zu < %zu bytes", workspace_bytes, need);
    CUDA_TRY(cudaSetDevice(c->device));
    const TrainParams P{conv_w, nullptr, bn_weight, bn_bias, nullptr, nullptr, out_w, nullptr};
    const TrainGrads G{g_conv_w, g_conv_b, g_bn_weight, g_bn_bias, g_out_w, g_out_b};
    bool any_batch = !(flags & WUNET_TRAIN_FROZEN_BN);
    if (bn_frozen && any_batch) {
        any_batch = false;
        for (int i = 0; i < 2 * c->n + 1; ++i) any_batch = any_batch || !bn_frozen[i];
    }
    const bool synced = c->bn_sync.fn && any_batch;
    if (train_backward(c->n, c->ci, x, y, dy, B, T, P, G, workspace, static_cast<cudaStream_t>(stream), part, prec, dx, tflags,
                       synced ? &c->bn_sync : nullptr, bn_frozen, blocks, g_act))
        return fail(WUNET_ECUDA, "%s", train_error());
    return WUNET_OK;
}

int wunet_train_backward_ex(wunet_ctx *c, const float *x, const float *y, const float *dy, int B, int T,
                            const float *const *conv_w, const float *const *bn_weight, const float *const *bn_bias,
                            const float *out_w, float *const *g_conv_w, float *const *g_conv_b, float *const *g_bn_weight,
                            float *const *g_bn_bias, float *g_out_w, float *g_out_b, void *workspace, size_t workspace_bytes,
                            void *stream, float *dx, int part, int precision, int flags)
{
    return train_backward_impl(c, x, y, dy, B, T, conv_w, bn_weight, bn_bias, out_w, g_conv_w, g_conv_b, g_bn_weight, g_bn_bias,
                               g_out_w, g_out_b, workspace, workspace_bytes, stream, dx, part, precision, flags, false, nullptr);
}

int wunet_train_backward_blocks(wunet_ctx *c, const float *x, const float *y, const float *dy, int B, int T,
                                const float *const *conv_w, const float *const *bn_weight, const float *const *bn_bias,
                                const float *out_w, float *const *g_conv_w, float *const *g_conv_b, float *const *g_bn_weight,
                                float *const *g_bn_bias, float *g_out_w, float *g_out_b, void *workspace, size_t workspace_bytes,
                                void *stream, float *dx, int part, int precision, int flags, const unsigned char *bn_frozen)
{
    return train_backward_impl(c, x, y, dy, B, T, conv_w, bn_weight, bn_bias, out_w, g_conv_w, g_conv_b, g_bn_weight, g_bn_bias,
                               g_out_w, g_out_b, workspace, workspace_bytes, stream, dx, part, precision, flags, true, bn_frozen);
}

int wunet_train_backward_inject(wunet_ctx *c, const float *x, const float *y, const float *dy, int B, int T,
                                const float *const *conv_w, const float *const *bn_weight, const float *const *bn_bias,
                                const float *out_w, float *const *g_conv_w, float *const *g_conv_b, float *const *g_bn_weight,
                                float *const *g_bn_bias, float *g_out_w, float *g_out_b, void *workspace, size_t workspace_bytes,
                                void *stream, float *dx, int part, int precision, int flags, const unsigned char *bn_frozen,
                                const float *const *g_act)
{
    return train_backward_impl(c, x, y, dy, B, T, conv_w, bn_weight, bn_bias, out_w, g_conv_w, g_conv_b, g_bn_weight, g_bn_bias,
                               g_out_w, g_out_b, workspace, workspace_bytes, stream, dx, part, precision, flags, true, bn_frozen,
                               g_act);
}

int wunet_train_set_bn_allreduce(wunet_ctx *c, wunet_bn_allreduce_fn fn, void *user, double *buf, size_t capacity)
{
    if (!c) return fail(WUNET_EINVAL, "null context");
    if (!fn) {
        c->bn_sync = BnSync{nullptr, nullptr, nullptr};
        return WUNET_OK;
    }
    const size_t need = 2 * (size_t)c->n * c->ci + 1;                 // [sum dy | sum dy zh | B L] of the widest block (n ci)
    if (!buf || capacity < need)
        return fail(WUNET_EINVAL, "BatchNorm all-reduce buffer too small: %zu < %zu doubles", buf ? capacity : (size_t)0, need);
    c->bn_sync = BnSync{fn, user, buf};
    return WUNET_OK;
}

int wunet_debug_train_conv(int pass, int precision, int mode, int ksize, int B, int L, int cin0, int cin1, int cout,
                           const float *src0, const float *src1, const float *w, const float *dz, float *out)
{
    const int prec = train_prec(precision);
    if (prec < 0) return WUNET_EINVAL;
    if (train_debug_conv(pass, prec, mode, ksize, B, L, cin0, cin1, cout, src0, src1, w, dz, out))
        return fail(WUNET_EINVAL, "%s", train_error());
    return WUNET_OK;
}

int wunet_debug_train_layout(int n_layers, int channels_interval, int B, int T, int precision, int block, long long *fields,
                             int capacity)
{
    if (n_layers < 1 || n_layers > 16 || channels_interval < 1 || B < 1 || T < 1 || (T % (1 << n_layers)) != 0)
        return fail(WUNET_EINVAL, "bad training layout query");
    const int prec = train_prec(precision);
    if (prec < 0) return WUNET_EINVAL;
    if (train_debug_layout(n_layers, channels_interval, B, T, prec, block, fields, capacity))
        return fail(WUNET_EINVAL, "%s", train_error());
    return WUNET_OK;
}

int wunet_debug_train_dz_scale(float amax) { return dz_scale_exp(amax); }

int wunet_debug_plan(int n_layers, int channels_interval, int B, int T, int block, int num_sms, int *fields, int capacity)
{
    return wunet_debug_plan_prec(n_layers, channels_interval, B, T, block, num_sms, fields, capacity, WUNET_PREC_BF16);
}

// the blocks of a plan query: the channel plan of wunet_create (model/unet_basic.py:38-39, :52-57, :59-62), no weights
static std::vector<TcBlockSrc> plan_query_blocks(int n, int ci)
{
    std::vector<TcBlockSrc> src;
    for (int i = 0; i < n; ++i) src.push_back(TcBlockSrc{i == 0 ? 1 : i * ci, (i + 1) * ci, 15, nullptr, nullptr, nullptr});
    src.push_back(TcBlockSrc{n * ci, n * ci, 15, nullptr, nullptr, nullptr});
    for (int j = 0; j < n; ++j)
        src.push_back(TcBlockSrc{j == 0 ? 2 * n * ci : (2 * (n - j) + 1) * ci, (n - j) * ci, 5, nullptr, nullptr, nullptr});
    return src;
}

int wunet_debug_plan_prec(int n_layers, int channels_interval, int B, int T, int block, int num_sms, int *fields, int capacity,
                          int precision)
{
    if (n_layers < 1 || n_layers > 16 || channels_interval < 1 || B < 1 || T < 1 || (T % (1 << n_layers)) != 0 || num_sms < 1)
        return fail(WUNET_EINVAL, "bad plan query");
    if (tc_mode(precision) < 0) return fail(WUNET_EINVAL, "only the tensor-core precisions (bf16, fp32_tc, fp16) have a tiling plan");
    const std::vector<TcBlockSrc> src = plan_query_blocks(n_layers, channels_interval);
    if (tc_debug_plan(n_layers, channels_interval, src.data(), (int)src.size(), B, T, block, num_sms, fields, capacity, tc_mode(precision)))
        return fail(WUNET_EINVAL, "%s", tc_error());
    return WUNET_OK;
}

int wunet_debug_plan_m2(int n_layers, int channels_interval, int B, int T, int block, int num_sms, int *fields, int capacity,
                        int precision)
{
    if (n_layers < 1 || n_layers > 16 || channels_interval < 1 || B < 1 || T < 1 || (T % (1 << n_layers)) != 0 || num_sms < 1)
        return fail(WUNET_EINVAL, "bad plan query");
    if (tc_mode(precision) < 0) return fail(WUNET_EINVAL, "only the tensor-core precisions (bf16, fp32_tc, fp16) have a tiling plan");
    const std::vector<TcBlockSrc> src = plan_query_blocks(n_layers, channels_interval);
    if (tc_debug_plan_m2(n_layers, channels_interval, src.data(), (int)src.size(), B, T, block, num_sms, fields, capacity, tc_mode(precision)))
        return fail(WUNET_EINVAL, "%s", tc_error());
    return WUNET_OK;
}

int wunet_debug_pair_weights(const float *w, int cout, int cin0, int cin1, int ksize, int decoder, float *out)
{
    if (tc_debug_pair_weights(w, cout, cin0, cin1, ksize, decoder, out)) return fail(WUNET_EINVAL, "%s", tc_error());
    return WUNET_OK;
}

int wunet_profile_enable(wunet_ctx *c, int enable)
{
    if (!c) return fail(WUNET_EINVAL, "null context");
    c->profile = enable != 0;
    c->ev_recorded = 0;
    return WUNET_OK;
}

int wunet_profile_read(wunet_ctx *c, float *ms, int capacity, int *count)
{
    if (!c || !ms || !count) return fail(WUNET_EINVAL, "null argument");
    if (c->ev_recorded < 2) return fail(WUNET_ESTATE, "no profiled forward recorded (call wunet_profile_enable, then wunet_forward)");
    const int nseg = c->ev_recorded - 1;
    if (capacity < nseg) return fail(WUNET_EINVAL, "capacity %d < %d", capacity, nseg);
    CUDA_TRY(cudaSetDevice(c->device));
    CUDA_TRY(cudaEventSynchronize(c->ev[c->ev_recorded - 1]));
    for (int i = 0; i < nseg; ++i) CUDA_TRY(cudaEventElapsedTime(&ms[i], c->ev[i], c->ev[i + 1]));
    *count = nseg;
    return WUNET_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------------------
// host-side data path (SURVEY §8f row N4): clips <-> zero-padded 16384-sample frames, the loop bodies of
// enhancement.py:57-62 / :68-71 for many clips at once, on several host threads (the single-threaded numpy copies of the
// Python shim were what bounded enhance_waveforms at ~26 k frames/s per process, a fifth of the device rate)
// ---------------------------------------------------------------------------------------------------------------------------
namespace {

struct FrameJob {
    const void *const *clips; const long long *len; int nclips; int SL; long long total; float scale;
    std::vector<long long> first;        // first frame of clip i; first[nclips] = frames used
};

inline int build_job(FrameJob &j)
{
    j.first.resize((size_t)j.nclips + 1);
    long long f = 0;
    for (int i = 0; i < j.nclips; ++i) {
        if (j.len[i] < 0 || (j.len[i] > 0 && !j.clips[i])) return -1;
        j.first[i] = f;
        f += std::max<long long>(1, (j.len[i] + j.SL - 1) / j.SL);     // an empty clip still takes one (silent) frame
    }
    j.first[j.nclips] = f;
    return f <= j.total ? 0 : -2;
}

template <class Fn> void run_threads(long long nitems, int nthreads, Fn fn)
{
    if (nthreads < 1) nthreads = 1;
    if (nthreads > 64) nthreads = 64;
    if ((long long)nthreads > nitems) nthreads = (int)std::max<long long>(1, nitems);
    if (nthreads == 1) { fn(0, nitems); return; }
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; ++t)
        th.emplace_back([=]() { fn(nitems * t / nthreads, nitems * (t + 1) / nthreads); });
    for (auto &x : th) x.join();
}

// O: element type of the frames (float, __half, __nv_bfloat16); each sample is computed in fp32 and rounded once to O
template <class O> inline O frame_cvt(float v) { return v; }
template <> inline __half frame_cvt<__half>(float v) { return __float2half_rn(v); }
template <> inline __nv_bfloat16 frame_cvt<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <class T, class O = float> int frame_clips(FrameJob &j, O *frames, int nthreads)
{
    if (!frames || j.SL <= 0 || j.nclips < 0 || j.total < 0 || (j.nclips > 0 && (!j.clips || !j.len))) return fail(WUNET_EINVAL, "frame_clips: bad argument");
    const int rc = build_job(j);
    if (rc == -1) return fail(WUNET_EINVAL, "frame_clips: negative length or null clip");
    if (rc == -2) return fail(WUNET_EINVAL, "frame_clips: %lld frames needed, room for %lld", j.first[j.nclips], j.total);
    const FrameJob *jp = &j;
    run_threads(j.total, nthreads, [jp, frames](long long f0, long long f1) {
        const FrameJob &q = *jp;
        int ci = (int)(std::upper_bound(q.first.begin(), q.first.end(), f0) - q.first.begin()) - 1;   // clip holding frame f0
        for (long long f = f0; f < f1; ++f) {
            O *dst = frames + f * q.SL;
            if (f >= q.first[q.nclips]) { std::memset(dst, 0, sizeof(O) * q.SL); continue; }         // silent frames behind the clips
            while (f >= q.first[ci + 1]) ++ci;
            const long long off = (f - q.first[ci]) * q.SL;
            const long long n = std::max<long long>(0, std::min<long long>(q.SL, q.len[ci] - off));
            const T *src = static_cast<const T *>(q.clips[ci]) + off;
            if (sizeof(T) == sizeof(float) && sizeof(O) == sizeof(float)) std::memcpy(dst, src, sizeof(float) * n);
            else if (sizeof(T) == sizeof(float)) for (long long k = 0; k < n; ++k) dst[k] = frame_cvt<O>((float)src[k]);
            else for (long long k = 0; k < n; ++k) dst[k] = frame_cvt<O>((float)src[k] * q.scale);
            if (n < q.SL) std::memset(dst + n, 0, sizeof(O) * (q.SL - n));                            // enhancement.py:58 padding
        }
    });
    return WUNET_OK;
}

}  // namespace

extern "C" {

int wunet_frame_clips_f32(const float *const *clips, const long long *lengths, int nclips, int sample_length, float *frames,
                          long long total_frames, int nthreads)
{
    FrameJob j{reinterpret_cast<const void *const *>(clips), lengths, nclips, sample_length, total_frames, 1.f, {}};
    return frame_clips<float>(j, frames, nthreads);
}

int wunet_frame_clips_i16(const int16_t *const *clips, const long long *lengths, int nclips, int sample_length, float *frames,
                          long long total_frames, int nthreads)
{
    FrameJob j{reinterpret_cast<const void *const *>(clips), lengths, nclips, sample_length, total_frames, 1.f / 32768.f, {}};
    return frame_clips<int16_t>(j, frames, nthreads);
}

int wunet_frame_clips_f32_io(const float *const *clips, const long long *lengths, int nclips, int sample_length, void *frames,
                             long long total_frames, int nthreads, int io)
{
    if (check_io(io) != WUNET_OK) return WUNET_EINVAL;
    FrameJob j{reinterpret_cast<const void *const *>(clips), lengths, nclips, sample_length, total_frames, 1.f, {}};
    if (io == WUNET_IO_F16) return frame_clips<float>(j, static_cast<__half *>(frames), nthreads);
    if (io == WUNET_IO_BF16) return frame_clips<float>(j, static_cast<__nv_bfloat16 *>(frames), nthreads);
    return frame_clips<float>(j, static_cast<float *>(frames), nthreads);
}

int wunet_frame_clips_i16_io(const int16_t *const *clips, const long long *lengths, int nclips, int sample_length, void *frames,
                             long long total_frames, int nthreads, int io)
{
    if (check_io(io) != WUNET_OK) return WUNET_EINVAL;
    FrameJob j{reinterpret_cast<const void *const *>(clips), lengths, nclips, sample_length, total_frames, 1.f / 32768.f, {}};
    if (io == WUNET_IO_F16) return frame_clips<int16_t>(j, static_cast<__half *>(frames), nthreads);
    if (io == WUNET_IO_BF16) return frame_clips<int16_t>(j, static_cast<__nv_bfloat16 *>(frames), nthreads);
    return frame_clips<int16_t>(j, static_cast<float *>(frames), nthreads);
}

int wunet_unframe_clips_f32(const float *frames, float *const *clips_out, const long long *lengths, int nclips, int sample_length,
                            long long total_frames, int nthreads)
{
    if (!frames || sample_length <= 0 || nclips < 0 || (nclips > 0 && (!clips_out || !lengths))) return fail(WUNET_EINVAL, "unframe_clips: bad argument");
    FrameJob j{reinterpret_cast<const void *const *>(clips_out), lengths, nclips, sample_length, total_frames, 1.f, {}};
    const int rc = build_job(j);
    if (rc == -1) return fail(WUNET_EINVAL, "unframe_clips: negative length or null clip");
    if (rc == -2) return fail(WUNET_EINVAL, "unframe_clips: %lld frames needed, %lld given", j.first[j.nclips], j.total);
    const FrameJob *jp = &j;
    run_threads(j.first[nclips], nthreads, [jp, frames, clips_out](long long f0, long long f1) {
        const FrameJob &q = *jp;
        int ci = (int)(std::upper_bound(q.first.begin(), q.first.end(), f0) - q.first.begin()) - 1;
        for (long long f = f0; f < f1; ++f) {
            while (f >= q.first[ci + 1]) ++ci;
            const long long off = (f - q.first[ci]) * q.SL;
            const long long n = std::max<long long>(0, std::min<long long>(q.SL, q.len[ci] - off));   // the trim of enhancement.py:69
            if (n > 0) std::memcpy(clips_out[ci] + off, frames + f * q.SL, sizeof(float) * n);
        }
    });
    return WUNET_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------------------
// training-side data path (SURVEY §8f row N4): what dataset/waveform_dataset.py:56-67 does per item - decode two wav files
// (librosa.load(path, sr=None): soundfile's float32 conversion, channels averaged) and cut the same random window out of
// both (util/utils.py:101-113) - as a wav reader plus a batched, multi-threaded crop straight into the (pinned) batch tensors.
// ---------------------------------------------------------------------------------------------------------------------------
namespace {

struct WavInfo { int fmt = 0, channels = 0, rate = 0, bits = 0; long long frames = 0, data_off = 0; };

inline uint32_t rd_u32(const unsigned char *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
inline uint16_t rd_u16(const unsigned char *p) { return (uint16_t)(p[0] | (p[1] << 8)); }

// RIFF/WAVE chunk walk: "fmt " (PCM = 1, IEEE float = 3, WAVE_FORMAT_EXTENSIBLE = 0xFFFE with the sub-format's first two bytes)
// and "data". Returns 0, or a negative code: -1 cannot open, -2 not a RIFF/WAVE file, -3 unsupported sample format.
int wav_parse(FILE *f, WavInfo &w)
{
    unsigned char h[12];
    if (fread(h, 1, 12, f) != 12 || memcmp(h, "RIFF", 4) != 0 || memcmp(h + 8, "WAVE", 4) != 0) return -2;
    bool have_fmt = false;
    for (;;) {
        unsigned char ch[8];
        if (fread(ch, 1, 8, f) != 8) return -2;
        const uint32_t sz = rd_u32(ch + 4);
        if (memcmp(ch, "fmt ", 4) == 0) {
            unsigned char b[40] = {0};
            const size_t n = sz < 40 ? sz : 40;
            if (n < 16 || fread(b, 1, n, f) != n) return -2;
            w.fmt = rd_u16(b); w.channels = rd_u16(b + 2); w.rate = (int)rd_u32(b + 4); w.bits = rd_u16(b + 14);
            if (w.fmt == 0xFFFE && n >= 26) w.fmt = rd_u16(b + 24);
            if (sz > n) fseek(f, (long)(sz - n), SEEK_CUR);
            if (sz & 1) fseek(f, 1, SEEK_CUR);
            have_fmt = true;
        } else if (memcmp(ch, "data", 4) == 0) {
            if (!have_fmt || w.channels < 1) return -2;
            const bool ok = (w.fmt == 1 && (w.bits == 8 || w.bits == 16 || w.bits == 24 || w.bits == 32)) || (w.fmt == 3 && (w.bits == 32 || w.bits == 64));
            if (!ok) return -3;
            w.data_off = ftell(f);
            long long bytes = sz;
            fseek(f, 0, SEEK_END);
            const long long avail = ftell(f) - w.data_off;            // a streamed file may carry a wrong (0 / 0xFFFFFFFF) data size
            if (bytes > avail || bytes == 0) bytes = avail;
            w.frames = bytes / ((long long)w.channels * (w.bits / 8));
            return 0;
        } else {
            if (fseek(f, (long)(sz + (sz & 1)), SEEK_CUR) != 0) return -2;
        }
    }
}

// one sample -> float32 the way libsndfile does for sf_read_float (librosa.load -> soundfile.read(dtype=float32)): integer PCM
// scaled by 2^-(bits-1) (8-bit wav is unsigned), float passed through
inline float wav_sample(const unsigned char *p, int fmt, int bits)
{
    if (fmt == 3) {
        if (bits == 32) { float v; memcpy(&v, p, 4); return v; }
        double d; memcpy(&d, p, 8); return (float)d;
    }
    switch (bits) {
    case 8: return (float)((int)p[0] - 128) * (1.f / 128.f);
    case 16: return (float)(int16_t)rd_u16(p) * (1.f / 32768.f);
    case 24: { int32_t v = (int32_t)((uint32_t)p[0] << 8 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 24); return (float)(v >> 8) * (1.f / 8388608.f); }
    default: return (float)(int32_t)rd_u32(p) * (1.f / 2147483648.f);
    }
}

}  // namespace

extern "C" {

int wunet_wav_info(const char *path, int *sample_rate, int *channels, long long *frames, int *bits, int *is_float)
{
    if (!path) return fail(WUNET_EINVAL, "wav_info: null path");
    FILE *f = fopen(path, "rb");
    if (!f) return fail(WUNET_EINVAL, "wav_info: cannot open %s", path);
    WavInfo w;
    const int rc = wav_parse(f, w);
    fclose(f);
    if (rc == -3) return fail(WUNET_EINVAL, "wav_info: %s: unsupported sample format (tag %d, %d bits)", path, w.fmt, w.bits);
    if (rc != 0) return fail(WUNET_EINVAL, "wav_info: %s is not a RIFF/WAVE file", path);
    if (sample_rate) *sample_rate = w.rate;
    if (channels) *channels = w.channels;
    if (frames) *frames = w.frames;
    if (bits) *bits = w.bits;
    if (is_float) *is_float = w.fmt == 3;
    return WUNET_OK;
}

int wunet_wav_read_f32(const char *path, long long first_frame, long long nframes, float *out)
{
    if (!path || !out || first_frame < 0 || nframes < 0) return fail(WUNET_EINVAL, "wav_read: bad argument");
    FILE *f = fopen(path, "rb");
    if (!f) return fail(WUNET_EINVAL, "wav_read: cannot open %s", path);
    WavInfo w;
    const int rc = wav_parse(f, w);
    if (rc != 0) { fclose(f); return fail(WUNET_EINVAL, "wav_read: %s: %s", path, rc == -3 ? "unsupported sample format" : "not a RIFF/WAVE file"); }
    if (first_frame + nframes > w.frames) { fclose(f); return fail(WUNET_EINVAL, "wav_read: %s has %lld frames, [%lld, %lld) wanted", path, w.frames, first_frame, first_frame + nframes); }
    const int bs = w.bits / 8, fb = bs * w.channels;
    std::vector<unsigned char> buf((size_t)std::min<long long>(nframes, 1 << 16) * fb);
    fseek(f, (long)(w.data_off + first_frame * fb), SEEK_SET);
    const float inv = 1.f / (float)w.channels;
    for (long long done = 0; done < nframes;) {
        const long long n = std::min<long long>(nframes - done, 1 << 16);
        if ((long long)fread(buf.data(), (size_t)fb, (size_t)n, f) != n) { fclose(f); return fail(WUNET_EINVAL, "wav_read: %s is truncated", path); }
        for (long long i = 0; i < n; ++i) {
            const unsigned char *p = buf.data() + i * fb;
            if (w.channels == 1) { out[done + i] = wav_sample(p, w.fmt, w.bits); continue; }
            float s = 0.f;                                          // librosa.to_mono: np.mean over the channel axis (float32)
            for (int c = 0; c < w.channels; ++c) s += wav_sample(p + c * bs, w.fmt, w.bits);
            out[done + i] = s * inv;
        }
        done += n;
    }
    fclose(f);
    return WUNET_OK;
}

int wunet_crop_pairs(const void *const *mixture, const void *const *clean, const long long *lengths, const long long *starts, int nitems,
                     int sample_length, int is_i16, float *mixture_out, float *clean_out, int nthreads)
{
    if (nitems < 0 || sample_length <= 0 || (nitems > 0 && (!mixture || !clean || !lengths || !starts || !mixture_out || !clean_out)))
        return fail(WUNET_EINVAL, "crop_pairs: bad argument");
    for (int i = 0; i < nitems; ++i) {
        // util/utils.py:104-105: both signals have the same length, at least sample_length; start in [0, len - sample_length]
        if (!mixture[i] || !clean[i]) return fail(WUNET_EINVAL, "crop_pairs: null clip %d", i);
        if (lengths[i] < sample_length) return fail(WUNET_EINVAL, "crop_pairs: item %d has %lld samples, sample_length is %d", i, lengths[i], sample_length);
        if (starts[i] < 0 || starts[i] + sample_length > lengths[i]) return fail(WUNET_EINVAL, "crop_pairs: item %d: start %lld outside [0, %lld]", i, starts[i], lengths[i] - sample_length);
    }
    const long long SL = sample_length;
    run_threads(2LL * nitems, nthreads, [=](long long j0, long long j1) {
        for (long long j = j0; j < j1; ++j) {
            const int i = (int)(j >> 1);
            const void *src = (j & 1) ? clean[i] : mixture[i];
            float *dst = ((j & 1) ? clean_out : mixture_out) + i * SL;
            if (!is_i16) std::memcpy(dst, static_cast<const float *>(src) + starts[i], sizeof(float) * SL);
            else {
                const int16_t *s = static_cast<const int16_t *>(src) + starts[i];
                for (long long k = 0; k < SL; ++k) dst[k] = (float)s[k] * (1.f / 32768.f);
            }
        }
    });
    return WUNET_OK;
}

}  // extern "C"
