// C-ABI of the fused joiner (include/rnnt.h, DESIGN.md §14) and of the pruned fused joiner (§15): workspace sizing,
// argument rules and the chunk loop, shared by both; the pruned calls run the same loop over N T R window rows.  The
// _drop entries (§16) are the same calls with dropout on h; the entries without it are them with p = 0.
// A translation unit of its own, so the kernels of rnnt_entry.cu compile exactly as they did without it.
#include <cuda_runtime.h>

#include <atomic>
#include <climits>
#include <cmath>
#include <cstdint>

#include "../../include/rnnt.h"
#include "rnnt_joiner.cuh"

using namespace b200joiner;

namespace {

thread_local int g_joiner_launches = 0;

constexpr size_t kAlign = 256;
constexpr size_t kScratchCap = size_t(256) << 20;   // the default chunk keeps its scratch at or below 256 MiB
constexpr int kSMs = 132;                             // an H100 SXM
constexpr int kSlabTarget = 2 * kSMs;                 // dW tiles x slabs: two CTAs per SM
constexpr int kMaxSlabs = 16;
constexpr int kMaxRows = 128;                         // rows of the largest logits tile: the scratch's row granule

// Rows per CTA of the logits kernels: 128 (8 warps) while the 128 h rows fit in shared memory beside the W stages
// with room to spare, 64 (4 warps) above H = 640.
int logits_rows(int hidden) { return hidden <= 640 ? 128 : 64; }

size_t up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Everything the entries derive from the extents: strides, chunk and workspace layout.
struct Plan {
    int N, T, U, H, V, Hp, Vp, cells, chunk, slabs;
    size_t lse, denc, dpred, dw, h, dlog, ds, bytes;   // byte offsets; bytes = total
};

bool extents_ok(int maxT, int maxU, int minibatch, int hidden, int alphabet_size, int chunk_cells) {
    if (maxT < 1 || maxU < 1 || minibatch < 1 || maxU > 1024) return false;
    if ((long long)minibatch * maxT * maxU >= (1LL << 31)) return false;
    if (hidden < 16 || hidden > 1024 || hidden % 16 != 0) return false;
    if (alphabet_size < 2 || alphabet_size > INT_MAX - TILE) return false;
    return chunk_cells >= 0;
}

// The pruned rules beyond extents_ok: a window of s_range >= 1 rows per frame and N T R < 2^31.
bool window_ok(int maxT, int minibatch, int s_range) {
    return s_range >= 1 && (long long)minibatch * maxT * s_range < (1LL << 31);
}

// rows_per_frame: maxU for the dense grid (b, u, t), s_range for the pruned rows (b, r, t).
Plan plan(int maxT, int maxU, int minibatch, int hidden, int alphabet_size, int chunk_cells, int rows_per_frame) {
    Plan p;
    p.N = minibatch, p.T = maxT, p.U = maxU, p.H = hidden, p.V = alphabet_size;
    p.Hp = (int)up(hidden + 1, TILE);           // column H of h is the constant 1 of dbias
    p.Vp = (int)up(alphabet_size, TILE);
    p.cells = minibatch * maxT * rows_per_frame;
    const size_t row = (size_t)p.Hp * 2 + (size_t)p.Vp * 2 + (size_t)p.H * 4;   // h, dlogits, ds
    if (chunk_cells == 0) {   // whole waves of 128-row CTAs where the cap allows
        const size_t wave = (size_t)kMaxRows * kSMs;
        size_t fit = kScratchCap / row;
        fit = fit >= wave ? fit / wave * wave : fit / kMaxRows * kMaxRows;
        chunk_cells = (int)(fit < kMaxRows ? kMaxRows : (fit > (size_t)INT_MAX / 2 ? INT_MAX / 2 : fit));
    }
    p.chunk = chunk_cells < p.cells ? chunk_cells : p.cells;
    const size_t rows = up(p.chunk, kMaxRows);
    const int tiles = (p.Vp / TILE) * (p.Hp / TILE);
    p.slabs = (kSlabTarget + tiles - 1) / tiles;
    if (p.slabs > kMaxSlabs) p.slabs = kMaxSlabs;
    if (p.slabs > (int)(rows / TILE)) p.slabs = (int)(rows / TILE);
    size_t o = 0;
    p.lse = o, o = up(o + (size_t)p.cells * 4, kAlign);
    p.denc = o, o = up(o + (size_t)p.N * p.T * p.H * 4, kAlign);
    p.dpred = o, o = up(o + (size_t)p.N * p.U * p.H * 4, kAlign);
    p.dw = o, o = up(o + (size_t)p.slabs * p.Vp * p.Hp * 4, kAlign);
    p.h = o, o = up(o + rows * p.Hp * 2, kAlign);
    p.dlog = o, o = up(o + rows * p.Vp * 2, kAlign);
    p.ds = o, o = up(o + rows * p.H * 4, kAlign);
    p.bytes = o;
    return p;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// The rules shared by forward and backward; the pointers each half needs beyond these are checked by it.
rnntStatus_t check_common(int activation, const void* enc, const void* pred, const void* weight, const void* bias,
                          const int* flat_labels, const int* label_lengths, const int* input_lengths, int hidden,
                          int alphabet_size, int minibatch, int chunk_cells, const void* workspace,
                          const rnntOptions& o) {
    if (activation != RNNT_B200_ACT_TANH && activation != RNNT_B200_ACT_RELU) return RNNT_STATUS_INVALID_VALUE;
    if (!extents_ok(o.maxT, o.maxU, minibatch, hidden, alphabet_size, chunk_cells)) return RNNT_STATUS_INVALID_VALUE;
    if (o.blank_label < 0 || o.blank_label >= alphabet_size) return RNNT_STATUS_INVALID_VALUE;
    if (!enc || !pred || !weight || !label_lengths || !input_lengths || !workspace) return RNNT_STATUS_INVALID_VALUE;
    if (!flat_labels && o.maxU > 1) return RNNT_STATUS_INVALID_VALUE;
    if (!aligned16(enc) || !aligned16(pred) || !aligned16(weight) || !aligned16(workspace))
        return RNNT_STATUS_INVALID_VALUE;
    if (bias && (reinterpret_cast<uintptr_t>(bias) & 1)) return RNNT_STATUS_INVALID_VALUE;
    return RNNT_STATUS_SUCCESS;
}

Geo geo(const Plan& p, int blank, const int* flat_labels, const int* label_lengths, const int* input_lengths) {
    Geo g;
    g.N = p.N, g.T = p.T, g.U = p.U, g.S = p.U - 1, g.H = p.H, g.V = p.V, g.Hp = p.Hp, g.Vp = p.Vp;
    g.c0 = 0, g.m = 0, g.blank = blank;
    g.xlen = input_lengths, g.ylen = label_lengths, g.labels = flat_labels;
    return g;
}

size_t logits_smem(int hidden) {
    return ((size_t)(hidden + TILE - 1) / TILE * (logits_rows(hidden) / TILE) + STAGES) * TILE_ELEMS * 2;
}
constexpr size_t kPairSmem = (size_t)2 * PAIR_STAGES * TILE_ELEMS * 2;

template <bool PRUNED>
bool allow_smem(cudaFuncAttribute attr, int big, int small) {
    return cudaFuncSetAttribute(joiner_lse_kernel<128, PRUNED>, attr, big) == cudaSuccess &&
           cudaFuncSetAttribute(joiner_dlogits_kernel<128, PRUNED>, attr, big) == cudaSuccess &&
           cudaFuncSetAttribute(joiner_lse_kernel<64, PRUNED>, attr, small) == cudaSuccess &&
           cudaFuncSetAttribute(joiner_dlogits_kernel<64, PRUNED>, attr, small) == cudaSuccess &&
           cudaFuncSetAttribute(joiner_ds_kernel<PRUNED>, attr, (int)kPairSmem) == cudaSuccess &&
           cudaFuncSetAttribute(joiner_ds_kernel<PRUNED, true>, attr, (int)kPairSmem) == cudaSuccess;
}

// The dynamic shared-memory opt-in of every kernel, dense and pruned, for the largest call, once per device: after
// one call on a device, calls made during CUDA-graph capture make no attribute calls.
bool allow_smem() {
    constexpr int kMaxDevices = 64;
    static std::atomic<bool> done[kMaxDevices];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return false;
    if (dev < kMaxDevices && done[dev].load()) return true;
    const auto attr = cudaFuncAttributeMaxDynamicSharedMemorySize;
    const int big = (int)logits_smem(640), small = (int)logits_smem(1024);   // the largest of each tile height
    const bool ok = allow_smem<false>(attr, big, small) && allow_smem<true>(attr, big, small) &&
                    cudaFuncSetAttribute(joiner_dw_kernel, attr, (int)kPairSmem) == cudaSuccess;
    if (ok && dev < kMaxDevices) done[dev].store(true);
    return ok;
}

int blocks(long long n, int threads) {
    const long long b = (n + threads - 1) / threads;
    return (int)(b < 1 ? 1 : (b > (1LL << 20) ? (1LL << 20) : b));
}

rnntStatus_t launched() {
    return cudaGetLastError() == cudaSuccess ? RNNT_STATUS_SUCCESS : RNNT_STATUS_EXECUTION_FAILED;
}

template <bool PRUNED>
void launch_h(const Geo& g, int act, const bf16* enc, const bf16* pred, bf16* h, int rows, cudaStream_t s,
              const Window& w, const Drop& d) {
    const int nb = blocks((long long)rows * (g.Hp / 8), 256);
    if (d.seed)
        joiner_h_kernel<PRUNED, true><<<nb, 256, 0, s>>>(g, act, enc, pred, h, rows, w, d);
    else
        joiner_h_kernel<PRUNED><<<nb, 256, 0, s>>>(g, act, enc, pred, h, rows, w);
    ++g_joiner_launches;
}

// The forward chunk loop of both entries (pruned: after filling px and py with -inf).
template <bool PRUNED>
rnntStatus_t forward(int activation, const void* enc, const void* pred, const void* weight, const void* bias,
                     const int* flat_labels, const int* label_lengths, const int* input_lengths, int hidden,
                     int alphabet_size, int minibatch, int chunk_cells, float* px, float* py, void* workspace,
                     const rnntOptions& options, const Window& w, const Drop& d) {
    const Plan p = plan(options.maxT, options.maxU, minibatch, hidden, alphabet_size, chunk_cells,
                        PRUNED ? w.R : options.maxU);
    char* ws = static_cast<char*>(workspace);
    float* lse = reinterpret_cast<float*>(ws + p.lse);
    bf16* h = reinterpret_cast<bf16*>(ws + p.h);
    cudaStream_t s = options.stream;
    const size_t smem = logits_smem(hidden);
    const int bm = logits_rows(hidden);
    if (!allow_smem()) return RNNT_STATUS_EXECUTION_FAILED;
    Geo g = geo(p, options.blank_label, flat_labels, label_lengths, input_lengths);
    const bf16* W = static_cast<const bf16*>(weight);
    const bf16* B = static_cast<const bf16*>(bias);
    if (PRUNED) {
        const long long npx = (long long)p.N * (p.U - 1) * p.T, npy = (long long)p.N * p.U * p.T;
        joiner_fill_kernel<<<blocks(npx + npy, 256), 256, 0, s>>>(px, npx, py, npy);
        ++g_joiner_launches;
    }
    for (int c0 = 0; c0 < p.cells; c0 += p.chunk) {
        g.c0 = c0;
        g.m = p.cells - c0 < p.chunk ? p.cells - c0 : p.chunk;
        const int tiles = (g.m + bm - 1) / bm;
        launch_h<PRUNED>(g, activation, static_cast<const bf16*>(enc), static_cast<const bf16*>(pred), h, tiles * bm,
                         s, w, d);
        if (bm == 128)
            joiner_lse_kernel<128, PRUNED><<<tiles, 256, smem, s>>>(g, h, W, B, lse, px, py, w);
        else
            joiner_lse_kernel<64, PRUNED><<<tiles, 128, smem, s>>>(g, h, W, B, lse, px, py, w);
        ++g_joiner_launches;
    }
    return launched();
}

// The backward chunk loop of both entries.
template <bool PRUNED>
rnntStatus_t backward(int activation, const void* enc, const void* pred, const void* weight, const void* bias,
                      const int* flat_labels, const int* label_lengths, const int* input_lengths, int hidden,
                      int alphabet_size, int minibatch, int chunk_cells, const float* dpx, const float* dpy,
                      void* grad_enc, void* grad_pred, void* grad_weight, void* grad_bias, void* workspace,
                      const rnntOptions& options, const Window& w, const Drop& d) {
    const Plan p = plan(options.maxT, options.maxU, minibatch, hidden, alphabet_size, chunk_cells,
                        PRUNED ? w.R : options.maxU);
    char* ws = static_cast<char*>(workspace);
    const float* lse = reinterpret_cast<const float*>(ws + p.lse);
    float* denc = reinterpret_cast<float*>(ws + p.denc);
    float* dpred = reinterpret_cast<float*>(ws + p.dpred);
    float* dw = reinterpret_cast<float*>(ws + p.dw);
    bf16* h = reinterpret_cast<bf16*>(ws + p.h);
    bf16* dlog = reinterpret_cast<bf16*>(ws + p.dlog);
    float* ds = reinterpret_cast<float*>(ws + p.ds);
    const bf16* W = static_cast<const bf16*>(weight);
    cudaStream_t s = options.stream;
    const size_t smem = logits_smem(hidden);
    const int bm = logits_rows(hidden);
    if (!allow_smem()) return RNNT_STATUS_EXECUTION_FAILED;
    // the fp32 accumulators (denc, dpred, dW slabs) are contiguous in the workspace
    if (cudaMemsetAsync(ws + p.denc, 0, p.h - p.denc, s) != cudaSuccess) return RNNT_STATUS_EXECUTION_FAILED;

    Geo g = geo(p, options.blank_label, flat_labels, label_lengths, input_lengths);
    const int per_b = PRUNED ? w.R : p.U;   // grid rows of T cells per utterance
    for (int c0 = 0; c0 < p.cells; c0 += p.chunk) {
        g.c0 = c0;
        g.m = p.cells - c0 < p.chunk ? p.cells - c0 : p.chunk;
        const int ltiles = (g.m + bm - 1) / bm, tiles = (g.m + TILE - 1) / TILE;
        launch_h<PRUNED>(g, activation, static_cast<const bf16*>(enc), static_cast<const bf16*>(pred), h,
                         ltiles * bm, s, w, d);
        if (bm == 128)
            joiner_dlogits_kernel<128, PRUNED><<<ltiles, 256, smem, s>>>(g, h, W, static_cast<const bf16*>(bias), lse,
                                                                         dpx, dpy, dlog, w);
        else
            joiner_dlogits_kernel<64, PRUNED><<<ltiles, 128, smem, s>>>(g, h, W, static_cast<const bf16*>(bias), lse,
                                                                        dpx, dpy, dlog, w);
        const dim3 ds_grid(tiles, (p.H + TILE - 1) / TILE);
        if (d.seed)
            joiner_ds_kernel<PRUNED, true><<<ds_grid, THREADS, kPairSmem, s>>>(
                g, activation, dlog, W, h, ds, w, d, static_cast<const bf16*>(enc), static_cast<const bf16*>(pred));
        else
            joiner_ds_kernel<PRUNED><<<ds_grid, THREADS, kPairSmem, s>>>(g, activation, dlog, W, h, ds, w);
        const int bu_lo = c0 / p.T, bu_hi = (c0 + g.m - 1) / p.T;
        const long long b_n = bu_hi / per_b - bu_lo / per_b + 1;
        // dense: one thread per (b, u) row and per (b, t) of the chunk; pruned: per (b, u) and (b, t) of its b
        const long long red = (PRUNED ? b_n * p.U : (long long)(bu_hi - bu_lo + 1)) * p.H + b_n * p.T * p.H;
        joiner_reduce_kernel<PRUNED><<<blocks(red, 256), 256, 0, s>>>(g, ds, denc, dpred, w);
        const int per = (tiles + p.slabs - 1) / p.slabs;
        joiner_dw_kernel<<<dim3(p.Vp / TILE, p.Hp / TILE, (tiles + per - 1) / per), THREADS, kPairSmem, s>>>(
            g, dlog, h, dw, tiles, per);
        g_joiner_launches += 4;
    }
    const long long n = (long long)p.V * p.H + p.V + (long long)p.N * p.T * p.H + (long long)p.N * p.U * p.H;
    joiner_round_kernel<<<blocks(n, 256), 256, 0, s>>>(g, p.slabs, dw, denc, dpred, static_cast<bf16*>(grad_weight),
                                                       static_cast<bf16*>(grad_bias), static_cast<bf16*>(grad_enc),
                                                       static_cast<bf16*>(grad_pred));
    ++g_joiner_launches;
    return launched();
}

// The dropout rules of the _drop entries: 0 <= p < 1 (NaN fails), a seed when p > 0, 8-byte aligned when given.
bool dropout_ok(const rnntJoinerDropout& o) {
    if (!(o.p >= 0.f && o.p < 1.f)) return false;
    if (o.p > 0.f && !o.seed) return false;
    return (reinterpret_cast<uintptr_t>(o.seed) & 7) == 0;
}

// The kernels' descriptor: no seed (the DROP = false kernels) when p == 0.
Drop drop(const rnntJoinerDropout& o) {
    if (!(o.p > 0.f)) return Drop{nullptr, 0u, 1.f};
    return Drop{o.seed, (uint32_t)floor((double)o.p * 4294967296.0), (float)(1.0 / (1.0 - (double)o.p))};
}

const rnntJoinerDropout kNoDropout = {0.f, nullptr};

}  // namespace

extern "C" {

rnntStatus_t rnnt_b200_joiner_workspace_size(int maxT, int maxU, int minibatch, int hidden, int alphabet_size,
                                             int chunk_cells, size_t* size_bytes) {
    if (!size_bytes || !extents_ok(maxT, maxU, minibatch, hidden, alphabet_size, chunk_cells))
        return RNNT_STATUS_INVALID_VALUE;
    *size_bytes = plan(maxT, maxU, minibatch, hidden, alphabet_size, chunk_cells, maxU).bytes;
    return RNNT_STATUS_SUCCESS;
}

rnntStatus_t rnnt_b200_joiner_forward(int activation, const void* enc, const void* pred, const void* weight,
                                      const void* bias, const int* flat_labels, const int* label_lengths,
                                      const int* input_lengths, int hidden, int alphabet_size, int minibatch,
                                      int chunk_cells, float* px, float* py, void* workspace,
                                      struct rnntOptions options) {
    return rnnt_b200_joiner_forward_drop(activation, enc, pred, weight, bias, flat_labels, label_lengths,
                                         input_lengths, hidden, alphabet_size, minibatch, chunk_cells, px, py,
                                         kNoDropout, workspace, options);
}

rnntStatus_t rnnt_b200_joiner_backward(int activation, const void* enc, const void* pred, const void* weight,
                                       const void* bias, const int* flat_labels, const int* label_lengths,
                                       const int* input_lengths, int hidden, int alphabet_size, int minibatch,
                                       int chunk_cells, const float* dpx, const float* dpy, void* grad_enc,
                                       void* grad_pred, void* grad_weight, void* grad_bias, void* workspace,
                                       struct rnntOptions options) {
    return rnnt_b200_joiner_backward_drop(activation, enc, pred, weight, bias, flat_labels, label_lengths,
                                          input_lengths, hidden, alphabet_size, minibatch, chunk_cells, dpx, dpy,
                                          grad_enc, grad_pred, grad_weight, grad_bias, kNoDropout, workspace, options);
}

rnntStatus_t rnnt_b200_joiner_forward_drop(int activation, const void* enc, const void* pred, const void* weight,
                                           const void* bias, const int* flat_labels, const int* label_lengths,
                                           const int* input_lengths, int hidden, int alphabet_size, int minibatch,
                                           int chunk_cells, float* px, float* py, struct rnntJoinerDropout dropout,
                                           void* workspace, struct rnntOptions options) {
    g_joiner_launches = 0;
    rnntStatus_t st = check_common(activation, enc, pred, weight, bias, flat_labels, label_lengths, input_lengths,
                                   hidden, alphabet_size, minibatch, chunk_cells, workspace, options);
    if (st != RNNT_STATUS_SUCCESS) return st;
    if (!dropout_ok(dropout)) return RNNT_STATUS_INVALID_VALUE;
    if (!py || (!px && options.maxU > 1)) return RNNT_STATUS_INVALID_VALUE;
    if (options.loc != RNNT_GPU) return RNNT_STATUS_EXECUTION_FAILED;
    return forward<false>(activation, enc, pred, weight, bias, flat_labels, label_lengths, input_lengths, hidden,
                          alphabet_size, minibatch, chunk_cells, px, py, workspace, options, Window{nullptr, 0},
                          drop(dropout));
}

rnntStatus_t rnnt_b200_joiner_backward_drop(int activation, const void* enc, const void* pred, const void* weight,
                                            const void* bias, const int* flat_labels, const int* label_lengths,
                                            const int* input_lengths, int hidden, int alphabet_size, int minibatch,
                                            int chunk_cells, const float* dpx, const float* dpy, void* grad_enc,
                                            void* grad_pred, void* grad_weight, void* grad_bias,
                                            struct rnntJoinerDropout dropout, void* workspace,
                                            struct rnntOptions options) {
    g_joiner_launches = 0;
    rnntStatus_t st = check_common(activation, enc, pred, weight, bias, flat_labels, label_lengths, input_lengths,
                                   hidden, alphabet_size, minibatch, chunk_cells, workspace, options);
    if (st != RNNT_STATUS_SUCCESS) return st;
    if (!dropout_ok(dropout)) return RNNT_STATUS_INVALID_VALUE;
    if (!dpy || (!dpx && options.maxU > 1) || !grad_enc || !grad_pred || !grad_weight)
        return RNNT_STATUS_INVALID_VALUE;
    if (options.loc != RNNT_GPU) return RNNT_STATUS_EXECUTION_FAILED;
    return backward<false>(activation, enc, pred, weight, bias, flat_labels, label_lengths, input_lengths, hidden,
                           alphabet_size, minibatch, chunk_cells, dpx, dpy, grad_enc, grad_pred, grad_weight,
                           grad_bias, workspace, options, Window{nullptr, 0}, drop(dropout));
}

rnntStatus_t rnnt_b200_pruned_joiner_workspace_size(int maxT, int maxU, int s_range, int minibatch, int hidden,
                                                    int alphabet_size, int chunk_cells, size_t* size_bytes) {
    if (!size_bytes || !extents_ok(maxT, maxU, minibatch, hidden, alphabet_size, chunk_cells) ||
        !window_ok(maxT, minibatch, s_range))
        return RNNT_STATUS_INVALID_VALUE;
    *size_bytes = plan(maxT, maxU, minibatch, hidden, alphabet_size, chunk_cells, s_range).bytes;
    return RNNT_STATUS_SUCCESS;
}

rnntStatus_t rnnt_b200_pruned_joiner_forward(int activation, const void* enc, const void* pred, const void* weight,
                                             const void* bias, const int* flat_labels, const int* label_lengths,
                                             const int* input_lengths, const int* ranges, int s_range, int hidden,
                                             int alphabet_size, int minibatch, int chunk_cells, float* px, float* py,
                                             void* workspace, struct rnntOptions options) {
    return rnnt_b200_pruned_joiner_forward_drop(activation, enc, pred, weight, bias, flat_labels, label_lengths,
                                                input_lengths, ranges, s_range, hidden, alphabet_size, minibatch,
                                                chunk_cells, px, py, kNoDropout, workspace, options);
}

rnntStatus_t rnnt_b200_pruned_joiner_backward(int activation, const void* enc, const void* pred, const void* weight,
                                              const void* bias, const int* flat_labels, const int* label_lengths,
                                              const int* input_lengths, const int* ranges, int s_range, int hidden,
                                              int alphabet_size, int minibatch, int chunk_cells, const float* dpx,
                                              const float* dpy, void* grad_enc, void* grad_pred, void* grad_weight,
                                              void* grad_bias, void* workspace, struct rnntOptions options) {
    return rnnt_b200_pruned_joiner_backward_drop(activation, enc, pred, weight, bias, flat_labels, label_lengths,
                                                 input_lengths, ranges, s_range, hidden, alphabet_size, minibatch,
                                                 chunk_cells, dpx, dpy, grad_enc, grad_pred, grad_weight, grad_bias,
                                                 kNoDropout, workspace, options);
}

rnntStatus_t rnnt_b200_pruned_joiner_forward_drop(int activation, const void* enc, const void* pred,
                                                  const void* weight, const void* bias, const int* flat_labels,
                                                  const int* label_lengths, const int* input_lengths,
                                                  const int* ranges, int s_range, int hidden, int alphabet_size,
                                                  int minibatch, int chunk_cells, float* px, float* py,
                                                  struct rnntJoinerDropout dropout, void* workspace,
                                                  struct rnntOptions options) {
    g_joiner_launches = 0;
    rnntStatus_t st = check_common(activation, enc, pred, weight, bias, flat_labels, label_lengths, input_lengths,
                                   hidden, alphabet_size, minibatch, chunk_cells, workspace, options);
    if (st != RNNT_STATUS_SUCCESS) return st;
    if (!dropout_ok(dropout)) return RNNT_STATUS_INVALID_VALUE;
    if (!ranges || !window_ok(options.maxT, minibatch, s_range)) return RNNT_STATUS_INVALID_VALUE;
    if (!py || (!px && options.maxU > 1)) return RNNT_STATUS_INVALID_VALUE;
    if (options.loc != RNNT_GPU) return RNNT_STATUS_EXECUTION_FAILED;
    return forward<true>(activation, enc, pred, weight, bias, flat_labels, label_lengths, input_lengths, hidden,
                         alphabet_size, minibatch, chunk_cells, px, py, workspace, options, Window{ranges, s_range},
                         drop(dropout));
}

rnntStatus_t rnnt_b200_pruned_joiner_backward_drop(int activation, const void* enc, const void* pred,
                                                   const void* weight, const void* bias, const int* flat_labels,
                                                   const int* label_lengths, const int* input_lengths,
                                                   const int* ranges, int s_range, int hidden, int alphabet_size,
                                                   int minibatch, int chunk_cells, const float* dpx,
                                                   const float* dpy, void* grad_enc, void* grad_pred,
                                                   void* grad_weight, void* grad_bias,
                                                   struct rnntJoinerDropout dropout, void* workspace,
                                                   struct rnntOptions options) {
    g_joiner_launches = 0;
    rnntStatus_t st = check_common(activation, enc, pred, weight, bias, flat_labels, label_lengths, input_lengths,
                                   hidden, alphabet_size, minibatch, chunk_cells, workspace, options);
    if (st != RNNT_STATUS_SUCCESS) return st;
    if (!dropout_ok(dropout)) return RNNT_STATUS_INVALID_VALUE;
    if (!ranges || !window_ok(options.maxT, minibatch, s_range)) return RNNT_STATUS_INVALID_VALUE;
    if (!dpy || (!dpx && options.maxU > 1) || !grad_enc || !grad_pred || !grad_weight)
        return RNNT_STATUS_INVALID_VALUE;
    if (options.loc != RNNT_GPU) return RNNT_STATUS_EXECUTION_FAILED;
    return backward<true>(activation, enc, pred, weight, bias, flat_labels, label_lengths, input_lengths, hidden,
                          alphabet_size, minibatch, chunk_cells, dpx, dpy, grad_enc, grad_pred, grad_weight,
                          grad_bias, workspace, options, Window{ranges, s_range}, drop(dropout));
}

int rnnt_b200_joiner_last_launch_count(void) { return g_joiner_launches; }

}  // extern "C"
