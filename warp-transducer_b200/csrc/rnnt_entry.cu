// rnnt_entry.cu — C-ABI of libwarprnnt.so (declared in include/rnnt.h) and the host-side
// orchestration of the three kernels.  Replaces reference src/rnnt_entrypoint.cpp and
// include/detail/gpu_rnnt.h (GpuRNNT<T>::compute_cost_and_score) for loc == RNNT_GPU.
//
// Per call, on options.stream:  [stage host labels/lengths if needed] -> rowstats -> lattice
// (alpha || beta) -> grad -> costs to host + ONE stream synchronise (sync API) / nothing (async API).
// No memset pass, no intermediate host synchronisation.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/rnnt.h"
#include "rnnt_chunk.cuh"
#include "rnnt_joint.cuh"
#include "rnnt_kernels.cuh"
#include "rnnt_lattice.cuh"
#include "rnnt_lattice_io.cuh"
#include "rnnt_viterbi.cuh"

using namespace b200rnnt;

namespace {

thread_local int g_last_launches = 0;

// Tuning hooks (README), read from the environment once per process.  A value outside a hook's accepted set
// leaves the default policy in place; the code that uses a hook checks its range.
int env_int(const char* name, int fallback) {
    const char* e = getenv(name);
    return e ? atoi(e) : fallback;
}
struct Hooks {
    int lpr = env_int("RNNT_B200_LPR", 0);                    // lanes per row of the register-tile kernels
    bool chunk = env_int("RNNT_B200_CHUNK", 1) != 0;          // 0: short rows go to the register-tile kernels
    int chunk_map = env_int("RNNT_B200_CHUNK_MAP", -1);       // 0 | 1: lane mapping of the chunk kernels
    int chunk_nt = env_int("RNNT_B200_CHUNK_NT", 0);          // 64 | 128 | 256: threads per fp32 chunk CTA
    int chunk_tpr = env_int("RNNT_B200_CHUNK_TPR", 0);        // 1 | 2 | 4 | 8: lanes per row of the chunk kernels
    uint32_t chunk_wait_ns = (uint32_t)env_int("RNNT_B200_CHUNK_WAIT_NS", 2000);   // chunk kernels' staging back-off
    bool pdl = env_int("RNNT_B200_PDL", 0) != 0;              // programmatic dependent launch (experimental), see run()
    int groups = env_int("RNNT_B200_GROUPS", 0);              // batch groups of the lattice overlap
    bool timeline = env_int("RNNT_B200_TIMELINE", 0) != 0;    // per-launch timeline of the grouped schedule
    int lat_ring = env_int("RNNT_B200_LAT_RING", 0);          // 8 | 16 | 32: factor ring of the multi-warp wavefront
    int joint_slices = env_int("RNNT_B200_JOINT_SLICES", 0);  // split-K slabs of the additive joint's S product
    bool joint_simt = env_int("RNNT_B200_JOINT_SIMT", 0) != 0;     // SIMT joint contractions instead of wgmma
    bool joint_fused = env_int("RNNT_B200_JOINT_FUSED", 1) != 0;   // 0: two-kernel dF / dG, not the fused kernel
    int df_tile = env_int("RNNT_B200_DF_TILE", 64);           // accumulator tile width cap of the two-kernel dF
    size_t fused_pad_smem = (size_t)env_int("RNNT_B200_FUSED_PAD_SMEM", 0);   // fused kernel: residency experiments
};
const Hooks& hooks() {
    static const Hooks h;
    return h;
}

// Optional per-kernel timing (bench.py's roofline leg): when enabled, events are recorded on the
// call's own stream around each of the three kernels, one event set per call (pooled), so a timed
// loop needs no host synchronisation; rnnt_b200_profile_collect() averages them afterwards.
struct EventSet {
    cudaEvent_t e[4] = {nullptr, nullptr, nullptr, nullptr};
    bool valid[4] = {false, false, false, false};
};
thread_local bool g_profile = false;
thread_local std::vector<EventSet> g_sets;
thread_local size_t g_used = 0;   // sets recorded since the last collect
inline void profile_begin_call() {
    if (!g_profile) return;
    if (g_used == g_sets.size()) g_sets.emplace_back();
    EventSet& es = g_sets[g_used++];
    for (int i = 0; i < 4; ++i) es.valid[i] = false;
}
inline void mark(int i, cudaStream_t s) {
    if (!g_profile || g_used == 0) return;
    EventSet& es = g_sets[g_used - 1];
    if (!es.e[i]) cudaEventCreate(&es.e[i]);
    es.valid[i] = cudaEventRecord(es.e[i], s) == cudaSuccess;
}
// ms of {rowstats, lattice, grad} for one recorded call; false where not measured
inline int read_set(EventSet& es, float* ms3) {
    int n = 0;
    for (int i = 0; i < 3; ++i) {
        ms3[i] = -1.0f;
        if (es.valid[i] && es.valid[i + 1] && cudaEventSynchronize(es.e[i + 1]) == cudaSuccess &&
            cudaEventElapsedTime(&ms3[i], es.e[i], es.e[i + 1]) == cudaSuccess)
            ++n;
    }
    return n;
}

// Dev aid, RNNT_B200_TIMELINE=1: timed events around every launch of the grouped (overlapped) schedule,
// printed to stderr relative to the call's start.  Synchronises the call; never on in production.
struct Timeline {
    std::vector<std::pair<std::string, cudaEvent_t>> ev;
    bool on = false;
    void tick(const char* what, int k, cudaStream_t s) {
        if (!on) return;
        cudaEvent_t e;
        cudaEventCreate(&e);
        cudaEventRecord(e, s);
        ev.emplace_back(std::string(what) + std::to_string(k), e);
    }
    void dump() {
        if (!on || ev.empty()) return;
        cudaDeviceSynchronize();
        for (auto& p : ev) {
            float ms = 0;
            cudaEventElapsedTime(&ms, ev[0].second, p.second);
            fprintf(stderr, "[timeline] %-14s %8.3f ms\n", p.first.c_str(), ms);
        }
        for (auto& p : ev) cudaEventDestroy(p.second);
        ev.clear();
    }
};

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Launch `kernel`; with pdl it may start while the previous kernel of the stream is still running (its
// CTAs block in griddepcontrol.wait until that kernel has completed and its writes are visible).
template <typename... KArgs, typename... Args>
void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, bool pdl, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kernel, KArgs(std::forward<Args>(args))...);
}

// cudaFuncSetAttribute once per (kernel, attribute, device) and host thread (again only for a larger value).  Keyed by the kernel's
// address: template instantiations with identical signatures share a function-pointer TYPE, so a static
// flag inside a generic lambda would be shared between them.
void func_attr_once(const void* kernel, cudaFuncAttribute attr, int value) {
    struct Key { const void* k; int attr, dev, value; };
    thread_local std::vector<Key> done;
    int dev = 0;
    cudaGetDevice(&dev);
    for (Key& e : done)
        if (e.k == kernel && e.attr == (int)attr && e.dev == dev) {
            if (value > e.value) {   // e.g. a larger dynamic shared-memory request than any before
                cudaFuncSetAttribute(kernel, attr, value);
                e.value = value;
            }
            return;
        }
    cudaFuncSetAttribute(kernel, attr, value);
    done.push_back(Key{kernel, (int)attr, dev, value});
}

// Side streams for overlapping the (latency-bound, few-SM) lattice kernel of one group of
// utterances with the (bandwidth-bound) streaming passes of the others.  High priority so the
// lattice CTAs are placed as soon as short-lived streaming CTAs retire.  Fork/join with events on
// the caller's stream only, so the call stays capturable and stream-ordered for the caller.
constexpr int kMaxGroups = 8;    // upper bound (RNNT_B200_GROUPS)
constexpr int kAutoGroups = 4;   // what the overlap heuristic picks
struct SidePool {
    cudaStream_t stream[kMaxGroups] = {};
    cudaEvent_t forked[kMaxGroups] = {};
    cudaEvent_t joined[kMaxGroups] = {};
    int device = -1;
    bool ok = false;
};
SidePool& side_pool() {
    // one pool per (host thread, device): a thread that alternates devices finds its pools again instead
    // of re-creating (and leaking) streams and events on every switch
    constexpr int kMaxDevices = 64;
    thread_local SidePool pools[kMaxDevices];
    int dev = 0;
    cudaGetDevice(&dev);
    SidePool& pool = pools[dev >= 0 && dev < kMaxDevices ? dev : 0];
    if (pool.device != dev) {
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        pool.ok = true;
        for (int g = 0; g < kMaxGroups; ++g) {
            pool.ok &= cudaStreamCreateWithPriority(&pool.stream[g], cudaStreamNonBlocking, hi) == cudaSuccess;
            pool.ok &= cudaEventCreateWithFlags(&pool.forked[g], cudaEventDisableTiming) == cudaSuccess;
            pool.ok &= cudaEventCreateWithFlags(&pool.joined[g], cudaEventDisableTiming) == cudaSuccess;
        }
        pool.device = dev;
    }
    return pool;
}

// ---- workspace carve-up (all sections 256-B aligned) -------------------------------------------
// Bump allocator over a caller's workspace; with a NULL base it only counts the bytes.
struct Carver {
    char* base;
    size_t off;
    explicit Carver(void* b)
        : base(static_cast<char*>(b)),
          off(align_up(reinterpret_cast<uintptr_t>(b), 256) - reinterpret_cast<uintptr_t>(b)) {}
    template <typename P = void> P* take(size_t n) {
        void* q = base ? base + off : nullptr;
        off = align_up(off + n, 256);
        return static_cast<P*>(q);
    }
};

struct Workspace {
    void* stat;     // pair<T>  [rows]   (row max, log sum exp)
    void* lp2;      // Lat<T>::fac [lat]  per-cell transition factors (16 B), diagonal-major
    void* alphas;   // Lat<T>::val [lat]  lat = N*(maxT+maxU-1)*maxU   (8 B: LogVal for fp32 - cell-major, using N*maxT*maxU
                    //                    of the entries -, double for fp64 - diagonal-major)
    void* betas;    // Lat<T>::val [lat]
    void* llf;      // Lat<T>::val [N]
    void* llb;      // Lat<T>::val [N]
    void* costs;    // T [N]
    int* labels;    // staging for host-side integer inputs
    int* ylen;
    int* xlen;
    size_t bytes;
};

Workspace carve(void* base, size_t rows, size_t lat, int N, int maxU, size_t dtype) {
    Workspace w;
    Carver c(base);
    w.stat = c.take(rows * 2 * dtype);
    w.lp2 = c.take(lat * 16);
    w.alphas = c.take(lat * 8);
    w.betas = c.take(lat * 8);
    w.llf = c.take((size_t)N * 8);
    w.llb = c.take((size_t)N * 8);
    w.costs = c.take(N * dtype);
    w.labels = c.take<int>((size_t)N * (maxU > 1 ? maxU - 1 : 1) * sizeof(int));
    w.ylen = c.take<int>(N * sizeof(int));
    w.xlen = c.take<int>(N * sizeof(int));
    // slack: a base pointer that is not 256-aligned, plus the speculative lattice reads one diagonal past
    // the last utterance (row_grad_setup_spec: at most (maxU + 1) * 8 bytes beyond `betas`)
    w.bytes = c.off + 256 + 16 * 1024;
    return w;
}

struct DeviceInfo {
    int sms = 0;
};
const DeviceInfo& device_info() {
    thread_local int cached_dev = -1;
    thread_local DeviceInfo info;
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev != cached_dev) {
        cudaDeviceGetAttribute(&info.sms, cudaDevAttrMultiProcessorCount, dev);
        cached_dev = dev;
    }
    return info;
}

bool is_device_pointer(const void* p) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

// gradient options (include/rnnt.h rnntGradOptions): validity, on/off, and the kernels' form of them
inline bool grad_options_valid(const rnntGradOptions& o) {
    return std::isfinite(o.fastemit_lambda) && o.fastemit_lambda >= 0.0f && !std::isnan(o.clamp);
}
inline bool grad_options_on(const rnntGradOptions& o) { return o.fastemit_lambda > 0.0f || o.clamp > 0.0f; }
// smoothing scales of the additive joint (include/rnnt.h rnntSmoothOptions)
// The sum may exceed 1 by one float32 ulp of 1: scales the caller chose to sum to exactly 1, such as (0.6, 0.4),
// arrive rounded to float32 and can sum to 1 + 3e-8 (c then becomes 0).
inline bool smooth_valid(const rnntSmoothOptions& o) {
    const double l = o.lm_only_scale, a = o.am_only_scale;
    return std::isfinite(l) && std::isfinite(a) && l >= 0.0 && a >= 0.0 && l + a <= 1.0 + 0x1p-23;
}
inline bool smooth_on(const rnntSmoothOptions& o) { return o.lm_only_scale != 0.0f || o.am_only_scale != 0.0f; }
// lattice options (include/rnnt.h rnntLatticeOptions): the delay penalty (DESIGN.md §10)
inline bool lattice_valid(const rnntLatticeOptions& o) {
    return std::isfinite(o.delay_penalty) && o.delay_penalty >= 0.0f;
}
inline bool delay_on(const rnntLatticeOptions& o) { return o.delay_penalty > 0.0f; }
template <typename T> GradReg<T> make_grad_reg(const rnntGradOptions& o, const Workspace& w) {
    GradReg<T> r;
    r.lp2 = static_cast<const typename Lat<T>::fac*>(w.lp2);
    const double lam = o.fastemit_lambda;
    r.log2_lam = lam > 0.0 ? (T)std::log2(lam) : -(T)INFINITY;
    r.log2_1p_lam = (T)(std::log1p(lam) / std::log(2.0));
    r.clamp = o.clamp > 0.0f ? (T)o.clamp : (T)INFINITY;
    return r;
}

// What a call does.  The reference API is FULL (stats -> lattice -> grad in one call); the
// operator splits a training step into FORWARD (stats + both lattices, costs out) and BACKWARD
// (gradient pass only, reading the lattices the forward left in the workspace).  ALIGN is forced alignment
// (DESIGN.md §12): pass 1, then the Viterbi wavefront and its backtrace; the costs are the best paths' scores.
enum Phase { kFull = 0, kForward = 1, kBackward = 2, kAlign = 3 };

// What one compute call asks for, besides its tensors.
struct Call {
    Phase phase;
    bool async;              // costs stay on the device and nothing synchronises
    bool want_beta;          // forward: the beta lattice too, for the backward that follows
    bool tunv;               // activations / gradients [T,U,N,V] (RNNT_B200_LAYOUT_TUNV) instead of [N,T,U,V]
    double scale;            // gradient multiplier, rounded to the arithmetic type
    const void* scale_vec;   // per-utterance gradient multipliers in the arithmetic type, or NULL
    rnntGradOptions grad;
    bool pruned = false;     // logits [N,maxT,R,V] over the windows Tensors::ranges (DESIGN.md §8)
    rnntSmoothOptions smooth = {0.0f, 0.0f};   // additive joint: lm-only / am-only scales (DESIGN.md §9)
    rnntLatticeOptions lattice = {0.0f};       // delay penalty of the label factors (DESIGN.md §10)
    int rnnt_type = RNNT_B200_RNNT_REGULAR;    // lattice topology (DESIGN.md §11)
};
Call full_call(double scale, bool async = true, bool tunv = false, rnntGradOptions grad = {0.0f, 0.0f}) {
    return Call{kFull, async, false, tunv, scale, nullptr, grad};
}
Call forward_call(int prepare_backward) {
    return Call{kForward, true, prepare_backward != 0, false, 1.0, nullptr, {0.0f, 0.0f}};
}
Call backward_call(double scale, const void* grad_costs, rnntGradOptions grad = {0.0f, 0.0f}) {
    return Call{kBackward, true, false, false, scale, grad_costs, grad};
}
Call align_call(bool tunv, int rnnt_type) {
    Call c{kAlign, true, false, tunv, 1.0, nullptr, {0.0f, 0.0f}};
    c.rnnt_type = rnnt_type;
    return c;
}

// The tensors and extents of a call, in the order the C-ABI entries take them.  For the additive joint, acts
// and grads are the transcription factor and its gradient.
struct Tensors {
    const void* acts;
    void* grads;   // NULL: loss only
    const int *labels, *ylen, *xlen;
    int V, N;
    void* costs;   // arithmetic type; NULL in the backward phase
    void* workspace;
    rnntOptions opt;
    const int* ranges = nullptr;   // pruned calls: [N, maxT] window starts
    int s_range = 0;               // pruned calls: R, rows per frame
    int* frames = nullptr;         // alignment calls: [N, maxU-1] label frames (NULL allowed when maxU == 1)
};

// The checks of every compute call, all before any device access; the first that fails decides the status.
rnntStatus_t check_call(const Tensors& t, const Call& c) {
    const rnntOptions& opt = t.opt;
    if (!grad_options_valid(c.grad) || !smooth_valid(c.smooth) || !lattice_valid(c.lattice) ||
        (c.rnnt_type != RNNT_B200_RNNT_REGULAR && c.rnnt_type != RNNT_B200_RNNT_MODIFIED))
        return RNNT_STATUS_INVALID_VALUE;
    if (!t.acts || !t.labels || !t.ylen || !t.xlen || (!t.costs && c.phase != kBackward) || !t.workspace ||
        t.V <= 0 || t.N <= 0 || opt.maxT <= 0 || opt.maxU <= 0 || (c.phase == kBackward && !t.grads))
        return RNNT_STATUS_INVALID_VALUE;  // reference src/rnnt_entrypoint.cpp:49-59
    if (c.phase == kAlign && (t.grads || (!t.frames && opt.maxU > 1))) return RNNT_STATUS_INVALID_VALUE;
    // pruned rows are counted with 32 bits like the dense ones; the pruned kernels index [N,maxT,R,V] only
    if (c.pruned && (!t.ranges || t.s_range < 1 || c.tunv || (uint64_t)t.N * opt.maxT * t.s_range >= (1ull << 31)))
        return RNNT_STATUS_INVALID_VALUE;
    if (opt.loc == RNNT_CPU) {
        fprintf(stderr, "b200-rnnt: CPU execution requested, but this library is the CUDA path only\n");
        return RNNT_STATUS_EXECUTION_FAILED;
    }
    if (opt.loc != RNNT_GPU) return RNNT_STATUS_INVALID_VALUE;  // :90-92
    if ((uint64_t)t.N * opt.maxT * opt.maxU >= (1ull << 31) || opt.blank_label < 0 || opt.blank_label >= t.V)
        return RNNT_STATUS_INVALID_VALUE;
    if (opt.maxU > 1024) {
        fprintf(stderr, "b200-rnnt: maxU > 1024 is not supported (the reference launches maxU threads per block and has the same limit)\n");
        return RNNT_STATUS_INVALID_VALUE;
    }
    return RNNT_STATUS_SUCCESS;
}

Dims make_dims(const Tensors& t, bool tmajor) {
    Dims d;
    d.N = t.N;
    d.maxT = t.opt.maxT;
    d.maxU = t.opt.maxU;
    d.V = t.V;
    d.blank = t.opt.blank_label;
    d.rows = (uint32_t)((uint64_t)t.N * t.opt.maxT * t.opt.maxU);
    d.divU = FastDiv(t.opt.maxU);
    d.divT = FastDiv(t.opt.maxT);
    d.divN = FastDiv(t.N);
    d.tmajor = tmajor ? 1 : 0;
    return d;
}

// One batch group of a call, and how its kernels launch.  Utterances are independent and every array is
// batch-major, so a group is the same problem on offset pointers; one group is the whole batch.
template <typename T, typename IO>
struct Group {
    Workspace w;
    Dims d;
    const IO* acts;
    IO* grads;
    const int *labels, *xlen, *ylen;
    T* costs;
    T scale;
    const T* scale_vec;
    bool reg;            // gradient options on: the REG gradient kernels, given `gr`
    GradReg<T> gr;
    cudaStream_t s;      // the call's stream (the grouped schedule runs each lattice on a side stream)
    bool pdl;            // launch the dependent kernels with programmatic stream serialization
    bool pruned;         // the PRUNED streaming kernels, given `pr` (the dense ones get ranges == NULL)
    Prune pr;
    bool delay;          // delay penalty on: the *_delay_kernel twins, given `pen` (pass 1) and `pen_log2` (pass 2)
    T pen;               // lambda
    T pen_log2;          // lambda log2(e)
    bool mod;            // modified topology: the *_mod_kernel gradient kernels (DESIGN.md §11)
    bool scaled() const { return scale != T(1) || scale_vec; }
};

// Calls f with one std::integral_constant<bool, ...> per flag, in order: each kernel choice becomes a template
// argument in one place, and the launch sites below name every streaming kernel once.
template <typename F> void with_flags(F&& f) { f(); }
template <typename F, typename... Flags> void with_flags(F&& f, bool first, Flags... rest) {
    if (first) with_flags([&](auto... c) { f(std::true_type{}, c...); }, rest...);
    else with_flags([&](auto... c) { f(std::false_type{}, c...); }, rest...);
}

// ---- streaming-kernel dispatch on (vector width, row length) -------------------------------------
// Long rows: one CTA per row (grid = rows).  Short rows: register tiles, 32/LPR rows per warp.
// Both grids are non-persistent on purpose (see rnnt_kernels.cuh).  Pass 1 is the log-softmax
// statistics and (blank, label) factors, pass 2 the gradient.
template <typename T, int VEC, int NV, typename IO>
void launch_row(const Group<T, IO>& g, int pass) {
    using Val = const typename Lat<T>::val*;
    with_flags([&](auto scaled, auto reg, auto pruned, auto delay) {
        constexpr bool SCALED = decltype(scaled)::value, REG = decltype(reg)::value, PRUNED = decltype(pruned)::value;
        constexpr bool DELAY = decltype(delay)::value;
        auto* stat = static_cast<typename Real<T>::pair*>(g.w.stat);
        auto* lp2 = static_cast<typename Lat<T>::fac*>(g.w.lp2);
        const dim3 grid(g.d.rows), block(RowThreads<IO>::value);
        if (pass == 1 && DELAY)
            rowstats_row_delay_kernel<T, VEC, NV, IO, PRUNED><<<grid, block, 0, g.s>>>(
                g.acts, g.labels, g.xlen, g.ylen, stat, lp2, g.d, g.pr, g.pen);
        else if (pass == 1)
            rowstats_row_kernel<T, VEC, NV, IO, PRUNED><<<grid, block, 0, g.s>>>(
                g.acts, g.labels, g.xlen, g.ylen, stat, lp2, g.d, g.pr);
        else if (g.mod)
            launch_k(grad_row_mod_kernel<T, VEC, NV, IO, PRUNED>, grid, block, 0, g.s, g.pdl, g.acts,
                     g.grads, g.labels, g.xlen, g.ylen, stat, static_cast<Val>(g.w.alphas), static_cast<Val>(g.w.betas),
                     static_cast<Val>(g.w.llf), g.scale, g.scale_vec, g.d, g.gr, g.pr, g.pen_log2);
        else if (DELAY)
            launch_k(grad_row_delay_kernel<T, VEC, NV, SCALED, IO, REG, PRUNED>, grid, block, 0, g.s, g.pdl, g.acts,
                     g.grads, g.labels, g.xlen, g.ylen, stat, static_cast<Val>(g.w.alphas), static_cast<Val>(g.w.betas),
                     static_cast<Val>(g.w.llf), g.scale, g.scale_vec, g.d, g.gr, g.pr, g.pen_log2);
        else
            launch_k(grad_row_kernel<T, VEC, NV, SCALED, IO, REG, PRUNED>, grid, block, 0, g.s, g.pdl, g.acts,
                     g.grads, g.labels, g.xlen, g.ylen, stat, static_cast<Val>(g.w.alphas), static_cast<Val>(g.w.betas),
                     static_cast<Val>(g.w.llf), g.scale, g.scale_vec, g.d, g.gr, g.pr);
    }, g.scaled(), g.reg, g.pruned, g.delay);
    ++g_last_launches;
}

template <typename T, int VEC, int LPR, typename IO>
void launch_tile(const Group<T, IO>& g, int pass) {
    using Val = const typename Lat<T>::val*;
    const uint64_t warps = ((uint64_t)g.d.rows * LPR + 31) / 32;
    const unsigned grid = (unsigned)((warps + 7) / 8);
    with_flags([&](auto scaled, auto reg, auto pruned, auto delay) {
        constexpr bool SCALED = decltype(scaled)::value, REG = decltype(reg)::value, PRUNED = decltype(pruned)::value;
        constexpr bool DELAY = decltype(delay)::value;
        auto* stat = static_cast<typename Real<T>::pair*>(g.w.stat);
        auto* lp2 = static_cast<typename Lat<T>::fac*>(g.w.lp2);
        if (pass == 1 && DELAY)
            rowstats_tile_delay_kernel<T, VEC, LPR, IO, PRUNED><<<grid, 256, 0, g.s>>>(
                g.acts, g.labels, g.xlen, g.ylen, stat, lp2, g.d, g.pr, g.pen);
        else if (pass == 1)
            rowstats_tile_kernel<T, VEC, LPR, IO, PRUNED><<<grid, 256, 0, g.s>>>(
                g.acts, g.labels, g.xlen, g.ylen, stat, lp2, g.d, g.pr);
        else if (g.mod)
            launch_k(grad_tile_mod_kernel<T, VEC, LPR, IO, PRUNED>, dim3(grid), dim3(256), 0, g.s,
                     g.pdl, g.acts, g.grads, g.labels, g.xlen, g.ylen, stat, static_cast<Val>(g.w.alphas),
                     static_cast<Val>(g.w.betas), static_cast<Val>(g.w.llf), g.scale, g.scale_vec, g.d, g.gr, g.pr,
                     g.pen_log2);
        else if (DELAY)
            launch_k(grad_tile_delay_kernel<T, VEC, LPR, SCALED, IO, REG, PRUNED>, dim3(grid), dim3(256), 0, g.s,
                     g.pdl, g.acts, g.grads, g.labels, g.xlen, g.ylen, stat, static_cast<Val>(g.w.alphas),
                     static_cast<Val>(g.w.betas), static_cast<Val>(g.w.llf), g.scale, g.scale_vec, g.d, g.gr, g.pr,
                     g.pen_log2);
        else
            launch_k(grad_tile_kernel<T, VEC, LPR, SCALED, IO, REG, PRUNED>, dim3(grid), dim3(256), 0, g.s, g.pdl,
                     g.acts, g.grads, g.labels, g.xlen, g.ylen, stat, static_cast<Val>(g.w.alphas),
                     static_cast<Val>(g.w.betas), static_cast<Val>(g.w.llf), g.scale, g.scale_vec, g.d, g.gr, g.pr);
    }, g.scaled(), g.reg, g.pruned, g.delay);
    ++g_last_launches;
}

// lanes per row for the register-tile kernels: the fewest lanes (>= 2) whose kVPL = 8 vector
// registers hold the row: V=28 -> 2 lanes, V=50 (float2) -> 4 lanes per row
inline int pick_lpr(int nv) {
    const int forced = hooks().lpr;
    int lpr = 2;
    while (lpr < 32 && lpr * kVPL < nv) lpr *= 2;
    if (forced >= 1 && forced <= 32 && (forced & (forced - 1)) == 0 && forced * kVPL >= nv) lpr = forced;
    return lpr;
}

template <typename T, int VEC, typename IO>
void stream_passes(const Group<T, IO>& g, int pass) {
    const int nv = g.d.V / VEC;
    if (nv > 32 * kVPL) {  // long rows: CTA per row; NV = vectors per thread per trip
        const int per_thread = (nv + RowThreads<IO>::value - 1) / RowThreads<IO>::value;
        if (sizeof(IO) <= 4 && VEC == 16 / (int)sizeof(IO)) {  // 16-B fast paths get an exact register count
            switch (per_thread) {
                case 1: return launch_row<T, VEC, 1, IO>(g, pass);
                case 2: return launch_row<T, VEC, 2, IO>(g, pass);
                case 3: return launch_row<T, VEC, 3, IO>(g, pass);
                case 4: return launch_row<T, VEC, 4, IO>(g, pass);
                case 5: return launch_row<T, VEC, 5, IO>(g, pass);
                case 6: return launch_row<T, VEC, 6, IO>(g, pass);
                default: return launch_row<T, VEC, 8, IO>(g, pass);
            }
        }
        if (per_thread <= 2) launch_row<T, VEC, 2, IO>(g, pass);
        else if (per_thread <= 4) launch_row<T, VEC, 4, IO>(g, pass);
        else launch_row<T, VEC, 8, IO>(g, pass);
        return;
    }
    switch (pick_lpr(nv)) {
        case 2: return launch_tile<T, VEC, 2, IO>(g, pass);
        case 4: return launch_tile<T, VEC, 4, IO>(g, pass);
        case 8: return launch_tile<T, VEC, 8, IO>(g, pass);
        case 16: return launch_tile<T, VEC, 16, IO>(g, pass);
        case 32: return launch_tile<T, VEC, 32, IO>(g, pass);
    }
}

// ---- short rows (<= 512 B): chunk kernels (rnnt_chunk.cuh), TMA bulk staging of R consecutive rows ----
// Threads per row: as FEW as keep a thread's share at <= 32 elements (two for even V, so that the walk can use
// 8-byte pairs) - every lane of a row repeats the row's fixed work (mapping, shuffles, reductions), and at
// V = 28 that fixed work dominates, so fewer lanes per row win.  Bank
// conflicts are dealt with by the lane mapping (chunk_walk_cost), not by the lane count.
// RNNT_B200_CHUNK=0 routes short rows to the register-tile kernels.
inline int pick_tpr(int V) {
    int tpr = 1;
    while (tpr < 32 && V > 32 * tpr) tpr *= 2;
    if (tpr == 1 && V % 2 == 0 && V > 16) tpr = 2;
    return tpr;
}
// Shared-memory wavefronts of one warp-wide access of the chunk kernels' element walk under either
// lane -> (row, slice) mapping (ChunkMap in rnnt_chunk.cuh).  A warp's access is served in phases of
// 128 bytes' worth of lanes; within a phase lanes that fall on the same bank group serialise.
inline int chunk_walk_cost(int V, int tpr, int elt, bool hmajor) {
    const int unit = V % 2 == 0 ? 2 * elt : elt;   // bytes per lane access (pairs for even V)
    const int per_phase = 128 / unit;
    const int rpw = 32 / tpr;
    int cost = 0;
    for (int p0 = 0; p0 < 32; p0 += per_phase) {
        int cnt[32] = {0}, worst = 0;
        for (int l = p0; l < p0 + per_phase; ++l) {
            const int il = hmajor ? l % rpw : l / tpr, h = hmajor ? l / rpw : l % tpr;
            const long addr = (long)il * V * elt / unit + h;
            worst = std::max(worst, ++cnt[addr % per_phase]);
        }
        cost += worst;
    }
    return cost;
}
// lane mapping of the chunk kernels: bank-aware choice, or what RNNT_B200_CHUNK_MAP = 0 | 1 forces (tuning hook)
inline int chunk_hmajor(int V, int tpr, int elt) {
    const int forced_map = hooks().chunk_map;
    if (forced_map == 0 || forced_map == 1) return forced_map;
    return chunk_walk_cost(V, tpr, elt, true) < chunk_walk_cost(V, tpr, elt, false);
}
template <typename T>
bool chunk_pass(const Group<T, T>& g, int pass) {
    using Pair = typename Real<T>::pair;
    using Fac = typename Lat<T>::fac;
    using Val = typename Lat<T>::val;
    const Hooks& hk = hooks();
    if (!hk.chunk || (size_t)g.d.V * sizeof(T) > 512) return false;
    if (reinterpret_cast<uintptr_t>(g.acts) % 16 || (pass == 2 && reinterpret_cast<uintptr_t>(g.grads) % 16)) return false;
    // threads per chunk CTA (tuning hook RNNT_B200_CHUNK_NT): fp64 always 128
    int nt = sizeof(T) >= 8 ? 128 : 256;
    if (sizeof(T) == 4 && (hk.chunk_nt == 64 || hk.chunk_nt == 128 || hk.chunk_nt == 256)) nt = hk.chunk_nt;
    int tpr = pick_tpr(g.d.V);
    if (hk.chunk_tpr == 1 || hk.chunk_tpr == 2 || hk.chunk_tpr == 4 || hk.chunk_tpr == 8) tpr = hk.chunk_tpr;   // tuning hook
    if (nt / tpr < 4) nt = 4 * tpr;   // a chunk is at least 4 rows (16-byte aligned chunk starts)
    const int rows_per = nt / tpr;
    const unsigned grid = (unsigned)(((uint64_t)g.d.rows + rows_per - 1) / rows_per);
    const size_t smem = (size_t)rows_per * g.d.V * sizeof(T);
    const uint32_t wait_ns = hk.chunk_wait_ns;
    const int hmajor = chunk_hmajor(g.d.V, tpr, (int)sizeof(T));
    // 8+ chunk CTAs per SM need most of the shared memory: ask for the largest carve-out once per kernel.
    // The chosen lane count keeps a chunk at <= 32 KB; a forced smaller one (CHUNK_TPR) stages more rows of the
    // same length, up to 128 KB (fp32, V = 128, one lane per row), which a launch gets only after opting in.
    auto prefer_smem = [smem](auto kernel) {
        func_attr_once(reinterpret_cast<const void*>(kernel), cudaFuncAttributePreferredSharedMemoryCarveout,
                       cudaSharedmemCarveoutMaxShared);
        if (smem > 32 * 1024)
            func_attr_once(reinterpret_cast<const void*>(kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        return kernel;
    };
    auto go = [&](auto tpr_c, auto nt_c) {
        constexpr int TPR = decltype(tpr_c)::value, NT = decltype(nt_c)::value;
        if constexpr (NT / TPR >= 4) {
            with_flags([&](auto scaled, auto reg, auto pruned, auto delay) {
                constexpr bool SCALED = decltype(scaled)::value, REG = decltype(reg)::value;
                constexpr bool PRUNED = decltype(pruned)::value, DELAY = decltype(delay)::value;
                Pair* stat = static_cast<Pair*>(g.w.stat);
                Fac* lp2 = static_cast<Fac*>(g.w.lp2);
                const Val *al = static_cast<const Val*>(g.w.alphas), *be = static_cast<const Val*>(g.w.betas);
                const Val* llf = static_cast<const Val*>(g.w.llf);
                if (pass == 1 && DELAY)
                    prefer_smem(rowstats_chunk_delay_kernel<T, TPR, NT, PRUNED>)<<<grid, NT, smem, g.s>>>(
                        g.acts, g.labels, g.xlen, g.ylen, stat, lp2, g.d, hmajor, wait_ns, g.pr, g.pen);
                else if (pass == 1)
                    prefer_smem(rowstats_chunk_kernel<T, TPR, NT, PRUNED>)<<<grid, NT, smem, g.s>>>(
                        g.acts, g.labels, g.xlen, g.ylen, stat, lp2, g.d, hmajor, wait_ns, g.pr);
                else if (g.mod)
                    launch_k(prefer_smem(grad_chunk_mod_kernel<T, TPR, NT, PRUNED>), dim3(grid),
                             dim3(NT), smem, g.s, g.pdl, g.acts, g.grads, g.labels, g.xlen, g.ylen, stat, al, be, llf,
                             g.scale, g.scale_vec, g.d, hmajor, wait_ns, g.gr, g.pr, g.pen_log2);
                else if (DELAY)
                    launch_k(prefer_smem(grad_chunk_delay_kernel<T, TPR, NT, SCALED, REG, PRUNED>), dim3(grid), dim3(NT),
                             smem, g.s, g.pdl, g.acts, g.grads, g.labels, g.xlen, g.ylen, stat, al, be, llf, g.scale,
                             g.scale_vec, g.d, hmajor, wait_ns, g.gr, g.pr, g.pen_log2);
                else
                    launch_k(prefer_smem(grad_chunk_kernel<T, TPR, NT, SCALED, REG, PRUNED>), dim3(grid), dim3(NT), smem,
                             g.s, g.pdl, g.acts, g.grads, g.labels, g.xlen, g.ylen, stat, al, be, llf, g.scale,
                             g.scale_vec, g.d, hmajor, wait_ns, g.gr, g.pr);
            }, g.scaled(), g.reg, g.pruned, g.delay);
        }
    };
    auto with_rpt = [&](auto tpr_c) {
        if constexpr (sizeof(T) >= 8) {
            go(tpr_c, std::integral_constant<int, 128>{});
        } else {
            if (nt == 64) go(tpr_c, std::integral_constant<int, 64>{});
            else if (nt == 128) go(tpr_c, std::integral_constant<int, 128>{});
            else go(tpr_c, std::integral_constant<int, 256>{});
        }
    };
    switch (tpr) {
        case 1: with_rpt(std::integral_constant<int, 1>{}); break;
        case 2: with_rpt(std::integral_constant<int, 2>{}); break;
        case 4: with_rpt(std::integral_constant<int, 4>{}); break;
        case 8: with_rpt(std::integral_constant<int, 8>{}); break;
        case 16: with_rpt(std::integral_constant<int, 16>{}); break;
        default: with_rpt(std::integral_constant<int, 32>{}); break;
    }
    ++g_last_launches;
    return true;
}

template <typename T, typename IO>
void stream_pass(const Group<T, IO>& g, int pass) {
    if constexpr (std::is_same<T, IO>::value) {
        if (chunk_pass<T>(g, pass)) return;
    }
    // widest vector the row pitch and the base pointers allow (16-B vectors on the fast path)
    const uintptr_t mis = reinterpret_cast<uintptr_t>(g.acts) | (pass == 2 ? reinterpret_cast<uintptr_t>(g.grads) : 0) |
                          ((uintptr_t)g.d.V * sizeof(IO));
    constexpr int kMaxVec = 16 / sizeof(IO);
    if (mis % 16 == 0)
        stream_passes<T, kMaxVec, IO>(g, pass);
    else if (sizeof(IO) == 4 && mis % 8 == 0)
        stream_passes<T, (sizeof(IO) == 4 ? 2 : 1), IO>(g, pass);
    else
        stream_passes<T, 1, IO>(g, pass);
}

// fp32 lattice: linear-domain wavefront with explicit exponents, COLS label columns per lane and a factor
// ring `depth` diagonals deep (rnnt_lattice.cuh); alpha, and beta in a second grid row when with_beta.
// The dense path and the additive joint share it.
// mod: the modified topology's wavefront (DESIGN.md §11).
void launch_lattice_lin(const float4* lp2, const int* xlen, const int* ylen, LogVal* alphas, LogVal* betas,
                        LogVal* llf, LogVal* llb, float* costs, const Dims& d, bool with_beta, int depth,
                        cudaStream_t s, bool pdl, bool mod = false) {
    const size_t ring = lattice_ring_bytes(d.maxU, depth);
    auto launch = [&](auto kernel, int static_smem) {
        if (ring + static_smem > 48 * 1024)
            func_attr_once(reinterpret_cast<const void*>(kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ring);
        launch_k(kernel, dim3(d.N, with_beta ? 2 : 1), dim3(lattice_threads(d.maxU)), ring, s, pdl, lp2, xlen, ylen,
                 alphas, betas, llf, llb, costs, d);
    };
    if (mod) {
        if (d.maxU <= 32) launch(lattice_lin_mod_kernel<1, false, 8>, 64);
        else if (d.maxU <= 64) launch(lattice_lin_mod_kernel<2, false, 8>, 64);
        else if (depth == 32) launch(lattice_lin_mod_kernel<1, true, 32>, kLinStaticSmem);
        else if (depth == 16) launch(lattice_lin_mod_kernel<1, true, 16>, kLinStaticSmem);
        else launch(lattice_lin_mod_kernel<1, true, 8>, kLinStaticSmem);
    } else if (d.maxU <= 32) launch(lattice_lin_kernel<1, false, 8>, 64);
    else if (d.maxU <= 64) launch(lattice_lin_kernel<2, false, 8>, 64);
    else if (depth == 32) launch(lattice_lin_kernel<1, true, 32>, kLinStaticSmem);
    else if (depth == 16) launch(lattice_lin_kernel<1, true, 16>, kLinStaticSmem);
    else launch(lattice_lin_kernel<1, true, 8>, kLinStaticSmem);
}

// fp64 lattice: log-domain wavefront (rnnt_kernels.cuh), one thread per label column; alpha, and beta in a second
// grid row when with_beta.  mod: the modified topology (DESIGN.md §11).
void launch_lattice_log(const double2* lp2, const int* xlen, const int* ylen, double* alphas, double* betas,
                        double* llf, double* llb, double* costs, const Dims& d, bool with_beta, cudaStream_t s,
                        bool pdl, bool mod) {
    const int threads = (d.maxU + 31) / 32 * 32;
    const size_t ring = (size_t)kRing * threads * sizeof(double2);
    auto launch = [&](auto kernel) {
        // opt-in when static + dynamic shared memory exceed the 48 KB default (maxU >= 353);
        // the attribute is per device and the call is rare and cheap next to such a wavefront
        if (ring + kLatticeStaticSmem > 48 * 1024)
            cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ring);
        launch_k(kernel, dim3(d.N, with_beta ? 2 : 1), dim3(threads), ring, s, pdl, lp2, xlen, ylen, alphas, betas,
                 llf, llb, costs, d);
    };
    if (mod && threads > 32) launch(lattice_mod_kernel<double, true>);
    else if (mod) launch(lattice_mod_kernel<double, false>);
    else if (threads > 32) launch(lattice_kernel<double, true>);
    else launch(lattice_kernel<double, false>);
}

// Forced alignment (rnnt_viterbi.cuh): one CTA per utterance, one thread per label column, a kRing-deep factor ring.
// The decision bits take the alphas section, which an alignment call does not otherwise use.
template <typename T>
void launch_viterbi(const void* lp2, const int* xlen, const int* ylen, void* alphas, int* frames, T* scores,
                    const Dims& d, bool mod, cudaStream_t s) {
    const int threads = viterbi_words(d.maxU) * 32;
    const size_t ring = (size_t)kRing * threads * 16;
    auto launch = [&](auto kernel, auto fac) {
        if (ring > 40 * 1024)
            func_attr_once(reinterpret_cast<const void*>(kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ring);
        kernel<<<d.N, threads, ring, s>>>(static_cast<decltype(fac)>(lp2), xlen, ylen, static_cast<uint32_t*>(alphas),
                                          frames, scores, d);
    };
    if constexpr (sizeof(T) == 4) {
        const float4* f = nullptr;
        if (mod && threads > 32) launch(viterbi_lin_mod_kernel<true>, f);
        else if (mod) launch(viterbi_lin_mod_kernel<false>, f);
        else if (threads > 32) launch(viterbi_lin_kernel<true>, f);
        else launch(viterbi_lin_kernel<false>, f);
    } else {
        const double2* f = nullptr;
        if (mod && threads > 32) launch(viterbi_mod_kernel<true>, f);
        else if (mod) launch(viterbi_mod_kernel<false>, f);
        else if (threads > 32) launch(viterbi_kernel<true>, f);
        else launch(viterbi_kernel<false>, f);
    }
}

template <typename IO>
rnntStatus_t run(const Tensors& t, const Call& c) {
    using T = typename ComputeOf<IO>::type;  // arithmetic type (float for the 16-bit storage types)
    if (const rnntStatus_t st = check_call(t, c)) return st;
    const rnntOptions& opt = t.opt;
    const int V = t.V, N = t.N;
    const IO* acts = static_cast<const IO*>(t.acts);
    IO* grads = static_cast<IO*>(t.grads);
    const int *labels = t.labels, *ylen = t.ylen, *xlen = t.xlen;
    T* costs = static_cast<T*>(t.costs);

    g_last_launches = 0;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(opt.stream);
    const int rows_u = c.pruned ? t.s_range : opt.maxU;   // logit rows per frame (stat is carved per row)
    const uint64_t rows64 = (uint64_t)N * opt.maxT * rows_u;
    const size_t lat = (size_t)N * (opt.maxT + opt.maxU - 1) * opt.maxU;
    Workspace w = carve(t.workspace, rows64, lat, N, opt.maxU, sizeof(T));

    // options.batch_first is IGNORED on purpose, exactly as the reference's GPU path ignores it
    // (include/detail/gpu_rnnt_kernel.h:7): the reference's own tests/test_gpu.cu:42-50 and
    // tests/test_time.cu pass it zero-initialised (false) with [N,T,U,V] data, so honouring or
    // rejecting it here would break every caller written against the reference.  The [T,U,N,V]
    // layout the reference's CPU path indexes (include/detail/cpu_rnnt.h:139-144) is available through
    // the explicit extension entry rnnt_b200_loss_async_layout (layout = RNNT_B200_LAYOUT_TUNV).
    Dims d = make_dims(t, c.tunv);
    d.rows = (uint32_t)rows64;

    // Integer inputs: device pointers are used in place; host pointers (the header's literal
    // contract, reference include/rnnt.h:84-89) are staged through the workspace.
    if (!c.async) {
        const size_t nl = (size_t)N * (opt.maxU > 1 ? opt.maxU - 1 : 0);
        if (!is_device_pointer(labels)) {
            if (nl && cudaMemcpyAsync(w.labels, labels, nl * sizeof(int), cudaMemcpyHostToDevice, s) != cudaSuccess)
                return RNNT_STATUS_MEMOPS_FAILED;
            labels = w.labels;
        }
        if (!is_device_pointer(ylen)) {
            if (cudaMemcpyAsync(w.ylen, ylen, N * sizeof(int), cudaMemcpyHostToDevice, s) != cudaSuccess)
                return RNNT_STATUS_MEMOPS_FAILED;
            ylen = w.ylen;
        }
        if (!is_device_pointer(xlen)) {
            if (cudaMemcpyAsync(w.xlen, xlen, N * sizeof(int), cudaMemcpyHostToDevice, s) != cudaSuccess)
                return RNNT_STATUS_MEMOPS_FAILED;
            xlen = w.xlen;
        }
    }

    // Overlap decision: the wavefront costs ~0.25 us per anti-diagonal whatever the batch; the
    // streaming passes cost 12 B/elt at ~3.0 TB/s (what they reach on an H100 SXM).  Worth splitting only
    // when the lattice is a visible share of a call that is long enough to amortise the extra launches.
    // The co-running lattice CTAs slow the streaming kernels a little, so the gain is modest, and there is none
    // when no pass 2 follows in the same call (loss-only / operator forward) - those stay in order.
    int groups = 1;
    if (c.phase == kFull && grads && N >= 2 * kAutoGroups && !d.tmajor) {
        const int forced = hooks().groups;
        const double lattice_us = 0.25 * (opt.maxT + opt.maxU) + 20.0;
        const double stream_us = (double)rows64 * V * sizeof(IO) * (grads ? 3.0 : 1.0) / 3.0e6;
        if (stream_us > 400.0 && lattice_us > 0.08 * stream_us) groups = kAutoGroups;
        if (forced >= 1 && forced <= kMaxGroups && forced <= N) groups = forced;
        if (groups > 1 && !side_pool().ok) groups = 1;
    }
    // EXPERIMENTAL, off unless RNNT_B200_PDL=1: launch the lattice and gradient kernels with programmatic
    // stream serialization, so their prologues (and the gradient kernel's first wave of logit loads) overlap
    // the tail of the kernel before them; each waits (griddepcontrol.wait) before it touches that kernel's
    // output.  The three kernels are each bound by their own latency chains rather than by the launch gaps,
    // so it stays opt-in.  (The event markers of the profiling mode would serialise the kernels anyway.)
    const bool pdl = hooks().pdl && groups == 1 && !g_profile;

    // ---- batch groups (Group).  One group = the plain in-order pipeline.  A pruned call's groups are offset by
    // maxT * R logit rows per utterance, its lattices by maxT * maxU cells as a dense call's.
    const size_t cell_stride = (size_t)opt.maxT * opt.maxU;            // lattice cells per utterance
    const size_t row_stride = (size_t)opt.maxT * rows_u;               // logit rows per utterance
    const size_t lat_stride = (size_t)(opt.maxT + opt.maxU - 1) * opt.maxU;
    const size_t lab_stride = opt.maxU > 1 ? opt.maxU - 1 : 0;
    using Pair = typename Real<T>::pair;
    T* cdev = c.async ? costs : static_cast<T*>(w.costs);
    const T* scale_vec = static_cast<const T*>(c.scale_vec);
    auto make_group = [&](int b0, int nb) {
        Group<T, IO> g;
        g.w = w;
        g.w.stat = static_cast<Pair*>(w.stat) + (size_t)b0 * row_stride;
        g.w.lp2 = static_cast<char*>(w.lp2) + (size_t)b0 * lat_stride * 16;
        // fp32 lattices are cell-major [b][t][u], fp64 ones diagonal-major (rnnt_kernels.cuh: cell / skew)
        const size_t val_stride = sizeof(T) == 4 ? cell_stride : lat_stride;
        g.w.alphas = static_cast<char*>(w.alphas) + (size_t)b0 * val_stride * 8;
        g.w.betas = static_cast<char*>(w.betas) + (size_t)b0 * val_stride * 8;
        g.w.llf = static_cast<char*>(w.llf) + (size_t)b0 * 8;
        g.w.llb = static_cast<char*>(w.llb) + (size_t)b0 * 8;
        g.d = d;
        g.d.N = nb;
        g.d.rows = (uint32_t)((size_t)nb * row_stride);
        g.acts = acts + (size_t)b0 * row_stride * V;
        g.grads = grads ? grads + (size_t)b0 * row_stride * V : nullptr;
        g.labels = labels + (size_t)b0 * lab_stride;
        g.xlen = xlen + b0;
        g.ylen = ylen + b0;
        g.costs = cdev ? cdev + b0 : nullptr;
        g.scale_vec = scale_vec ? scale_vec + b0 : nullptr;
        g.scale = (T)c.scale;
        g.reg = grad_options_on(c.grad);
        g.gr = make_grad_reg<T>(c.grad, g.w);
        g.s = s;
        g.pdl = pdl;
        g.pruned = c.pruned;
        g.pr = Prune{c.pruned ? t.ranges + (size_t)b0 * opt.maxT : nullptr, FastDiv((uint32_t)rows_u)};
        g.delay = delay_on(c.lattice);
        g.pen = (T)c.lattice.delay_penalty;
        g.pen_log2 = (T)((double)c.lattice.delay_penalty * 1.4426950408889634);
        g.mod = c.rnnt_type == RNNT_B200_RNNT_MODIFIED;
        return g;
    };
    const bool with_beta = grads || c.want_beta;
    bool co_running = false;   // set when the lattice of one group shares the GPU with the streaming passes of others
    auto launch_lattice = [&](const Group<T, IO>& g, cudaStream_t st) {
        if constexpr (sizeof(T) == 4) {
            launch_lattice_lin(static_cast<const float4*>(g.w.lp2), g.xlen, g.ylen, static_cast<LogVal*>(g.w.alphas),
                               static_cast<LogVal*>(g.w.betas), static_cast<LogVal*>(g.w.llf),
                               static_cast<LogVal*>(g.w.llb), g.costs, g.d, with_beta,
                               lattice_ring_depth(opt.maxU, co_running, hooks().lat_ring), st, g.pdl, g.mod);
        } else {
            launch_lattice_log(static_cast<const double2*>(g.w.lp2), g.xlen, g.ylen, static_cast<double*>(g.w.alphas),
                               static_cast<double*>(g.w.betas), static_cast<double*>(g.w.llf),
                               static_cast<double*>(g.w.llb), g.costs, g.d, with_beta, st, g.pdl, g.mod);
        }
        ++g_last_launches;
    };

    profile_begin_call();
    mark(0, s);
    if (c.pruned && c.phase != kBackward) {
        // log-zero factors for the cells no row covers (pass 1 writes the covered ones): 16 B per lattice cell
        using Fac = typename Lat<T>::fac;
        lattice_fill_kernel<T><<<(unsigned)std::min<size_t>((lat + 255) / 256, 4096), 256, 0, s>>>(
            static_cast<Fac*>(w.lp2), lat);
        ++g_last_launches;
    }
    if (groups == 1) {
        const Group<T, IO> g = make_group(0, N);
        if (c.phase != kBackward) {
            // pass 1: log-softmax statistics + (blank, label) log-prob gather
            stream_pass(g, 1);
            mark(1, s);
            if (c.phase == kAlign) {
                // best path and its label frames (DESIGN.md §12)
                launch_viterbi<T>(g.w.lp2, g.xlen, g.ylen, g.w.alphas, t.frames, g.costs, g.d, g.mod, s);
                ++g_last_launches;
            } else {
                // lattice: alpha (and beta when gradients are or will be wanted)
                launch_lattice(g, s);
            }
        } else {
            mark(1, s);
        }
        mark(2, s);
        // pass 2: dense gradient (+ zeros on padding)
        if (grads && c.phase != kForward) {
            stream_pass(g, 2);
            mark(3, s);
        }
    } else {
        SidePool& pool = side_pool();
        co_running = true;
        bool fork_ok = true;   // a failed fork/join would leave the gradient pass unordered against a lattice
        Timeline tl;
        tl.on = hooks().timeline;
        tl.tick("start", 0, s);
        Group<T, IO> gs[kMaxGroups];
        for (int k = 0; k < groups; ++k) {
            const int b0 = (int)((int64_t)N * k / groups), b1 = (int)((int64_t)N * (k + 1) / groups);
            gs[k] = make_group(b0, b1 - b0);
        }
        // main stream: pass 1 of every group back to back; each group's lattice forks off behind it
        for (int k = 0; k < groups; ++k) {
            stream_pass(gs[k], 1);
            tl.tick("rowstats_end", k, s);
            fork_ok &= cudaEventRecord(pool.forked[k], s) == cudaSuccess;
            fork_ok &= cudaStreamWaitEvent(pool.stream[k], pool.forked[k], 0) == cudaSuccess;
            tl.tick("lattice_beg", k, pool.stream[k]);
            launch_lattice(gs[k], pool.stream[k]);
            tl.tick("lattice_end", k, pool.stream[k]);
            fork_ok &= cudaEventRecord(pool.joined[k], pool.stream[k]) == cudaSuccess;
        }
        mark(1, s);
        // main stream: join each lattice, then that group's pass 2 (or just join, forward-only)
        for (int k = 0; k < groups; ++k) {
            fork_ok &= cudaStreamWaitEvent(s, pool.joined[k], 0) == cudaSuccess;
            if (k == 0) mark(2, s);
            tl.tick("grad_beg", k, s);
            if (grads && c.phase != kForward) stream_pass(gs[k], 2);
            tl.tick("grad_end", k, s);
        }
        tl.dump();
        if (grads && c.phase != kForward) mark(3, s);
        if (!fork_ok) {
            cudaStreamSynchronize(s);
            return RNNT_STATUS_EXECUTION_FAILED;
        }
    }

    if (cudaGetLastError() != cudaSuccess) return RNNT_STATUS_EXECUTION_FAILED;
    if (c.async) return RNNT_STATUS_SUCCESS;

    // costs to the caller (host memory in the reference contract) and the call's single sync
    const cudaMemcpyKind kind = is_device_pointer(costs) ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    if (cudaMemcpyAsync(costs, w.costs, N * sizeof(T), kind, s) != cudaSuccess)
        return RNNT_STATUS_MEMOPS_FAILED;
    if (cudaStreamSynchronize(s) != cudaSuccess) return RNNT_STATUS_EXECUTION_FAILED;
    return RNNT_STATUS_SUCCESS;
}

// ---- additive-joint variant (rnnt_joint.cuh) ----------------------------------------------------
constexpr int kJointSlices = 16;  // max split-K slabs of the S = Ef.Eg^T contraction (K = V is the long axis)
inline int joint_slices(int V) {
    const int forced = hooks().joint_slices;
    if (forced >= 1 && forced <= kJointSlices) return forced;   // tuning hook
    return std::max(1, std::min(kJointSlices, V / 320));
}
struct JointWorkspace {
    float *ef, *eg, *mf, *mg, *inv_s, *wm, *bk, *lb, *part;
    float4* lp2;
    LogVal *alphas, *betas, *llf, *llb;
    // smoothing sections (DESIGN.md §9), after the plain ones: carved only for a smoothed workspace
    float *sg, *A, *ug, *lug, *msum, *amw, *ou, *bu, *lu, *h;
    double* cpart;
    float2 *coef_f, *coef_g;
    size_t bytes;
};
JointWorkspace carve_joint(void* base, int N, int T, int U, int V, bool smooth = false) {
    JointWorkspace w;
    Carver c(base);
    const size_t C = (size_t)N * T * U, D = (size_t)N * (T + U - 1) * U;
    // the lattice sections first: their offsets do not depend on V, so the pruning-ranges entry finds them
    w.lp2 = c.take<float4>(D * 16);
    w.alphas = c.take<LogVal>(D * 8);
    w.betas = c.take<LogVal>(D * 8);
    w.llf = c.take<LogVal>((size_t)N * 8);
    w.llb = c.take<LogVal>((size_t)N * 8);
    w.ef = c.take<float>((size_t)N * T * V * 4);
    w.eg = c.take<float>((size_t)N * U * V * 4);
    w.mf = c.take<float>((size_t)N * T * 4);
    w.mg = c.take<float>((size_t)N * U * 4);
    w.inv_s = c.take<float>(C * 4);
    w.wm = c.take<float>(std::max(C, (size_t)N * T * wg::kWmPad) * 4);   // rows padded for the fused gradient kernel
    w.bk = c.take<float>(C * 4);
    w.lb = c.take<float>(C * 4);
    w.part = c.take<float>(C * 4 * kJointSlices);
    if (smooth) {
        const size_t NT = (size_t)N * T, NU = (size_t)N * U;
        w.sg = c.take<float>(NU * 4);
        w.A = c.take<float>(NT * 4);
        w.ug = c.take<float>((size_t)V * 4);
        w.lug = c.take<float>((size_t)V * 4);
        w.msum = c.take<float>(4);
        w.amw = c.take<float>(NT * 4);
        w.ou = c.take<float>(NU * 4);
        w.bu = c.take<float>(NU * 4);
        w.lu = c.take<float>(NU * 4);
        w.h = c.take<float>((size_t)V * 4);
        w.cpart = c.take<double>((size_t)kSmoothChunks * V * 8);
        w.coef_f = c.take<float2>(NT * 8);
        w.coef_g = c.take<float2>(NU * 8);
    }
    w.bytes = c.off + 256;
    return w;
}

// ---- tensor-core contractions of the additive joint (rnnt_wgmma.cuh) ---------------------------------
// N (accumulator columns per CTA) is the smallest instantiated width that holds `n`, tiled beyond 128
// (a thread holds N/2 accumulators: 128 columns keep two CTAs of 256 threads resident per SM).
// SMOOTH: the gradient epilogue adds the smoothing terms `sm` (DESIGN.md §9).  STAGEWISE: the stage-wise
// accumulation of S (rnnt_wgmma.cuh Stagewise), in tiles of at most 64 columns.
template <int A_MODE, int B_MODE, int KS, bool SMOOTH = false, bool STAGEWISE = false>
void launch_wgmma(const wg::Operand& A, const wg::Operand& B, int m, int n, int K, int slices, int batch,
                 const wg::Epilogue& epi, cudaStream_t s, int max_tile = 128, const wg::Smooth& sm = wg::Smooth{}) {
    auto go = [&](auto tile) {
        constexpr int NT = decltype(tile)::value;
        const size_t smem = wg::gemm_smem_bytes<NT, KS>();
        dim3 grid((unsigned)(slices * ((n + NT - 1) / NT)), (unsigned)((m + 127) / 128), (unsigned)batch);
        if constexpr (SMOOTH) {
            auto kernel = wg::gemm_kernel<A_MODE, B_MODE, NT, KS, wg::Smooth>;
            func_attr_once(reinterpret_cast<const void*>(kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            kernel<<<grid, wg::kThreads, smem, s>>>(A, B, K, slices, epi, sm);
        } else if constexpr (STAGEWISE) {
            auto kernel = wg::gemm_kernel<A_MODE, B_MODE, NT, KS, wg::Stagewise>;
            func_attr_once(reinterpret_cast<const void*>(kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            kernel<<<grid, wg::kThreads, smem, s>>>(A, B, K, slices, epi, wg::Stagewise{});
        } else {
            auto kernel = wg::gemm_kernel<A_MODE, B_MODE, NT, KS>;
            func_attr_once(reinterpret_cast<const void*>(kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            kernel<<<grid, wg::kThreads, smem, s>>>(A, B, K, slices, epi);
        }
    };
    if (n <= 32) go(std::integral_constant<int, 32>{});
    else if (STAGEWISE || n <= 64 || max_tile <= 64) go(std::integral_constant<int, 64>{});
    else if constexpr (!STAGEWISE) go(std::integral_constant<int, 128>{});
}

// t.acts / t.grads: the transcription factor f [N,T,V] and its gradient; g / dG: the prediction factor
// [N,U,V] and its gradient.  Only FastEmit of the gradient options applies (the entry rejects a clamp).
rnntStatus_t run_add_joint(const Tensors& t, const float* g, float* dG, const Call& c) {
    const float* f = static_cast<const float*>(t.acts);
    float* dF = static_cast<float*>(t.grads);
    if (!g || (dF == nullptr) != (dG == nullptr)) return RNNT_STATUS_INVALID_VALUE;
    if (const rnntStatus_t st = check_call(t, c)) return st;
    const rnntOptions& opt = t.opt;
    const int T = opt.maxT, U = opt.maxU, V = t.V, N = t.N;
    // the contraction kernels index inside one utterance's factor with 32-bit offsets
    if ((uint64_t)std::max(T, U) * (uint64_t)V >= (1ull << 31)) return RNNT_STATUS_INVALID_VALUE;
    const int *labels = t.labels, *ylen = t.ylen, *xlen = t.xlen;
    float* costs = static_cast<float*>(t.costs);
    const float scale = (float)c.scale;
    const float* scale_vec = static_cast<const float*>(c.scale_vec);
    const float fastemit_lambda = c.grad.fastemit_lambda;
    g_last_launches = 0;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(opt.stream);
    // smoothing (DESIGN.md §9): the SMOOTH instantiations and the extra kernels; both scales 0 is the plain joint
    const bool sm = smooth_on(c.smooth);
    const float lml = c.smooth.lm_only_scale, lma = c.smooth.am_only_scale;
    const float cfull = (float)std::max(0.0, 1.0 - (double)lml - (double)lma);
    JointWorkspace w = carve_joint(t.workspace, N, T, U, V, sm);
    JointDims jd{N, T, U, V, opt.blank_label};
    const Dims d = make_dims(t, false);
    const bool want_grad = dF != nullptr && c.phase != kForward;
    const bool with_beta = dF != nullptr || c.want_beta;

    if (c.phase != kBackward) {
    // J1: factor-wise max and exponentials (SUM: and sum[row] = sum_k e_k wv[k], wv NULL: 1); padded rows (t >= T_b
    // of f, u >= U_b of g) are not read and come out as zeros
    auto prep = [&](auto sum, const float* x, float* e, float* mx, const int* len, int add, int R,
                    const float* wv = nullptr, float* rowsum = nullptr) {
        constexpr bool SUM = decltype(sum)::value;
        const int rows = N * R;
        const int per = (V / 4 + 255) / 256;   // float4 per thread when one CTA owns a row
        const bool vec = V % 4 == 0 && per <= 8 && V >= 1024 && reinterpret_cast<uintptr_t>(x) % 16 == 0;
        if (!vec) joint_prep_kernel<SUM><<<(rows + 7) / 8, 256, 0, s>>>(x, e, mx, rows, V, len, add, R, wv, rowsum);
        else if (per <= 1) joint_prep_row_kernel<1, SUM><<<rows, 256, 0, s>>>(x, e, mx, V, len, add, R, wv, rowsum);
        else if (per <= 2) joint_prep_row_kernel<2, SUM><<<rows, 256, 0, s>>>(x, e, mx, V, len, add, R, wv, rowsum);
        else if (per <= 4) joint_prep_row_kernel<4, SUM><<<rows, 256, 0, s>>>(x, e, mx, V, len, add, R, wv, rowsum);
        else if (per <= 5) joint_prep_row_kernel<5, SUM><<<rows, 256, 0, s>>>(x, e, mx, V, len, add, R, wv, rowsum);
        else joint_prep_row_kernel<8, SUM><<<rows, 256, 0, s>>>(x, e, mx, V, len, add, R, wv, rowsum);
    };
    using Plain = std::false_type;
    using Sum = std::true_type;
    if (!sm) {
        prep(Plain{}, f, w.ef, w.mf, xlen, 0, T);
        prep(Plain{}, g, w.eg, w.mg, ylen, 1, U);
    } else {
        // g first (Eg and its row sums sg), then the unigram of the valid pred rows, then f (with A = Ef . ug)
        prep(Sum{}, g, w.eg, w.mg, ylen, 1, U, nullptr, w.sg);
        if (lma != 0.0f) {
            const int chunks = smooth_chunks(N * U);
            joint_colsum_kernel<true><<<dim3((V + 255) / 256, chunks), 256, 0, s>>>(w.eg, w.sg, ylen, 1, N, U, V,
                                                                                  chunks, w.cpart);
            joint_unigram_kernel<<<(V + 255) / 256, 256, 0, s>>>(w.cpart, chunks, ylen, N, U, V, w.ug, w.lug, w.msum);
            prep(Sum{}, f, w.ef, w.mf, xlen, 0, T, w.ug, w.A);
            g_last_launches += 2;
        } else {
            prep(Plain{}, f, w.ef, w.mf, xlen, 0, T);
        }
    }
    // J2: S = Ef . Eg^T in kJointSlices deterministic K-slabs, then lse + lattice log-prob pairs
    {
        const int slices = joint_slices(V);
        if (!hooks().joint_simt) {
            // wgmma: M = t (tiles of 128), N = u, K = v split into `slices` slabs
            wg::Operand A{w.ef, (long long)T * V, V, 1, T}, B{w.eg, (long long)U * V, V, 1, U};
            // float4 operand fetches when every row of Ef / Eg starts on a 16-byte boundary
            // partial sums of slice ks land in slab ks: part[ks][b][t][u]
            const wg::Epilogue epi{nullptr, 0, 0, 0, w.part, (long long)d.rows, (long long)T * U, U, 1};
            // slabs of more than 8 stages (256 columns) accumulate stage-wise: one accumulator would take more
            // than 96 MMAs, each truncating toward zero (rnnt_wgmma.cuh Stagewise)
            const bool stagewise = (V + slices - 1) / slices > 256;
            if (V % 4 == 0) {
                if (stagewise) launch_wgmma<2, 2, 32, false, true>(A, B, T, U, V, slices, N, epi, s);
                else launch_wgmma<2, 2, 32>(A, B, T, U, V, slices, N, epi, s);
            } else {
                if (stagewise) launch_wgmma<1, 1, 32, false, true>(A, B, T, U, V, slices, N, epi, s);
                else launch_wgmma<1, 1, 32>(A, B, T, U, V, slices, N, epi, s);
            }
        } else {
            Operand A{w.ef, (size_t)T * V, V, 1}, B{w.eg, (size_t)U * V, V, 1};
            dim3 grid((U + 63) / 64, (T + 63) / 64, N * slices);
            if (U <= 32) {
                grid.x = (U + 31) / 32;
                joint_gemm_kernel<EpiPartial, 32, 32><<<grid, 256, 0, s>>>(
                    A, B, T, U, V, slices, EpiPartial{w.part, (size_t)d.rows, T, U, slices});
            } else {
                joint_gemm_kernel<EpiPartial, 64, 32><<<grid, 256, 0, s>>>(
                    A, B, T, U, V, slices, EpiPartial{w.part, (size_t)d.rows, T, U, slices});
            }
        }
        // the delay penalty (DESIGN.md §10) goes into the factors here; every later kernel reads them from lp2
        const bool dl = delay_on(c.lattice);
        const unsigned sgrid = (d.rows + 255) / 256;
        if (!sm) {
            if (!dl) {
                EpiStats<> epi{f, g, w.mf, w.mg, labels, xlen, ylen, w.inv_s, w.lp2, jd, d};
                joint_stats_kernel<<<sgrid, 256, 0, s>>>(w.part, slices, epi);
            } else {
                EpiStats<false, true> epi{f, g, w.mf, w.mg, labels, xlen, ylen, w.inv_s, w.lp2, jd, d};
                epi.delay = c.lattice.delay_penalty;
                joint_stats_delay_kernel<<<sgrid, 256, 0, s>>>(w.part, slices, epi);
            }
        } else {
            if (!dl) {
                EpiStats<true> epi{f, g, w.mf, w.mg, labels, xlen, ylen, w.inv_s, w.lp2, jd, d, w.sg, w.A, w.lug,
                                   cfull, lml, lma};
                joint_stats_kernel<true><<<sgrid, 256, 0, s>>>(w.part, slices, epi);
            } else {
                EpiStats<true, true> epi{f, g, w.mf, w.mg, labels, xlen, ylen, w.inv_s, w.lp2, jd, d, w.sg, w.A,
                                         w.lug, cfull, lml, lma, c.lattice.delay_penalty};
                joint_stats_delay_kernel<true><<<sgrid, 256, 0, s>>>(w.part, slices, epi);
            }
        }
    }
    // lattice: the dense path's fp32 wavefront, with the default ring depth and no PDL
    launch_lattice_lin(w.lp2, xlen, ylen, w.alphas, w.betas, w.llf, w.llb, costs, d, with_beta, 8, s, false,
                       c.rnnt_type == RNNT_B200_RNNT_MODIFIED);
    g_last_launches += 5;
    }  // phase != kBackward
    if (want_grad) {
        const Hooks& hk = hooks();
        const bool use_fused = hk.joint_fused && !hk.joint_simt && U <= wg::kWmPad &&
                               (uint64_t)N * T * wg::kWmPad < (1ull << 31);   // padded weights are indexed with 32 bits
        const int wm_pitch = use_fused ? wg::kWmPad : U;
        const unsigned wm_entries = (unsigned)N * T * wm_pitch;
        auto weights = fastemit_lambda > 0.0f ? (sm ? joint_weights_kernel<true, true> : joint_weights_kernel<true>)
                                              : (sm ? joint_weights_kernel<false, true> : joint_weights_kernel<false>);
        if (c.rnnt_type == RNNT_B200_RNNT_MODIFIED)   // the modified topology (DESIGN.md §11)
            weights = fastemit_lambda > 0.0f
                          ? (sm ? joint_weights_mod_kernel<true, true> : joint_weights_mod_kernel<true>)
                          : (sm ? joint_weights_mod_kernel<false, true> : joint_weights_mod_kernel<false>);
        weights<<<(wm_entries + 255) / 256, 256, 0, s>>>(w.lp2, w.alphas, w.betas, w.llf, w.inv_s, xlen, ylen, w.wm, w.bk,
                                                         w.lb, scale, scale_vec, d, wm_pitch, fastemit_lambda, cfull);
        // smoothing: the per-row epilogue coefficients of dF and dG, and h (the gradient through ug) when lma > 0
        wg::Smooth smf{}, smg{};
        if (sm) {
            joint_smooth_rows_kernel<<<(N * (T + U) + 7) / 8, 256, 0, s>>>(w.bk, w.lb, w.A, xlen, ylen, jd, lma,
                                                                              w.coef_f, w.amw, w.ou, w.bu, w.lu);
            const float* h = nullptr;
            if (lma != 0.0f) {
                const int chunks = smooth_chunks(N * T);
                joint_colsum_kernel<false><<<dim3((V + 255) / 256, chunks), 256, 0, s>>>(w.ef, w.amw, xlen, 0, N, T, V,
                                                                                       chunks, w.cpart);
                joint_unigram_grad_kernel<<<(V + 255) / 256, 256, 0, s>>>(w.cpart, chunks, w.ug, w.bu, w.lu, labels,
                                                                          ylen, jd, lma, w.h);
                h = w.h;
                g_last_launches += 2;
            }
            joint_smooth_g_kernel<<<(N * U + 7) / 8, 256, 0, s>>>(w.eg, w.sg, h, w.ou, w.msum, ylen, jd, lml, w.coef_g);
            // without the am-only term the dF coefficients are zero: no smoothing term on dF at all
            if (lma != 0.0f) smf = wg::Smooth{w.coef_f, T, w.ug};
            smg = wg::Smooth{w.coef_g, U, h};
            g_last_launches += 2;
        }
        if (!hk.joint_simt) {
            // wgmma, vocabulary index on the accumulator rows (32-byte sectors in the epilogue):
            //   dF[t,v] = Ef[t,v] * sum_u Eg[u,v] Wm[t,u]      M = v, N = t, K = u
            //   dG[u,v] = Eg[u,v] * sum_t Ef[t,v] Wm[t,u]      M = v, N = u, K = t
            wg::Operand EgT{w.eg, (long long)U * V, 1, V, V}, EfT{w.ef, (long long)T * V, 1, V, V};
            wg::Operand WmTU{w.wm, (long long)T * U, U, 1, T};   // (n = t, k = u): k-contiguous
            wg::Operand WmUT{w.wm, (long long)T * U, 1, U, U};   // (n = u, k = t): n-contiguous
            if (use_fused) {
                // both contractions in one pass over Ef (rnnt_wgmma.cuh: grad_fused_kernel)
                const wg::GradFused gf{w.ef, w.eg, w.wm, dF, dG, T, U, V, smf, smg};
                const size_t smem = wg::GradFusedGeom<32, 32>::total + hk.fused_pad_smem;   // pad: residency experiment hook
                auto go = [&](auto kernel) {
                    func_attr_once(reinterpret_cast<const void*>(kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
                    kernel<<<dim3((unsigned)((V + 127) / 128), 1, (unsigned)N), wg::kThreads, smem, s>>>(gf);
                };
                if (sm) {
                    if (V % 4 == 0) go(wg::grad_fused_kernel<32, 32, 3, true>);
                    else go(wg::grad_fused_kernel<32, 32, 0, true>);
                } else {
                    if (V % 4 == 0) go(wg::grad_fused_kernel<32, 32, 3>);
                    else go(wg::grad_fused_kernel<32, 32, 0>);
                }
            } else {
            // dF in 64-column accumulator tiles by default: small register / shared-memory footprint -> several
            // CTAs per SM, and the whole tile's Ef fetches are in flight before the accumulator is read
            const wg::Epilogue epf{w.ef, (long long)T * V, 1, V, dF, 0, (long long)T * V, 1, V};
            const wg::Epilogue epg{w.eg, (long long)U * V, 1, V, dG, 0, (long long)U * V, 1, V};
            if (!sm) {
                if (V % 4 == 0) launch_wgmma<3, 1, 24>(EgT, WmTU, V, T, U, 1, N, epf, s, hk.df_tile);   // 16-byte aligned rows
                else launch_wgmma<0, 1, 24>(EgT, WmTU, V, T, U, 1, N, epf, s, hk.df_tile);
                if (V % 4 == 0) launch_wgmma<3, 0, 24>(EfT, WmUT, V, U, T, 1, N, epg, s);
                else launch_wgmma<0, 0, 24>(EfT, WmUT, V, U, T, 1, N, epg, s);
            } else {
                if (V % 4 == 0) launch_wgmma<3, 1, 24, true>(EgT, WmTU, V, T, U, 1, N, epf, s, hk.df_tile, smf);
                else launch_wgmma<0, 1, 24, true>(EgT, WmTU, V, T, U, 1, N, epf, s, hk.df_tile, smf);
                if (V % 4 == 0) launch_wgmma<3, 0, 24, true>(EfT, WmUT, V, U, T, 1, N, epg, s, 128, smg);
                else launch_wgmma<0, 0, 24, true>(EfT, WmUT, V, U, T, 1, N, epg, s, 128, smg);
            }
            }
        } else if (V >= 512) {  // long vocabulary: one thread per column, thin contraction
            {   // dF[t,v] = Ef[t,v] * sum_u Wm[t,u] Eg[u,v]
                dim3 grid((V + 255) / 256, (T + kJointRT - 1) / kJointRT, N);
                if (!sm) joint_thin_kernel<<<grid, 256, 0, s>>>(w.wm, U, 1, (size_t)T * U, w.eg, w.ef, dF, T, U, V,
                                                                nullptr, nullptr);
                else joint_thin_kernel<true><<<grid, 256, 0, s>>>(w.wm, U, 1, (size_t)T * U, w.eg, w.ef, dF, T, U, V,
                                                                  smf.coef, smf.w);
            }
            {   // dG[u,v] = Eg[u,v] * sum_t Wm[t,u] Ef[t,v]
                dim3 grid((V + 255) / 256, (U + kJointRT - 1) / kJointRT, N);
                if (!sm) joint_thin_kernel<<<grid, 256, 0, s>>>(w.wm, 1, U, (size_t)T * U, w.ef, w.eg, dG, U, T, V,
                                                                nullptr, nullptr);
                else joint_thin_kernel<true><<<grid, 256, 0, s>>>(w.wm, 1, U, (size_t)T * U, w.ef, w.eg, dG, U, T, V,
                                                                  smg.coef, smg.w);
            }
        } else {  // short vocabulary: tiled GEMM
            {
                Operand A{w.wm, (size_t)T * U, U, 1}, B{w.eg, (size_t)U * V, 1, V};
                dim3 grid((V + 63) / 64, (T + 63) / 64, N);
                if (!sm) joint_gemm_kernel<EpiGrad<>><<<grid, 256, 0, s>>>(A, B, T, V, U, 1, EpiGrad<>{w.ef, dF, T, V});
                else joint_gemm_kernel<EpiGrad<true>><<<grid, 256, 0, s>>>(
                    A, B, T, V, U, 1, EpiGrad<true>{w.ef, dF, T, V, smf.coef, smf.w});
            }
            {
                Operand A{w.wm, (size_t)T * U, 1, U}, B{w.ef, (size_t)T * V, 1, V};
                dim3 grid((V + 63) / 64, (U + 63) / 64, N);
                if (!sm) joint_gemm_kernel<EpiGrad<>><<<grid, 256, 0, s>>>(A, B, U, V, T, 1, EpiGrad<>{w.eg, dG, U, V});
                else joint_gemm_kernel<EpiGrad<true>><<<grid, 256, 0, s>>>(
                    A, B, U, V, T, 1, EpiGrad<true>{w.eg, dG, U, V, smg.coef, smg.w});
            }
        }
        if (!sm) {
            joint_sparse_f_kernel<<<(N * T + 3) / 4, 128, 0, s>>>(dF, w.bk, w.lb, labels, ylen, jd, 1.0f);
            joint_sparse_g_kernel<<<(N * U + 3) / 4, 128, 0, s>>>(dG, w.bk, w.lb, labels, xlen, ylen, jd, 1.0f);
        } else {
            joint_sparse_f_kernel<true><<<(N * T + 3) / 4, 128, 0, s>>>(dF, w.bk, w.lb, labels, ylen, jd, cfull + lma);
            joint_sparse_g_kernel<true><<<(N * U + 3) / 4, 128, 0, s>>>(dG, w.bk, w.lb, labels, xlen, ylen, jd,
                                                                        cfull + lml);
        }
        g_last_launches += 5;
    }
    return cudaGetLastError() == cudaSuccess ? RNNT_STATUS_SUCCESS : RNNT_STATUS_EXECUTION_FAILED;
}

// storage-type code of the C-ABI (include/rnnt.h) -> run<IO>; an unknown code is INVALID_VALUE
rnntStatus_t run_as(int dtype, const Tensors& t, const Call& c) {
    switch (dtype) {
        case RNNT_B200_FP32: return run<float>(t, c);
        case RNNT_B200_FP64: return run<double>(t, c);
        case RNNT_B200_BF16: return run<__nv_bfloat16>(t, c);
        case RNNT_B200_FP16: return run<__half>(t, c);
    }
    return RNNT_STATUS_INVALID_VALUE;
}
inline bool is_16bit(int dtype) { return dtype == RNNT_B200_BF16 || dtype == RNNT_B200_FP16; }
inline bool is_layout(int layout) { return layout == RNNT_B200_LAYOUT_NTUV || layout == RNNT_B200_LAYOUT_TUNV; }

// ---- the loss, gradient and alignment on caller-supplied factors (DESIGN.md §13) --------------------------------
// The tensors of a lattice call: px [N, maxU-1, maxT], py [N, maxU, maxT] and their gradients in the storage type.
struct LatticeTensors {
    const void *px, *py;
    void *px_grad, *py_grad;   // backward
    const int *ylen, *xlen;
    int N;
    void* costs;               // forward: costs; align: scores (arithmetic type)
    int* frames;               // align
    void* workspace;
    rnntOptions opt;
};

inline size_t lattice_cells(int N, int maxT, int maxU) { return (size_t)N * (maxT + maxU - 1) * maxU; }

// check_call's extent rules without its V and blank rules; every check before any device access.  px, px_grad and
// frames have no element when maxU == 1 and may then be NULL.
rnntStatus_t check_lattice(int dtype, const LatticeTensors& t, const Call& c) {
    const rnntOptions& opt = t.opt;
    if ((dtype != RNNT_B200_FP32 && dtype != RNNT_B200_FP64 && !is_16bit(dtype)) ||
        (c.rnnt_type != RNNT_B200_RNNT_REGULAR && c.rnnt_type != RNNT_B200_RNNT_MODIFIED))
        return RNNT_STATUS_INVALID_VALUE;
    const bool labels = opt.maxU > 1;
    if (!t.ylen || !t.xlen || !t.workspace || t.N <= 0 || opt.maxT <= 0 || opt.maxU <= 0)
        return RNNT_STATUS_INVALID_VALUE;
    if (c.phase == kBackward ? (!t.py_grad || (labels && !t.px_grad))
                             : (!t.py || (labels && !t.px) || !t.costs || (c.phase == kAlign && labels && !t.frames)))
        return RNNT_STATUS_INVALID_VALUE;
    if (opt.loc == RNNT_CPU) {
        fprintf(stderr, "b200-rnnt: CPU execution requested, but this library is the CUDA path only\n");
        return RNNT_STATUS_EXECUTION_FAILED;
    }
    if (opt.loc != RNNT_GPU || (uint64_t)t.N * opt.maxT * opt.maxU >= (1ull << 31) || opt.maxU > 1024)
        return RNNT_STATUS_INVALID_VALUE;
    return RNNT_STATUS_SUCCESS;
}

// One batch group, no PDL, no host synchronisation.  Forward: import, then the wavefront (alpha, and beta when
// want_beta) - 2 launches.  Backward: the gradient kernel on the workspace alone - 1.  Align: import, then the
// Viterbi kernel - 2.
template <typename IO>
rnntStatus_t run_lattice(const LatticeTensors& t, const Call& c) {
    using T = typename ComputeOf<IO>::type;
    const rnntOptions& opt = t.opt;
    const int N = t.N;
    g_last_launches = 0;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(opt.stream);
    Workspace w = carve(t.workspace, 0, lattice_cells(N, opt.maxT, opt.maxU), N, opt.maxU, sizeof(T));
    Tensors dt{nullptr, nullptr, nullptr, t.ylen, t.xlen, 1, N, nullptr, nullptr, opt};
    dt.opt.blank_label = 0;
    const Dims d = make_dims(dt, false);
    const bool mod = c.rnnt_type == RNNT_B200_RNNT_MODIFIED;
    using Fac = typename Lat<T>::fac;
    using Val = typename Lat<T>::val;
    const unsigned blocks = lattice_io_blocks(d);
    T* costs = static_cast<T*>(t.costs);
    if (c.phase != kBackward) {
        lattice_import_kernel<IO><<<blocks, 256, 0, s>>>(static_cast<const IO*>(t.px), static_cast<const IO*>(t.py),
                                                        t.xlen, t.ylen, static_cast<Fac*>(w.lp2), d);
        ++g_last_launches;
    }
    if (c.phase == kForward) {
        if constexpr (sizeof(T) == 4)
            launch_lattice_lin(static_cast<const float4*>(w.lp2), t.xlen, t.ylen, static_cast<LogVal*>(w.alphas),
                               static_cast<LogVal*>(w.betas), static_cast<LogVal*>(w.llf),
                               static_cast<LogVal*>(w.llb), costs, d, c.want_beta,
                               lattice_ring_depth(opt.maxU, false, hooks().lat_ring), s, false, mod);
        else
            launch_lattice_log(static_cast<const double2*>(w.lp2), t.xlen, t.ylen, static_cast<double*>(w.alphas),
                               static_cast<double*>(w.betas), static_cast<double*>(w.llf),
                               static_cast<double*>(w.llb), costs, d, c.want_beta, s, false, mod);
    } else if (c.phase == kAlign) {
        launch_viterbi<T>(w.lp2, t.xlen, t.ylen, w.alphas, t.frames, costs, d, mod, s);
    } else {
        auto kernel = mod ? lattice_grad_kernel<IO, T, true> : lattice_grad_kernel<IO, T, false>;
        kernel<<<blocks, 256, 0, s>>>(static_cast<const Fac*>(w.lp2), static_cast<const Val*>(w.alphas),
                                      static_cast<const Val*>(w.betas), static_cast<const Val*>(w.llf), t.xlen, t.ylen,
                                      static_cast<IO*>(t.px_grad), static_cast<IO*>(t.py_grad), (T)c.scale,
                                      static_cast<const T*>(c.scale_vec), d);
    }
    ++g_last_launches;
    return cudaGetLastError() == cudaSuccess ? RNNT_STATUS_SUCCESS : RNNT_STATUS_EXECUTION_FAILED;
}

rnntStatus_t run_lattice_as(int dtype, const LatticeTensors& t, const Call& c) {
    if (const rnntStatus_t st = check_lattice(dtype, t, c)) return st;
    switch (dtype) {
        case RNNT_B200_FP32: return run_lattice<float>(t, c);
        case RNNT_B200_FP64: return run_lattice<double>(t, c);
        case RNNT_B200_BF16: return run_lattice<__nv_bfloat16>(t, c);
        case RNNT_B200_FP16: return run_lattice<__half>(t, c);
    }
    return RNNT_STATUS_INVALID_VALUE;
}

}  // namespace

extern "C" {

int get_warprnnt_version(void) { return 1; }

const char* rnntGetStatusString(rnntStatus_t status) {
    switch (status) {
        case RNNT_STATUS_SUCCESS: return "no error";
        case RNNT_STATUS_MEMOPS_FAILED: return "cuda memcpy or memset failed";
        case RNNT_STATUS_INVALID_VALUE: return "invalid value";
        case RNNT_STATUS_EXECUTION_FAILED: return "execution failed";
        case RNNT_STATUS_UNKNOWN_ERROR:
        default: return "unknown error";
    }
}

rnntStatus_t compute_rnnt_loss(const float* const activations, float* gradients,
                               const int* const flat_labels, const int* const label_lengths,
                               const int* const input_lengths, int alphabet_size, int minibatch,
                               float* costs, void* workspace, rnntOptions options) {
    return run_as(RNNT_B200_FP32, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size,
                                   minibatch, costs, workspace, options}, full_call(1.0, false));
}

rnntStatus_t compute_rnnt_loss_fp64(const double* const activations, double* gradients,
                                    const int* const flat_labels,
                                    const int* const label_lengths,
                                    const int* const input_lengths, int alphabet_size,
                                    int minibatch, double* costs, void* workspace,
                                    rnntOptions options) {
    return run_as(RNNT_B200_FP64, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size,
                                   minibatch, costs, workspace, options}, full_call(1.0, false));
}

rnntStatus_t compute_rnnt_loss_async(const float* const activations, float* gradients,
                                     const int* const flat_labels,
                                     const int* const label_lengths,
                                     const int* const input_lengths, int alphabet_size,
                                     int minibatch, float* costs_device, float grad_scale,
                                     void* workspace, rnntOptions options) {
    return run_as(RNNT_B200_FP32, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size,
                                   minibatch, costs_device, workspace, options}, full_call(grad_scale));
}

rnntStatus_t compute_rnnt_loss_async_fp64(const double* const activations, double* gradients,
                                          const int* const flat_labels,
                                          const int* const label_lengths,
                                          const int* const input_lengths, int alphabet_size,
                                          int minibatch, double* costs_device, double grad_scale,
                                          void* workspace, rnntOptions options) {
    return run_as(RNNT_B200_FP64, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size,
                                   minibatch, costs_device, workspace, options}, full_call(grad_scale));
}

rnntStatus_t rnnt_b200_forward(const float* const activations, const int* const flat_labels,
                               const int* const label_lengths, const int* const input_lengths,
                               int alphabet_size, int minibatch, float* costs_device,
                               int prepare_backward, void* workspace, rnntOptions options) {
    return run_as(RNNT_B200_FP32, {activations, nullptr, flat_labels, label_lengths, input_lengths, alphabet_size,
                                   minibatch, costs_device, workspace, options}, forward_call(prepare_backward));
}

rnntStatus_t rnnt_b200_forward_fp64(const double* const activations, const int* const flat_labels,
                                    const int* const label_lengths, const int* const input_lengths,
                                    int alphabet_size, int minibatch, double* costs_device,
                                    int prepare_backward, void* workspace, rnntOptions options) {
    return run_as(RNNT_B200_FP64, {activations, nullptr, flat_labels, label_lengths, input_lengths, alphabet_size,
                                   minibatch, costs_device, workspace, options}, forward_call(prepare_backward));
}

rnntStatus_t rnnt_b200_backward(const float* const activations, float* gradients,
                                const int* const flat_labels, const int* const label_lengths,
                                const int* const input_lengths, int alphabet_size, int minibatch,
                                const float* grad_costs_device, float grad_scale, void* workspace,
                                rnntOptions options) {
    return run_as(RNNT_B200_FP32, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size,
                                   minibatch, nullptr, workspace, options}, backward_call(grad_scale, grad_costs_device));
}

rnntStatus_t rnnt_b200_backward_fp64(const double* const activations, double* gradients,
                                     const int* const flat_labels, const int* const label_lengths,
                                     const int* const input_lengths, int alphabet_size,
                                     int minibatch, const double* grad_costs_device,
                                     double grad_scale, void* workspace, rnntOptions options) {
    return run_as(RNNT_B200_FP64, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size,
                                   minibatch, nullptr, workspace, options}, backward_call(grad_scale, grad_costs_device));
}

// ---- explicit activation layout ([N,T,U,V] or [T,U,N,V]) ------------------------------------------
rnntStatus_t rnnt_b200_loss_async_layout(int layout, const float* activations, float* gradients,
                                         const int* flat_labels, const int* label_lengths,
                                         const int* input_lengths, int alphabet_size, int minibatch,
                                         float* costs_device, float grad_scale, void* workspace,
                                         rnntOptions options) {
    if (!is_layout(layout)) return RNNT_STATUS_INVALID_VALUE;
    return run_as(RNNT_B200_FP32, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size,
                                   minibatch, costs_device, workspace, options},
                  full_call(grad_scale, true, layout == RNNT_B200_LAYOUT_TUNV));
}

rnntStatus_t rnnt_b200_loss_async_layout_fp64(int layout, const double* activations, double* gradients,
                                              const int* flat_labels, const int* label_lengths,
                                              const int* input_lengths, int alphabet_size, int minibatch,
                                              double* costs_device, double grad_scale, void* workspace,
                                              rnntOptions options) {
    if (!is_layout(layout)) return RNNT_STATUS_INVALID_VALUE;
    return run_as(RNNT_B200_FP64, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size,
                                   minibatch, costs_device, workspace, options},
                  full_call(grad_scale, true, layout == RNNT_B200_LAYOUT_TUNV));
}

// ---- 16-bit storage (bf16 / fp16 logits and gradients, fp32 arithmetic and costs) ---------------
rnntStatus_t rnnt_b200_loss_async_16(int dtype, const void* activations, void* gradients,
                                     const int* flat_labels, const int* label_lengths,
                                     const int* input_lengths, int alphabet_size, int minibatch,
                                     float* costs_device, float grad_scale, void* workspace,
                                     rnntOptions options) {
    if (!is_16bit(dtype)) return RNNT_STATUS_INVALID_VALUE;
    return run_as(dtype, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          costs_device, workspace, options}, full_call(grad_scale));
}

rnntStatus_t rnnt_b200_forward_16(int dtype, const void* activations, const int* flat_labels,
                                  const int* label_lengths, const int* input_lengths,
                                  int alphabet_size, int minibatch, float* costs_device,
                                  int prepare_backward, void* workspace, rnntOptions options) {
    if (!is_16bit(dtype)) return RNNT_STATUS_INVALID_VALUE;
    return run_as(dtype, {activations, nullptr, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          costs_device, workspace, options}, forward_call(prepare_backward));
}

rnntStatus_t rnnt_b200_backward_16(int dtype, const void* activations, void* gradients,
                                   const int* flat_labels, const int* label_lengths,
                                   const int* input_lengths, int alphabet_size, int minibatch,
                                   const float* grad_costs_device, float grad_scale, void* workspace,
                                   rnntOptions options) {
    if (!is_16bit(dtype)) return RNNT_STATUS_INVALID_VALUE;
    return run_as(dtype, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          nullptr, workspace, options}, backward_call(grad_scale, grad_costs_device));
}

// ---- gradient options (FastEmit, clamp) for every storage type -------------------------------------
rnntStatus_t rnnt_b200_loss_async_ex(int dtype, int layout, const void* activations, void* gradients,
                                     const int* flat_labels, const int* label_lengths,
                                     const int* input_lengths, int alphabet_size, int minibatch,
                                     void* costs_device, double grad_scale, rnntGradOptions grad_options,
                                     void* workspace, rnntOptions options) {
    const bool tunv = layout == RNNT_B200_LAYOUT_TUNV;
    if (!is_layout(layout) || (tunv && is_16bit(dtype))) return RNNT_STATUS_INVALID_VALUE;
    return run_as(dtype, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          costs_device, workspace, options}, full_call(grad_scale, true, tunv, grad_options));
}

rnntStatus_t rnnt_b200_backward_ex(int dtype, const void* activations, void* gradients,
                                   const int* flat_labels, const int* label_lengths,
                                   const int* input_lengths, int alphabet_size, int minibatch,
                                   const void* grad_costs_device, double grad_scale,
                                   rnntGradOptions grad_options, void* workspace, rnntOptions options) {
    return run_as(dtype, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          nullptr, workspace, options}, backward_call(grad_scale, grad_costs_device, grad_options));
}

// ---- lattice options (delay penalty, DESIGN.md §10) and topology (DESIGN.md §11) for every storage type -----
// The *_lat entries are the *_topo ones with the regular topology.
rnntStatus_t rnnt_b200_loss_async_topo(int dtype, int layout, const void* activations, void* gradients,
                                       const int* flat_labels, const int* label_lengths,
                                       const int* input_lengths, int alphabet_size, int minibatch,
                                       void* costs_device, double grad_scale, rnntGradOptions grad_options,
                                       rnntLatticeOptions lattice_options, int rnnt_type, void* workspace,
                                       rnntOptions options) {
    const bool tunv = layout == RNNT_B200_LAYOUT_TUNV;
    if (!is_layout(layout) || (tunv && is_16bit(dtype))) return RNNT_STATUS_INVALID_VALUE;
    Call c = full_call(grad_scale, true, tunv, grad_options);
    c.lattice = lattice_options;
    c.rnnt_type = rnnt_type;
    return run_as(dtype, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          costs_device, workspace, options}, c);
}
rnntStatus_t rnnt_b200_loss_async_lat(int dtype, int layout, const void* activations, void* gradients,
                                      const int* flat_labels, const int* label_lengths,
                                      const int* input_lengths, int alphabet_size, int minibatch,
                                      void* costs_device, double grad_scale, rnntGradOptions grad_options,
                                      rnntLatticeOptions lattice_options, void* workspace, rnntOptions options) {
    return rnnt_b200_loss_async_topo(dtype, layout, activations, gradients, flat_labels, label_lengths, input_lengths,
                                     alphabet_size, minibatch, costs_device, grad_scale, grad_options, lattice_options,
                                     RNNT_B200_RNNT_REGULAR, workspace, options);
}

rnntStatus_t rnnt_b200_forward_topo(int dtype, const void* activations, const int* flat_labels,
                                    const int* label_lengths, const int* input_lengths, int alphabet_size,
                                    int minibatch, void* costs_device, int prepare_backward,
                                    rnntLatticeOptions lattice_options, int rnnt_type, void* workspace,
                                    rnntOptions options) {
    Call c = forward_call(prepare_backward);
    c.lattice = lattice_options;
    c.rnnt_type = rnnt_type;
    return run_as(dtype, {activations, nullptr, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          costs_device, workspace, options}, c);
}
rnntStatus_t rnnt_b200_forward_lat(int dtype, const void* activations, const int* flat_labels,
                                   const int* label_lengths, const int* input_lengths, int alphabet_size,
                                   int minibatch, void* costs_device, int prepare_backward,
                                   rnntLatticeOptions lattice_options, void* workspace, rnntOptions options) {
    return rnnt_b200_forward_topo(dtype, activations, flat_labels, label_lengths, input_lengths, alphabet_size,
                                  minibatch, costs_device, prepare_backward, lattice_options, RNNT_B200_RNNT_REGULAR,
                                  workspace, options);
}

rnntStatus_t rnnt_b200_backward_topo(int dtype, const void* activations, void* gradients,
                                     const int* flat_labels, const int* label_lengths,
                                     const int* input_lengths, int alphabet_size, int minibatch,
                                     const void* grad_costs_device, double grad_scale,
                                     rnntGradOptions grad_options, rnntLatticeOptions lattice_options, int rnnt_type,
                                     void* workspace, rnntOptions options) {
    Call c = backward_call(grad_scale, grad_costs_device, grad_options);
    c.lattice = lattice_options;
    c.rnnt_type = rnnt_type;
    return run_as(dtype, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          nullptr, workspace, options}, c);
}
rnntStatus_t rnnt_b200_backward_lat(int dtype, const void* activations, void* gradients,
                                    const int* flat_labels, const int* label_lengths,
                                    const int* input_lengths, int alphabet_size, int minibatch,
                                    const void* grad_costs_device, double grad_scale,
                                    rnntGradOptions grad_options, rnntLatticeOptions lattice_options,
                                    void* workspace, rnntOptions options) {
    return rnnt_b200_backward_topo(dtype, activations, gradients, flat_labels, label_lengths, input_lengths,
                                   alphabet_size, minibatch, grad_costs_device, grad_scale, grad_options,
                                   lattice_options, RNNT_B200_RNNT_REGULAR, workspace, options);
}

rnntStatus_t rnnt_b200_pruned_loss_async_topo(int dtype, int layout, const void* activations, void* gradients,
                                              const int* ranges, int s_range, const int* flat_labels,
                                              const int* label_lengths, const int* input_lengths, int alphabet_size,
                                              int minibatch, void* costs_device, double grad_scale,
                                              rnntGradOptions grad_options, rnntLatticeOptions lattice_options,
                                              int rnnt_type, void* workspace, rnntOptions options) {
    if (!is_layout(layout)) return RNNT_STATUS_INVALID_VALUE;
    Call c = full_call(grad_scale, true, layout == RNNT_B200_LAYOUT_TUNV, grad_options);
    c.pruned = true;
    c.lattice = lattice_options;
    c.rnnt_type = rnnt_type;
    return run_as(dtype, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          costs_device, workspace, options, ranges, s_range}, c);
}
rnntStatus_t rnnt_b200_pruned_loss_async_lat(int dtype, int layout, const void* activations, void* gradients,
                                             const int* ranges, int s_range, const int* flat_labels,
                                             const int* label_lengths, const int* input_lengths, int alphabet_size,
                                             int minibatch, void* costs_device, double grad_scale,
                                             rnntGradOptions grad_options, rnntLatticeOptions lattice_options,
                                             void* workspace, rnntOptions options) {
    return rnnt_b200_pruned_loss_async_topo(dtype, layout, activations, gradients, ranges, s_range, flat_labels,
                                            label_lengths, input_lengths, alphabet_size, minibatch, costs_device,
                                            grad_scale, grad_options, lattice_options, RNNT_B200_RNNT_REGULAR,
                                            workspace, options);
}

rnntStatus_t rnnt_b200_pruned_forward_topo(int dtype, const void* activations, const int* ranges, int s_range,
                                           const int* flat_labels, const int* label_lengths, const int* input_lengths,
                                           int alphabet_size, int minibatch, void* costs_device, int prepare_backward,
                                           rnntLatticeOptions lattice_options, int rnnt_type, void* workspace,
                                           rnntOptions options) {
    Call c = forward_call(prepare_backward);
    c.pruned = true;
    c.lattice = lattice_options;
    c.rnnt_type = rnnt_type;
    return run_as(dtype, {activations, nullptr, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          costs_device, workspace, options, ranges, s_range}, c);
}
rnntStatus_t rnnt_b200_pruned_forward_lat(int dtype, const void* activations, const int* ranges, int s_range,
                                          const int* flat_labels, const int* label_lengths, const int* input_lengths,
                                          int alphabet_size, int minibatch, void* costs_device, int prepare_backward,
                                          rnntLatticeOptions lattice_options, void* workspace, rnntOptions options) {
    return rnnt_b200_pruned_forward_topo(dtype, activations, ranges, s_range, flat_labels, label_lengths,
                                         input_lengths, alphabet_size, minibatch, costs_device, prepare_backward,
                                         lattice_options, RNNT_B200_RNNT_REGULAR, workspace, options);
}

rnntStatus_t rnnt_b200_pruned_backward_topo(int dtype, const void* activations, void* gradients, const int* ranges,
                                            int s_range, const int* flat_labels, const int* label_lengths,
                                            const int* input_lengths, int alphabet_size, int minibatch,
                                            const void* grad_costs_device, double grad_scale,
                                            rnntGradOptions grad_options, rnntLatticeOptions lattice_options,
                                            int rnnt_type, void* workspace, rnntOptions options) {
    Call c = backward_call(grad_scale, grad_costs_device, grad_options);
    c.pruned = true;
    c.lattice = lattice_options;
    c.rnnt_type = rnnt_type;
    return run_as(dtype, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          nullptr, workspace, options, ranges, s_range}, c);
}
rnntStatus_t rnnt_b200_pruned_backward_lat(int dtype, const void* activations, void* gradients, const int* ranges,
                                           int s_range, const int* flat_labels, const int* label_lengths,
                                           const int* input_lengths, int alphabet_size, int minibatch,
                                           const void* grad_costs_device, double grad_scale,
                                           rnntGradOptions grad_options, rnntLatticeOptions lattice_options,
                                           void* workspace, rnntOptions options) {
    return rnnt_b200_pruned_backward_topo(dtype, activations, gradients, ranges, s_range, flat_labels, label_lengths,
                                          input_lengths, alphabet_size, minibatch, grad_costs_device, grad_scale,
                                          grad_options, lattice_options, RNNT_B200_RNNT_REGULAR, workspace, options);
}

// the joint's forward with smoothing and lattice options; the backward entries read the penalised factors
rnntStatus_t rnnt_b200_add_joint_forward_topo(const float* trans, const float* pred, const int* flat_labels,
                                              const int* label_lengths, const int* input_lengths, int alphabet_size,
                                              int minibatch, float* costs_device, int prepare_backward,
                                              rnntSmoothOptions smooth, rnntLatticeOptions lattice_options,
                                              int rnnt_type, void* workspace, rnntOptions options) {
    Call c = forward_call(prepare_backward);
    c.smooth = smooth;
    c.lattice = lattice_options;
    c.rnnt_type = rnnt_type;
    return run_add_joint({trans, nullptr, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          costs_device, workspace, options}, pred, nullptr, c);
}
rnntStatus_t rnnt_b200_add_joint_forward_lat(const float* trans, const float* pred, const int* flat_labels,
                                             const int* label_lengths, const int* input_lengths, int alphabet_size,
                                             int minibatch, float* costs_device, int prepare_backward,
                                             rnntSmoothOptions smooth, rnntLatticeOptions lattice_options,
                                             void* workspace, rnntOptions options) {
    return rnnt_b200_add_joint_forward_topo(trans, pred, flat_labels, label_lengths, input_lengths, alphabet_size,
                                            minibatch, costs_device, prepare_backward, smooth, lattice_options,
                                            RNNT_B200_RNNT_REGULAR, workspace, options);
}
// the joint's backward half of any topology, with gradient and smoothing options (the forward's)
rnntStatus_t rnnt_b200_add_joint_backward_topo(const float* trans, const float* pred, float* grad_trans,
                                               float* grad_pred, const int* flat_labels, const int* label_lengths,
                                               const int* input_lengths, int alphabet_size, int minibatch,
                                               const float* grad_costs_device, float grad_scale,
                                               rnntGradOptions grad_options, rnntSmoothOptions smooth, int rnnt_type,
                                               void* workspace, rnntOptions options) {
    if (grad_options.clamp != 0.0f) return RNNT_STATUS_INVALID_VALUE;   // as rnnt_b200_add_joint_backward_ex
    Call c = backward_call(grad_scale, grad_costs_device, grad_options);
    c.smooth = smooth;
    c.rnnt_type = rnnt_type;
    return run_add_joint({trans, grad_trans, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          nullptr, workspace, options}, pred, grad_pred, c);
}
// ---- additive joint network, logits never materialised -------------------------------------------
rnntStatus_t rnnt_b200_add_joint_loss(const float* trans, const float* pred, float* grad_trans,
                                      float* grad_pred, const int* flat_labels,
                                      const int* label_lengths, const int* input_lengths,
                                      int alphabet_size, int minibatch, float* costs_device,
                                      float grad_scale, void* workspace, rnntOptions options) {
    return run_add_joint({trans, grad_trans, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          costs_device, workspace, options}, pred, grad_pred, full_call(grad_scale));
}

rnntStatus_t rnnt_b200_add_joint_forward(const float* trans, const float* pred, const int* flat_labels,
                                         const int* label_lengths, const int* input_lengths,
                                         int alphabet_size, int minibatch, float* costs_device,
                                         int prepare_backward, void* workspace, rnntOptions options) {
    return run_add_joint({trans, nullptr, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          costs_device, workspace, options}, pred, nullptr, forward_call(prepare_backward));
}

rnntStatus_t rnnt_b200_add_joint_backward(const float* trans, const float* pred, float* grad_trans,
                                          float* grad_pred, const int* flat_labels,
                                          const int* label_lengths, const int* input_lengths,
                                          int alphabet_size, int minibatch, const float* grad_costs_device,
                                          float grad_scale, void* workspace, rnntOptions options) {
    return run_add_joint({trans, grad_trans, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          nullptr, workspace, options}, pred, grad_pred, backward_call(grad_scale, grad_costs_device));
}

rnntStatus_t rnnt_b200_add_joint_backward_ex(const float* trans, const float* pred, float* grad_trans,
                                             float* grad_pred, const int* flat_labels,
                                             const int* label_lengths, const int* input_lengths,
                                             int alphabet_size, int minibatch, const float* grad_costs_device,
                                             float grad_scale, rnntGradOptions grad_options, void* workspace,
                                             rnntOptions options) {
    // the joint's gradients are contractions over weights, never per-logit values: nothing to clip
    if (grad_options.clamp != 0.0f) return RNNT_STATUS_INVALID_VALUE;
    return run_add_joint({trans, grad_trans, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          nullptr, workspace, options}, pred, grad_pred,
                         backward_call(grad_scale, grad_costs_device, grad_options));
}

rnntStatus_t rnnt_b200_add_joint_workspace_size(int maxT, int maxU, int minibatch, int alphabet_size,
                                                size_t* size_bytes) {
    if (minibatch <= 0 || maxT <= 0 || maxU <= 0 || alphabet_size <= 0 || size_bytes == nullptr)
        return RNNT_STATUS_INVALID_VALUE;
    *size_bytes = carve_joint(nullptr, minibatch, maxT, maxU, alphabet_size).bytes;
    return RNNT_STATUS_SUCCESS;
}

// ---- smoothed additive joint (DESIGN.md §9) --------------------------------------------------------------
rnntStatus_t rnnt_b200_add_joint_smoothed_workspace_size(int maxT, int maxU, int minibatch, int alphabet_size,
                                                         size_t* size_bytes) {
    if (minibatch <= 0 || maxT <= 0 || maxU <= 0 || alphabet_size <= 0 || size_bytes == nullptr)
        return RNNT_STATUS_INVALID_VALUE;
    *size_bytes = carve_joint(nullptr, minibatch, maxT, maxU, alphabet_size, true).bytes;
    return RNNT_STATUS_SUCCESS;
}

rnntStatus_t rnnt_b200_add_joint_smoothed_forward(const float* trans, const float* pred, const int* flat_labels,
                                                  const int* label_lengths, const int* input_lengths,
                                                  int alphabet_size, int minibatch, float* costs_device,
                                                  int prepare_backward, rnntSmoothOptions smooth, void* workspace,
                                                  rnntOptions options) {
    Call c = forward_call(prepare_backward);
    c.smooth = smooth;
    return run_add_joint({trans, nullptr, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          costs_device, workspace, options}, pred, nullptr, c);
}

rnntStatus_t rnnt_b200_add_joint_smoothed_backward(const float* trans, const float* pred, float* grad_trans,
                                                   float* grad_pred, const int* flat_labels,
                                                   const int* label_lengths, const int* input_lengths,
                                                   int alphabet_size, int minibatch, const float* grad_costs_device,
                                                   float grad_scale, rnntGradOptions grad_options,
                                                   rnntSmoothOptions smooth, void* workspace, rnntOptions options) {
    if (grad_options.clamp != 0.0f) return RNNT_STATUS_INVALID_VALUE;   // as rnnt_b200_add_joint_backward_ex
    Call c = backward_call(grad_scale, grad_costs_device, grad_options);
    c.smooth = smooth;
    return run_add_joint({trans, grad_trans, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          nullptr, workspace, options}, pred, grad_pred, c);
}

// ---- pruned RNN-T loss (DESIGN.md §8): logits [N,maxT,R,V] over the windows `ranges` ---------------------
rnntStatus_t rnnt_b200_pruned_workspace_size(int maxT, int maxU, int s_range, int minibatch, size_t dtype_size,
                                             size_t* size_bytes) {
    if (minibatch <= 0 || maxT <= 0 || maxU <= 0 || s_range < 1 || size_bytes == nullptr)
        return RNNT_STATUS_INVALID_VALUE;
    if (dtype_size != sizeof(double)) dtype_size = sizeof(float);
    const size_t rows = (size_t)minibatch * maxT * s_range;
    const size_t lat = (size_t)minibatch * (maxT + maxU - 1) * maxU;
    *size_bytes = carve(nullptr, rows, lat, minibatch, maxU, dtype_size).bytes;
    return RNNT_STATUS_SUCCESS;
}

rnntStatus_t rnnt_b200_pruned_loss_async_ex(int dtype, int layout, const void* activations, void* gradients,
                                            const int* ranges, int s_range, const int* flat_labels,
                                            const int* label_lengths, const int* input_lengths, int alphabet_size,
                                            int minibatch, void* costs_device, double grad_scale,
                                            rnntGradOptions grad_options, void* workspace, rnntOptions options) {
    if (!is_layout(layout)) return RNNT_STATUS_INVALID_VALUE;
    Call c = full_call(grad_scale, true, layout == RNNT_B200_LAYOUT_TUNV, grad_options);
    c.pruned = true;
    return run_as(dtype, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          costs_device, workspace, options, ranges, s_range}, c);
}

rnntStatus_t rnnt_b200_pruned_forward(int dtype, const void* activations, const int* ranges, int s_range,
                                      const int* flat_labels, const int* label_lengths, const int* input_lengths,
                                      int alphabet_size, int minibatch, void* costs_device, int prepare_backward,
                                      void* workspace, rnntOptions options) {
    Call c = forward_call(prepare_backward);
    c.pruned = true;
    return run_as(dtype, {activations, nullptr, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          costs_device, workspace, options, ranges, s_range}, c);
}

rnntStatus_t rnnt_b200_pruned_backward_ex(int dtype, const void* activations, void* gradients, const int* ranges,
                                          int s_range, const int* flat_labels, const int* label_lengths,
                                          const int* input_lengths, int alphabet_size, int minibatch,
                                          const void* grad_costs_device, double grad_scale,
                                          rnntGradOptions grad_options, void* workspace, rnntOptions options) {
    Call c = backward_call(grad_scale, grad_costs_device, grad_options);
    c.pruned = true;
    return run_as(dtype, {activations, gradients, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
                          nullptr, workspace, options, ranges, s_range}, c);
}

rnntStatus_t rnnt_b200_add_joint_prune_ranges_topo(const int* label_lengths, const int* input_lengths, int minibatch,
                                                   int s_range, int* ranges, const void* workspace, int rnnt_type,
                                                   rnntOptions options) {
    if (rnnt_type != RNNT_B200_RNNT_REGULAR && rnnt_type != RNNT_B200_RNNT_MODIFIED) return RNNT_STATUS_INVALID_VALUE;
    const bool mod = rnnt_type == RNNT_B200_RNNT_MODIFIED;
    const int T = options.maxT, U = options.maxU, N = minibatch;
    if (!label_lengths || !input_lengths || !ranges || !workspace || N <= 0 || T <= 0 || U <= 0 || s_range < 2)
        return RNNT_STATUS_INVALID_VALUE;
    if (options.loc != RNNT_GPU || (uint64_t)N * T * U >= (1ull << 31) || U > 1024) return RNNT_STATUS_INVALID_VALUE;
    const size_t smem = prune_ranges_smem(T, U);
    int dev = 0, optin = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
        smem > (size_t)optin)
        return RNNT_STATUS_INVALID_VALUE;   // maxT beyond ~50k frames: the window starts no longer fit on chip
    const auto kernel = mod ? joint_prune_ranges_mod_kernel : joint_prune_ranges_kernel;
    if (smem > 48 * 1024)
        func_attr_once(reinterpret_cast<const void*>(kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const JointWorkspace w = carve_joint(const_cast<void*>(workspace), N, T, U, 1);   // lattice sections: V-free
    Tensors t{nullptr, nullptr, nullptr, label_lengths, input_lengths, 1, N, nullptr, nullptr, options};
    kernel<<<N, kRangeWarps * 32, smem, reinterpret_cast<cudaStream_t>(options.stream)>>>(
        w.lp2, w.alphas, w.betas, w.llf, input_lengths, label_lengths, ranges, make_dims(t, false), s_range);
    g_last_launches = 1;
    return cudaGetLastError() == cudaSuccess ? RNNT_STATUS_SUCCESS : RNNT_STATUS_EXECUTION_FAILED;
}
rnntStatus_t rnnt_b200_add_joint_prune_ranges(const int* label_lengths, const int* input_lengths, int minibatch,
                                              int s_range, int* ranges, const void* workspace, rnntOptions options) {
    return rnnt_b200_add_joint_prune_ranges_topo(label_lengths, input_lengths, minibatch, s_range, ranges, workspace,
                                                 RNNT_B200_RNNT_REGULAR, options);
}

// ---- forced alignment (DESIGN.md §12): the best path's label frames and score, on the device ---------------
rnntStatus_t rnnt_b200_align(int dtype, int layout, const void* activations, const int* flat_labels,
                             const int* label_lengths, const int* input_lengths, int alphabet_size, int minibatch,
                             int rnnt_type, int* frames, void* scores_device, void* workspace, rnntOptions options) {
    const bool tunv = layout == RNNT_B200_LAYOUT_TUNV;
    if (!is_layout(layout) || (tunv && is_16bit(dtype))) return RNNT_STATUS_INVALID_VALUE;
    Tensors t{activations, nullptr, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
              scores_device, workspace, options};
    t.frames = frames;
    return run_as(dtype, t, align_call(tunv, rnnt_type));
}
rnntStatus_t rnnt_b200_pruned_align(int dtype, const void* activations, const int* ranges, int s_range,
                                    const int* flat_labels, const int* label_lengths, const int* input_lengths,
                                    int alphabet_size, int minibatch, int rnnt_type, int* frames,
                                    void* scores_device, void* workspace, rnntOptions options) {
    Call c = align_call(false, rnnt_type);
    c.pruned = true;
    Tensors t{activations, nullptr, flat_labels, label_lengths, input_lengths, alphabet_size, minibatch,
              scores_device, workspace, options, ranges, s_range};
    t.frames = frames;
    return run_as(dtype, t, c);
}

// ---- the loss, gradient and alignment on caller-supplied factors (DESIGN.md §13) -------------------------------
rnntStatus_t rnnt_b200_lattice_workspace_size(int maxT, int maxU, int minibatch, size_t dtype_size,
                                              size_t* size_bytes) {
    if (minibatch <= 0 || maxT <= 0 || maxU <= 0 || size_bytes == nullptr) return RNNT_STATUS_INVALID_VALUE;
    if (dtype_size != sizeof(double)) dtype_size = sizeof(float);
    *size_bytes = carve(nullptr, 0, lattice_cells(minibatch, maxT, maxU), minibatch, maxU, dtype_size).bytes;
    return RNNT_STATUS_SUCCESS;
}

rnntStatus_t rnnt_b200_lattice_forward(int dtype, const void* px, const void* py, const int* label_lengths,
                                       const int* input_lengths, int minibatch, int rnnt_type, void* costs_device,
                                       int prepare_backward, void* workspace, rnntOptions options) {
    Call c = forward_call(prepare_backward);
    c.rnnt_type = rnnt_type;
    return run_lattice_as(dtype, {px, py, nullptr, nullptr, label_lengths, input_lengths, minibatch, costs_device,
                                  nullptr, workspace, options}, c);
}

rnntStatus_t rnnt_b200_lattice_backward(int dtype, void* px_grad, void* py_grad, const int* label_lengths,
                                        const int* input_lengths, int minibatch, int rnnt_type,
                                        const void* grad_costs_device, double grad_scale, void* workspace,
                                        rnntOptions options) {
    Call c = backward_call(grad_scale, grad_costs_device);
    c.rnnt_type = rnnt_type;
    return run_lattice_as(dtype, {nullptr, nullptr, px_grad, py_grad, label_lengths, input_lengths, minibatch, nullptr,
                                  nullptr, workspace, options}, c);
}

rnntStatus_t rnnt_b200_lattice_align(int dtype, const void* px, const void* py, const int* label_lengths,
                                     const int* input_lengths, int minibatch, int rnnt_type, int* frames,
                                     void* scores_device, void* workspace, rnntOptions options) {
    return run_lattice_as(dtype, {px, py, nullptr, nullptr, label_lengths, input_lengths, minibatch, scores_device,
                                  frames, workspace, options}, align_call(false, rnnt_type));
}

rnntStatus_t get_workspace_size(int maxT, int maxU, int minibatch, bool gpu, size_t* size_bytes,
                                size_t dtype_size) {
    if (minibatch <= 0 || maxT <= 0 || maxU <= 0 || size_bytes == nullptr)
        return RNNT_STATUS_INVALID_VALUE;  // reference src/rnnt_entrypoint.cpp:102-105
    if (dtype_size != sizeof(double)) dtype_size = sizeof(float);
    const size_t rows = (size_t)minibatch * maxT * maxU;
    if (!gpu) {
        // No CPU path here; the reference's figure (alphas, betas, 2-wide log-prob cache) is
        // returned so host-side sizing code keeps working.  src/rnnt_entrypoint.cpp:113-118
        *size_bytes = dtype_size * rows * 4;
        return RNNT_STATUS_SUCCESS;
    }
    const size_t lat = (size_t)minibatch * (maxT + maxU - 1) * maxU;
    *size_bytes = carve(nullptr, rows, lat, minibatch, maxU, dtype_size).bytes;
    return RNNT_STATUS_SUCCESS;
}

rnntStatus_t get_rnnt_workspace_size(int maxT, int maxU, int minibatch, bool gpu,
                                     size_t* size_bytes, size_t dtype_size) {
    return get_workspace_size(maxT, maxU, minibatch, gpu, size_bytes, dtype_size);
}

int rnnt_b200_last_launch_count(void) { return g_last_launches; }

// Debug / test hook: forward and backward log-likelihoods (natural log) left in a workspace by the last
// call that produced both lattices.  The reference asserts their agreement in debug builds
// (include/detail/cpu_rnnt.h:167-170).  Synchronises the device.
rnntStatus_t rnnt_b200_debug_log_likelihoods(const void* workspace, int maxT, int maxU, int minibatch,
                                             size_t dtype_size, double* llf_host, double* llb_host) {
    if (!workspace || !llf_host || !llb_host || maxT <= 0 || maxU <= 0 || minibatch <= 0)
        return RNNT_STATUS_INVALID_VALUE;
    if (dtype_size != sizeof(double)) dtype_size = sizeof(float);
    const size_t rows = (size_t)minibatch * maxT * maxU;
    const size_t lat = (size_t)minibatch * (maxT + maxU - 1) * maxU;
    const Workspace w = carve(const_cast<void*>(workspace), rows, lat, minibatch, maxU, dtype_size);
    std::vector<unsigned char> f((size_t)minibatch * 8), b((size_t)minibatch * 8);
    if (cudaDeviceSynchronize() != cudaSuccess) return RNNT_STATUS_EXECUTION_FAILED;
    if (cudaMemcpy(f.data(), w.llf, f.size(), cudaMemcpyDeviceToHost) != cudaSuccess ||
        cudaMemcpy(b.data(), w.llb, b.size(), cudaMemcpyDeviceToHost) != cudaSuccess)
        return RNNT_STATUS_MEMOPS_FAILED;
    for (int i = 0; i < minibatch; ++i) {
        if (dtype_size == sizeof(double)) {
            llf_host[i] = reinterpret_cast<const double*>(f.data())[i];
            llb_host[i] = reinterpret_cast<const double*>(b.data())[i];
        } else {
            const LogVal lf = reinterpret_cast<const LogVal*>(f.data())[i];
            const LogVal lb = reinterpret_cast<const LogVal*>(b.data())[i];
            llf_host[i] = ((double)lf.e + (double)lf.l) * 0.6931471805599453;
            llb_host[i] = ((double)lb.e + (double)lb.l) * 0.6931471805599453;
        }
    }
    return RNNT_STATUS_SUCCESS;
}

void rnnt_b200_set_profiling(int enabled) { g_profile = enabled != 0; }

int rnnt_b200_last_kernel_ms(float* ms3) {
    if (!ms3 || g_used == 0) return 0;
    return read_set(g_sets[g_used - 1], ms3);
}

int rnnt_b200_profile_collect(float* ms3_mean) {
    if (!ms3_mean) return 0;
    double acc[3] = {0, 0, 0};
    int cnt[3] = {0, 0, 0};
    for (size_t k = 0; k < g_used; ++k) {
        float ms[3];
        read_set(g_sets[k], ms);
        for (int i = 0; i < 3; ++i)
            if (ms[i] >= 0) {
                acc[i] += ms[i];
                ++cnt[i];
            }
    }
    for (int i = 0; i < 3; ++i) ms3_mean[i] = cnt[i] ? (float)(acc[i] / cnt[i]) : -1.0f;
    const int calls = (int)g_used;
    g_used = 0;
    return calls;
}

int rnnt_b200_debug_policy(int what, int a, int b) {
    switch (what) {
        case 0: return (size_t)a * (size_t)b > 512 || a <= 0 ? 0 : pick_tpr(a);
        case 1: {
            if ((size_t)a * (size_t)b > 512 || a <= 0) return 0;
            const int tpr = pick_tpr(a);
            return chunk_walk_cost(a, tpr, b, true) < chunk_walk_cost(a, tpr, b, false) ? 1 : 0;
        }
        case 2: return lattice_cols(a);
        case 3: return lattice_threads(a);
        case 4: return lattice_ring_depth(a, b != 0, hooks().lat_ring);
        case 5: return joint_slices(a);
        case 6: return (size_t)a * (size_t)b > 512 || a <= 0 ? 0 : chunk_hmajor(a, pick_tpr(a), b);
        case 7: return hooks().pdl ? 1 : 0;
        default: return -1;
    }
}

const char* rnnt_b200_build_info(void) { return "b200-rnnt sm_90a built " __DATE__ " " __TIME__; }

}  // extern "C"
