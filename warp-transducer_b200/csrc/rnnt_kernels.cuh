// rnnt_kernels.cuh — the three sm_90a kernels of the RNN-T loss + gradient path (each streaming
// pass comes as a CTA-per-row kernel for long rows and a register-tile kernel for short rows).
//
//   rowstats_*       pass 1 over the logits [N,T,U,V]: per lattice cell the log-softmax statistics
//                    (row max m, log sum exp(x-m)) and the two log-probs the lattice needs
//                    (blank, label y_u).      replaces reference reduce_max + reduce_exp
//                    (include/detail/reduce.h:45-146, gpu_rnnt.h:73-80) and the per-step logp()
//                    gathers (gpu_rnnt_kernel.h:5-9); analogue of CpuRNNT setup_probs (cpu_rnnt.h:115-128)
//   lattice_kernel   alpha and beta anti-diagonal wavefronts, one CTA per (utterance, direction),
//                    one thread per u, running concurrently.   replaces compute_alphas_kernel /
//                    compute_betas_kernel (gpu_rnnt_kernel.h:11-47,79-113)
//   grad_*           pass 2 over the logits: dense gradient w.r.t. logits, zeros on padded cells.
//                    replaces cudaMemsetAsync + compute_grad_kernel (gpu_rnnt.h:107-110,
//                    gpu_rnnt_kernel.h:143-179); REG instantiations add FastEmit and clamp (GradReg)
//
// HBM traffic: 4 B/elt (pass 1) + 8 B/elt (pass 2) + ~(16+16+16) B per lattice cell.
#pragma once
#include "rnnt_common.cuh"

namespace b200rnnt {

struct Dims {
    int N, maxT, maxU, V, blank;
    uint32_t rows;  // N*maxT*maxU  (< 2^31)
    FastDiv divU, divT, divN;
    int tmajor;     // 0: activations [N,T,U,V] (batch_first);  1: [T,U,N,V] (rnntOptions.batch_first == false,
                    // the layout reference include/detail/cpu_rnnt.h:139-144 indexes)
    // physical row index (position of the V-vector in the activation tensor) -> lattice coordinates
    __device__ __forceinline__ void decode(uint32_t r, uint32_t& b, uint32_t& t, uint32_t& u) const {
        if (tmajor) {
            uint32_t tu;
            divN.divmod(r, tu, b);
            divU.divmod(tu, t, u);
        } else {
            uint32_t bt;
            divU.divmod(r, bt, u);
            divT.divmod(bt, b, t);
        }
    }
};

// The factor array lp2 (and, on the fp64 path, alphas / betas) is stored DIAGONAL-MAJOR per utterance: cell (t,u)
// lives at (t+u)*maxU + u inside a block of (maxT+maxU-1)*maxU entries.  The wavefront kernel
// touches one anti-diagonal per step, so its loads and stores are contiguous across the u-threads
// (one or two 128-B lines per warp instead of 32 scattered sectors in the row-major form).
__host__ __device__ __forceinline__ size_t lattice_block(const Dims& d) {
    return (size_t)(d.maxT + d.maxU - 1) * d.maxU;
}
__device__ __forceinline__ size_t skew(const Dims& d, uint32_t b, uint32_t t, uint32_t u) {
    return (size_t)b * lattice_block(d) + (size_t)(t + u) * d.maxU + u;
}
// fp32 path: the transition factors (lp2) stay diagonal-major - the wavefront prefetches them a ring of
// diagonals ahead with one 16-byte copy per lane - but ALPHA and BETA are stored CELL-MAJOR [b][t][u],
// (t+1,u) at +maxU, (t,u+1) at +1: the consumer is pass 2, whose rows arrive in (b,t,u) order, so a warp's
// fetch of its rows' lattice values is one or two cache lines instead of one line per row (ncu, round 2:
// those scattered loads - not the element sweep - held the short-row gradient kernel's memory pipe).
// The wavefront pays with a strided 8-byte store per step, off its dependent chain.
__device__ __forceinline__ size_t cell(const Dims& d, uint32_t b, uint32_t t, uint32_t u) {
    return ((size_t)b * d.maxT + t) * d.maxU + u;
}

// clamp the per-utterance extents into the tensor so corrupt lengths cannot index outside it
__device__ __forceinline__ void utt_extent(const Dims& d, const int* __restrict__ xlen,
                                           const int* __restrict__ ylen, int b, int& T, int& U) {
    T = min(max(__ldg(xlen + b), 1), d.maxT);
    U = min(max(__ldg(ylen + b) + 1, 1), d.maxU);
}

// ---- pruned logits (DESIGN.md §8) -----------------------------------------------------------------------
// Each streaming kernel takes `bool PRUNED` as its last template parameter and a Prune by value as its last
// argument.  Pruned logits are [N, maxT, R, V]: row (b, t, s) holds lattice cell (t, u = ranges[b*maxT + t] + s),
// and Dims.rows counts those rows.  The dense instantiations get ranges == NULL and never read the Prune.
struct Prune {
    const int* ranges;   // [N, maxT] window start per frame (any int32)
    FastDiv divR;        // R = rows per frame
};
// row -> (b, t, u).  Pruned: u is ranges + s in 32-bit two's complement; a negative or too large u lands at or
// above 2^31 as unsigned, where row_padding() catches it together with u >= U_b
template <bool PRUNED>
__device__ __forceinline__ void row_decode(const Dims d, const Prune p, uint32_t r, uint32_t& b, uint32_t& t,
                                           uint32_t& u) {
    if constexpr (PRUNED) {
        uint32_t bt, s;
        p.divR.divmod(r, bt, s);
        d.divT.divmod(bt, b, t);
        u = (uint32_t)__ldg(p.ranges + bt) + s;
    } else {
        d.decode(r, b, t, u);
    }
}
template <bool PRUNED> __device__ __forceinline__ bool row_padding(uint32_t t, uint32_t u, int Tb, int Ub) {
    if constexpr (PRUNED) return (int)t >= Tb || u >= (uint32_t)Ub;
    else return (int)t >= Tb || (int)u >= Ub;
}
// An utterance without a path through its pruned lattice (log-likelihood log zero) gets a zero gradient.  Only the
// pruned instantiations ask: a dense lattice always has a path.
__device__ __forceinline__ bool ll_dead(const LogVal* llf, uint32_t b) { return llf[b].e < kEDead; }
__device__ __forceinline__ bool ll_dead(const double* llf, uint32_t b) { return llf[b] == -(double)INFINITY; }
// padding of pass 2 in the pruned instantiations: row_padding, and every row of an utterance without a path.  The
// dense instantiations spell out their test, t >= T_b or u >= U_b, where they use it: returned from a helper, it
// compiled to other index code in every dense gradient kernel, and grad_row_kernel<float, 4, 5> (C3) ran 0.9 %
// slower (H100 80GB HBM3, 400 W).
template <typename Val>
__device__ __forceinline__ bool pruned_grad_padding(uint32_t t, uint32_t u, int Tb, int Ub, const Val* llf, uint32_t b) {
    return row_padding<true>(t, u, Tb, Ub) || ll_dead(llf, b);
}
// padding of pass 2 in the dense MOD instantiations: a modified lattice (DESIGN.md §11) has no path when
// U_b - 1 > T_b, so they ask ll_dead as the pruned ones do.  (The regular ones keep the test spelled out.)
template <typename Val>
__device__ __forceinline__ bool mod_grad_padding(uint32_t t, uint32_t u, int Tb, int Ub, const Val* llf, uint32_t b) {
    return (int)t >= Tb || (int)u >= Ub || ll_dead(llf, b);
}

// ---- delay penalty (DESIGN.md §10) ----------------------------------------------------------------------
// Each streaming kernel has a twin *_delay_kernel running the same body at DELAY = true.  Pass 1 adds
// lambda ((T_b - 1)/2 - t) to the label log-factor of every cell with a label transition; pass 2 adds the same
// penalty, in the exp2 domain, to the label offset cL.  The bracket is exact in T (t < 2^24), so the only
// rounding is the product with lambda.  The plain kernels run the body at DELAY = false and keep their code.
template <typename T> __device__ __forceinline__ T delay_bracket(int Tb, uint32_t t) {
    return T(Tb - 1) * T(0.5) - T(t);
}

// Pruned calls start from log-zero factors everywhere, so that a cell no row covers has neither transition; pass 1
// then writes the covered cells.  (has_label = true: the fp64 factor keeps its label log-prob only then.)
template <typename T>
__global__ void __launch_bounds__(256) lattice_fill_kernel(typename Lat<T>::fac* __restrict__ lp2, size_t n) {
    const typename Lat<T>::fac z = Lat<T>::make(Real<T>::neg_inf(), Real<T>::neg_inf(), true);
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (size_t)gridDim.x * 256) lp2[i] = z;
}

// =================================================================================================
// Pass 1, long rows: ONE CTA PER ROW, non-persistent grid (grid = N*T*U blocks of 256 threads).
// A short-lived block that issues all its loads and retires streams faster than a persistent grid-stride
// loop over the same bytes (tools/probe/bw_probe.cu compares the two) - block turnover keeps the DRAM
// access window compact.
// Thread i owns vectors i, i+256, ... (NV per trip, all loads issued before first use; one trip
// when V/VEC <= 256*NV, i.e. V <= 8192 in fp32).  Per trip the statistics are the exact two-pass
// max / sum exp(x-max) from registers; trips are merged online.  Block combine: warp shuffles, one
// shared-memory exchange, one __syncthreads.
// =================================================================================================
// threads per CTA-per-row block: 256 for 4/8-byte logits, 128 for 16-bit logits (a 16-bit row is
// half as long, so the smaller block keeps ~5 16-B loads in flight per thread)
template <typename IO> struct RowThreads { static constexpr int value = sizeof(IO) >= 4 ? 256 : 128; };

#ifndef RNNT_ROWSTATS_MINB
#define RNNT_ROWSTATS_MINB 7
#endif
template <typename T, int VEC, int NV, typename IO, bool PRUNED, bool DELAY>
__device__ __forceinline__ void rowstats_row(const IO* __restrict__ acts, const int* __restrict__ labels,
                                             const int* __restrict__ xlen, const int* __restrict__ ylen,
                                             typename Real<T>::pair* __restrict__ stat,
                                             typename Lat<T>::fac* __restrict__ lp2, const Dims d, const Prune p,
                                             const T delay) {
    using R = Real<T>;
    constexpr int kRowThreads = RowThreads<IO>::value;
    __shared__ T sh_m[kRowThreads / 32], sh_s[kRowThreads / 32];
    pdl_trigger();   // the lattice kernel may be launched as soon as every CTA of this grid has started
    const uint32_t r = blockIdx.x;
    uint32_t u, b, t;
    row_decode<PRUNED>(d, p, r, b, t, u);
    int Tb, Ub;
    utt_extent(d, xlen, ylen, b, Tb, Ub);
    if (row_padding<PRUNED>(t, u, Tb, Ub)) return;  // padded cell: nothing to read (block-uniform)
    const int nv = d.V / VEC;
    const IO* row = acts + (uint64_t)r * d.V;
    T m = R::neg_inf(), s = 0;
    if constexpr (sizeof(IO) == 2 && VEC >= 2) {
        // 16-bit logits (issue-bound, not DRAM-bound: ncu round 2, 11.5 instructions per element at 75 % issue
        // activity).  The trip's maximum is taken on the PACKED words (two elements per HMNMX2, no conversion);
        // every element is converted once, for its exponential, and the exponent is one FFMA:
        // 2^(x*log2e - fl(m*log2e)).  The rounding of m*log2e is |m| * 6e-8 in the exponent - three orders
        // below the 16-bit input quantisation (the fp32 path keeps the exact (x - m) form).
        using P = typename Pack<sizeof(IO) * VEC>::type;
        using H = Packed16<IO>;
        constexpr int W = VEC / 2;
        for (int base = threadIdx.x; base < nv; base += kRowThreads * NV) {
            union { P p; unsigned w[W]; } raw[NV];
#pragma unroll
            for (int j = 0; j < NV; ++j) {
                const int i = base + j * kRowThreads;
                if (i < nv) {
                    raw[j].p = __ldg(reinterpret_cast<const P*>(row + (size_t)i * VEC));
                } else {
#pragma unroll
                    for (int c = 0; c < W; ++c) raw[j].w[c] = H::kNegInf2;
                }
            }
            unsigned m2 = raw[0].w[0];
#pragma unroll
            for (int j = 0; j < NV; ++j)
#pragma unroll
                for (int c = 0; c < W; ++c) m2 = H::max2(m2, raw[j].w[c]);
            float mlo, mhi;
            H::to_floats(m2, mlo, mhi);
            const float vm = fmaxf(mlo, mhi);
            if (vm > m) {
                s *= R::exp(m - vm);
                m = vm;
            }
            const float negML = -((m == R::neg_inf()) ? 0.0f : m) * R::kLog2e;
#pragma unroll
            for (int j = 0; j < NV; ++j)
#pragma unroll
                for (int c = 0; c < W; ++c) {
                    float lo, hi;
                    H::to_floats(raw[j].w[c], lo, hi);
                    s += R::exp2(fmaf(lo, R::kLog2e, negML));
                    s += R::exp2(fmaf(hi, R::kLog2e, negML));
                }
        }
    } else
    for (int base = threadIdx.x; base < nv; base += kRowThreads * NV) {
        VecT<T, VEC> x[NV];
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const int i = base + j * kRowThreads;
            if (i < nv) {
                x[j] = ld_keep<T, VEC>(row + (size_t)i * VEC);
            } else {
#pragma unroll
                for (int c = 0; c < VEC; ++c) x[j].v[c] = R::neg_inf();
            }
        }
        T vm = x[0].v[0];
#pragma unroll
        for (int j = 0; j < NV; ++j)
#pragma unroll
            for (int c = 0; c < VEC; ++c) vm = R::max(vm, x[j].v[c]);
        if (vm > m) {
            s *= R::exp(m - vm);
            m = vm;
        }
        const T mm = (m == R::neg_inf()) ? T(0) : m;
#pragma unroll
        for (int j = 0; j < NV; ++j)
#pragma unroll
            for (int c = 0; c < VEC; ++c) s += R::exp(x[j].v[c] - mm);
    }
    // warp combine, then the 8 warp results through shared memory
    const T Mw = group_max<32>(m);
    const T Sw = group_sum<32>((m == R::neg_inf()) ? T(0) : s * R::exp(m - Mw));
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) {
        sh_m[warp] = Mw;
        sh_s[warp] = Sw;
    }
    __syncthreads();
    if (warp == 0) {
        constexpr int NW = kRowThreads / 32;
        const T mw = lane < NW ? sh_m[lane] : R::neg_inf();
        const T sw = lane < NW ? sh_s[lane] : T(0);
        const T M = group_max<NW>(mw);
        const T S = group_sum<NW>((mw == R::neg_inf()) ? T(0) : sw * R::exp(mw - M));
        if (lane == 0) {
            const T lse = R::log(S);
            typename R::pair st;
            st.x = M;
            st.y = lse;
            stat[r] = st;
            const T lpb = (ld_scalar<T>(row + d.blank) - M) - lse;
            T lpl = 0;
            const bool has_label = (int)u < Ub - 1;
            if (has_label) {
                const int y = __ldg(labels + (size_t)b * (d.maxU - 1) + u);
                lpl = (ld_scalar<T>(row + y) - M) - lse;
                if (DELAY) lpl += delay * delay_bracket<T>(Tb, t);
            }
            lp2[skew(d, b, t, u)] = Lat<T>::make(lpb, lpl, has_label);
        }
    }
}
template <typename T, int VEC, int NV, typename IO, bool PRUNED>
__global__ void __launch_bounds__(RowThreads<IO>::value, (sizeof(IO) >= 4 ? RNNT_ROWSTATS_MINB : 8))
rowstats_row_kernel(const IO* __restrict__ acts, const int* __restrict__ labels,
                    const int* __restrict__ xlen, const int* __restrict__ ylen,
                    typename Real<T>::pair* __restrict__ stat, typename Lat<T>::fac* __restrict__ lp2,
                    const Dims d, const Prune p) {
    rowstats_row<T, VEC, NV, IO, PRUNED, false>(acts, labels, xlen, ylen, stat, lp2, d, p, T(0));
}
template <typename T, int VEC, int NV, typename IO, bool PRUNED>
__global__ void __launch_bounds__(RowThreads<IO>::value, (sizeof(IO) >= 4 ? RNNT_ROWSTATS_MINB : 8))
rowstats_row_delay_kernel(const IO* __restrict__ acts, const int* __restrict__ labels,
                          const int* __restrict__ xlen, const int* __restrict__ ylen,
                          typename Real<T>::pair* __restrict__ stat, typename Lat<T>::fac* __restrict__ lp2,
                          const Dims d, const Prune p, const T delay) {
    rowstats_row<T, VEC, NV, IO, PRUNED, true>(acts, labels, xlen, ylen, stat, lp2, d, p, delay);
}

// =================================================================================================
// Pass 1, short rows (V/VEC <= 8*LPR): the whole row lives in registers — each of the LPR lanes
// of a row holds up to kVPL vectors, all loads are issued before the first use (32*kVPL*16 B in
// flight per warp whatever V is), and the statistics are the exact two-pass max / sum exp(x-max).
// Small LPR keeps the per-row bookkeeping (index decode, length checks, lattice stores) off most
// lanes: at V=28 two lanes own a row, at V=50 (float2) four do.
// =================================================================================================
#ifndef RNNT_VPL
#define RNNT_VPL 8
#endif
constexpr int kVPL = RNNT_VPL;

template <typename T, int VEC, int LPR, typename IO, bool PRUNED, bool DELAY>
__device__ __forceinline__ void rowstats_tile(const IO* __restrict__ acts, const int* __restrict__ labels,
                                              const int* __restrict__ xlen, const int* __restrict__ ylen,
                                              typename Real<T>::pair* __restrict__ stat,
                                              typename Lat<T>::fac* __restrict__ lp2, const Dims d, const Prune p,
                                              const T delay) {
    using R = Real<T>;
    constexpr int RPW = kWarp / LPR;
    const int lane = threadIdx.x & 31;
    const int sub = lane / LPR, sl = lane % LPR;
    const uint64_t gw = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int nv = d.V / VEC;
    pdl_trigger();

    {   // non-persistent: one tile of RPW rows per warp (see rowstats_row_kernel for why)
        const uint64_t r0 = gw * RPW;
        const uint32_t r = (uint32_t)r0 + sub;
        bool valid = r0 + sub < d.rows;
        uint32_t u = 0, b = 0, t = 0;
        int Tb = 0, Ub = 0;
        if (valid) {
            row_decode<PRUNED>(d, p, r, b, t, u);
            utt_extent(d, xlen, ylen, b, Tb, Ub);
            valid = !row_padding<PRUNED>(t, u, Tb, Ub);
        }
        const IO* row = acts + (uint64_t)r * d.V;
        VecT<T, VEC> x[kVPL];
#pragma unroll
        for (int j = 0; j < kVPL; ++j) {
            const int i = sl + j * LPR;
            if (valid && i < nv) {
                x[j] = ld_keep<T, VEC>(row + (size_t)i * VEC);
            } else {
#pragma unroll
                for (int c = 0; c < VEC; ++c) x[j].v[c] = R::neg_inf();
            }
        }
        T m = x[0].v[0];
#pragma unroll
        for (int j = 0; j < kVPL; ++j)
#pragma unroll
            for (int c = 0; c < VEC; ++c) m = R::max(m, x[j].v[c]);
        const T M = group_max<LPR>(m);
        const ExpSum<T> es((M == R::neg_inf()) ? T(0) : M);
        T s = 0;
#pragma unroll
        for (int j = 0; j < kVPL; ++j)
#pragma unroll
            for (int c = 0; c < VEC; ++c) s += es.term(x[j].v[c]);
        const T S = group_sum<LPR>(s);
        if (valid && sl == 0) {
            const T lse = es.log_of(S);
            typename R::pair st;
            st.x = M;
            st.y = lse;
            stat[r] = st;
            const T lpb = (ld_scalar<T>(row + d.blank) - M) - lse;
            T lpl = 0;
            const bool has_label = (int)u < Ub - 1;
            if (has_label) {
                const int y = __ldg(labels + (size_t)b * (d.maxU - 1) + u);
                lpl = (ld_scalar<T>(row + y) - M) - lse;
                if (DELAY) lpl += delay * delay_bracket<T>(Tb, t);
            }
            lp2[skew(d, b, t, u)] = Lat<T>::make(lpb, lpl, has_label);
        }
    }
}
template <typename T, int VEC, int LPR, typename IO, bool PRUNED>
__global__ void __launch_bounds__(256)
rowstats_tile_kernel(const IO* __restrict__ acts, const int* __restrict__ labels,
                     const int* __restrict__ xlen, const int* __restrict__ ylen,
                     typename Real<T>::pair* __restrict__ stat,
                     typename Lat<T>::fac* __restrict__ lp2, const Dims d, const Prune p) {
    rowstats_tile<T, VEC, LPR, IO, PRUNED, false>(acts, labels, xlen, ylen, stat, lp2, d, p, T(0));
}
template <typename T, int VEC, int LPR, typename IO, bool PRUNED>
__global__ void __launch_bounds__(256)
rowstats_tile_delay_kernel(const IO* __restrict__ acts, const int* __restrict__ labels,
                           const int* __restrict__ xlen, const int* __restrict__ ylen,
                           typename Real<T>::pair* __restrict__ stat,
                           typename Lat<T>::fac* __restrict__ lp2, const Dims d, const Prune p, const T delay) {
    rowstats_tile<T, VEC, LPR, IO, PRUNED, true>(acts, labels, xlen, ylen, stat, lp2, d, p, delay);
}

// =================================================================================================
// Lattice DP.  grid = (N, 2): blockIdx.y 0 -> alpha (forward), 1 -> beta (backward); the two
// directions of an utterance run concurrently on different SMs.  One thread per u; anti-diagonal
// n = t + u is the step index, so thread u handles cell (n - u, u) at step n.
//
//  * The (blank,label) log-prob pairs of the next kRing-2 diagonals are in flight as cp.async
//    copies into a shared-memory ring (the lattice is diagonal-major, so a diagonal is one
//    contiguous run).  cp.async completion is counted in order (wait_group), unlike register
//    prefetches whose scoreboard slots alias and collapse the prefetch distance to one step.
//  * The u-1 (u+1) neighbour's running value comes by warp shuffle; across warps through a
//    double-buffered shared slot and ONE __syncthreads per diagonal (a __syncwarp when maxU <= 32).
//  * Boundary cells need no branches: a column starts from -inf (alpha) so "stay" vanishes at
//    t = 0, the emit log-prob is forced to -inf at u = 0 (alpha) / u = U-1 (beta), and beta's
//    virtual cell beta(T, U-1) = 0 makes the terminal cell fall out of the same recurrence.
//  * alpha/beta are carried and stored in double; the dependent chain per step is
//    SHFL -> DADD -> DADD -> F2F -> FMNMX/FMUL -> MUFU.EX2 -> FADD -> MUFU.LG2 -> FMUL -> F2F -> DADD.
// =================================================================================================
constexpr int kRing = 8;
constexpr int kLatticeStaticSmem = 2 * 32 * (int)sizeof(double);   // lattice_kernel's `edge` exchange slots

template <int BYTES>
__device__ __forceinline__ void cp_async(void* smem_dst, const void* gmem_src) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(d), "l"(gmem_src), "n"(BYTES) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// log(e^x + e^y) for the lattice: doubles in/out, correction term in the caller's precision.
template <typename T> __device__ __forceinline__ double lse2(double x, double y) {
    if (sizeof(T) == 4) {
        const float df = (float)(x - y);          // +-inf when one side is -inf, NaN when both are
        // (-inf) - (-inf) is the only legitimate NaN here; a NaN operand (a NaN logit upstream)
        // must reach the cost, as the reference's log_plus lets it (rnnt_helper.h:16-24)
        if (!(df == df)) return (x == y) ? x : x + y;
        const double mx = df > 0.0f ? x : y;
        const float nd = -fabsf(df) * 1.4426950408889634f;
        float e, l;
        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(nd));
        asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(1.0f + e));
        return mx + (double)(l * 0.6931471805599453f);
    } else {
        if (x != x || y != y) return x + y;   // fmax/fmin drop a NaN operand; the reference's log_plus keeps it
        const double mx = fmax(x, y), mn = fmin(x, y);
        if (mx == -(double)INFINITY) return mx;
        return mx + log1p(::exp(mn - mx));
    }
}

// MOD: the modified topology (DESIGN.md §11).  The label term of cell (t,u) comes from (t-1,u-1) (alpha) /
// (t+1,u+1) (beta), which the neighbouring thread held one step before the value it offers today: alpha offers
// `off` = alpha + lp_label of its cell on the previous diagonal, beta offers `bprev` = its value of one step
// earlier.  Alpha runs one diagonal further, to the virtual cell (T, U-1), the log-likelihood.
template <typename T, bool MULTI, bool MOD>
__device__ __forceinline__ void lattice_body(const typename Real<T>::pair* __restrict__ lp2, const int* __restrict__ xlen,
                                             const int* __restrict__ ylen, double* __restrict__ alphas,
                                             double* __restrict__ betas, double* __restrict__ llf,
                                             double* __restrict__ llb, T* __restrict__ costs, const Dims& d,
                                             unsigned char* ring_raw, double (*edge)[32]) {
    using P = typename Real<T>::pair;
    constexpr double NINF = -(double)INFINITY;
    P* ring = reinterpret_cast<P*>(ring_raw);  // [kRing][blockDim.x]
    const int b = blockIdx.x;
    const int u = threadIdx.x;
    const int NT = blockDim.x;
    const int lane = u & 31, warp = u >> 5;
    const int nwarps = NT >> 5;
    int Tb, Ub;
    utt_extent(d, xlen, ylen, b, Tb, Ub);
    pdl_trigger();
    pdl_wait();   // pass 1's factors are complete
    const size_t base = (size_t)b * lattice_block(d);
    const int last = Tb + Ub - 2;
    const int mU = d.maxU;
    // thread u owns one cell on each diagonal dg with 0 <= dg - u < width (width = 0: no column)
    const unsigned width = u < Ub ? (unsigned)Tb : 0u;
    const P* lp_u = lp2 + base + u;  // diagonal-major: lp_u[dg*mU] = cell (dg-u, u)
    const unsigned ring_elems = kRing * NT;
    // All per-step addresses are carried as running pointers / wrapped slot offsets: the step loop
    // is one warp per scheduler, so every integer instruction is exposed latency.

    if (blockIdx.y == 0) {
        // ------------------------------------------------------------------ alpha
        double* sp = alphas + base + u;  // store pointer, advances one diagonal per step
        double a = (u == 0) ? 0.0 : NINF;  // alpha(t-1, u) of this thread's column
        if (u == 0) *sp = 0.0;
        const P* gp = lp_u;  // next diagonal to fetch
        unsigned fslot = u, fdg = 0;
#pragma unroll
        for (int k = 0; k < kRing - 1; ++k) {
            if (fdg - (unsigned)u < width) cp_async<sizeof(P)>(&ring[fslot], gp);
            cp_async_commit();
            gp += mU;
            ++fdg;
            fslot += NT;
        }
        unsigned rslot = u;  // slot of diagonal n-1
        double off = NINF, ll_mod = NINF;   // MOD only
        for (int n = 1; n <= last + (MOD ? 1 : 0); ++n) {
            cp_async_wait<kRing - 2>();  // diagonal n-1 has landed (this thread's part)
            if (MULTI) {
                if (lane == 31) edge[n & 1][warp] = MOD ? off : a;
                __syncthreads();
            } else {
                __syncwarp();
            }
            // fetch diagonal n+kRing-2 into the slot of diagonal n-2, which nobody reads any more
            if (fdg - (unsigned)u < width) cp_async<sizeof(P)>(&ring[fslot], gp);
            cp_async_commit();
            gp += mU;
            ++fdg;
            fslot += NT;
            if (fslot >= ring_elems) fslot -= ring_elems;
            double a_left = __shfl_up_sync(0xffffffffu, MOD ? off : a, 1);
            if (MULTI && lane == 0 && warp > 0) a_left = edge[n & 1][warp - 1];
            sp += mU;
            if (MOD) {
                // alpha(t,u) = lse(alpha(t-1,u) + lp_blank(t-1,u), alpha(t-1,u-1) + lp_label(t-1,u-1))
                const P* slot = ring + rslot;   // this column's cell (n-1-u, u)
                const bool prev_on = (unsigned)(n - 1 - u) < width;
                const double left = u > 0 ? a_left : NINF;
                const double stay = prev_on ? a + (double)slot[0].x : NINF;
                const double a_prev = a;
                if ((unsigned)(n - u) < width) {
                    a = lse2<T>(stay, left);
                    *sp = a;
                } else if (n == last + 1 && u == Ub - 1) {
                    ll_mod = lse2<T>(stay, left);   // the virtual cell (T, U-1)
                }
                off = prev_on && u < Ub - 1 ? a_prev + (double)slot[0].y : NINF;
            } else if ((unsigned)(n - u) < width) {
                const P* slot = ring + rslot;
                const T sx = n > u ? slot[0].x : T(0);                   // lp_blank(t-1, u)
                const T ey = u > 0 ? slot[-1].y : Real<T>::neg_inf();    // lp_label(t, u-1)
                a = lse2<T>(a + (double)sx, a_left + (double)ey);
                *sp = a;
            }
            rslot += NT;
            if (rslot >= ring_elems) rslot -= ring_elems;
        }
        if (u == Ub - 1) {
            cp_async_wait<0>();
            const double ll = MOD ? ll_mod : a + (double)lp_u[(size_t)last * mU].x;
            llf[b] = ll;
            costs[b] = (T)(-ll);
        }
    } else {
        // ------------------------------------------------------------------ beta
        double* sp = betas + base + u + (size_t)last * mU;
        double bv = (u == Ub - 1) ? 0.0 : NINF;  // beta(t+1, u); virtual beta(T, U-1) = 0
        const P* gp = lp_u + (size_t)last * mU;
        unsigned fslot = (unsigned)(last & (kRing - 1)) * NT + u;
        int fdg = last;
        const unsigned rstart = fslot;
#pragma unroll
        for (int k = 0; k < kRing - 1; ++k) {
            if ((unsigned)(fdg - u) < width) cp_async<sizeof(P)>(&ring[fslot], gp);
            cp_async_commit();
            gp -= mU;
            --fdg;
            fslot = fslot >= (unsigned)NT ? fslot - NT : fslot + ring_elems - NT;
        }
        unsigned rslot = rstart;  // slot of diagonal n
        double bprev = NINF;      // MOD: bv of one step earlier, beta(t+1,u+1) for the thread u-1
        for (int n = last; n >= 0; --n) {
            cp_async_wait<kRing - 2>();  // this thread's cell of diagonal n has landed
            if (MULTI) {
                if (lane == 0) edge[n & 1][warp] = MOD ? bprev : bv;
                __syncthreads();
            }
            // slot of diagonal n+1: written and read by this thread only
            if ((unsigned)(fdg - u) < width) cp_async<sizeof(P)>(&ring[fslot], gp);
            cp_async_commit();
            gp -= mU;
            --fdg;
            fslot = fslot >= (unsigned)NT ? fslot - NT : fslot + ring_elems - NT;
            double b_right = __shfl_down_sync(0xffffffffu, MOD ? bprev : bv, 1);
            if (MULTI && lane == 31 && warp + 1 < nwarps) b_right = edge[n & 1][warp + 1];
            const double bold = bv;
            if ((unsigned)(n - u) < width) {
                const P p = ring[rslot];
                const T py = u < Ub - 1 ? p.y : Real<T>::neg_inf();
                bv = lse2<T>(bv + (double)p.x, b_right + (double)py);
                *sp = bv;
            }
            if (MOD) bprev = bold;
            sp -= mU;
            rslot = rslot >= (unsigned)NT ? rslot - NT : rslot + ring_elems - NT;
        }
        if (u == 0) llb[b] = bv;
    }
}
template <typename T, bool MULTI>
__global__ void __launch_bounds__(1024)
lattice_kernel(const typename Real<T>::pair* __restrict__ lp2, const int* __restrict__ xlen,
               const int* __restrict__ ylen, double* __restrict__ alphas,
               double* __restrict__ betas, double* __restrict__ llf, double* __restrict__ llb,
               T* __restrict__ costs, const Dims d) {
    extern __shared__ __align__(16) unsigned char ring_raw[];
    __shared__ double edge[2][32];
    lattice_body<T, MULTI, false>(lp2, xlen, ylen, alphas, betas, llf, llb, costs, d, ring_raw, edge);
}
template <typename T, bool MULTI>
__global__ void __launch_bounds__(1024)
lattice_mod_kernel(const typename Real<T>::pair* __restrict__ lp2, const int* __restrict__ xlen,
                   const int* __restrict__ ylen, double* __restrict__ alphas,
                   double* __restrict__ betas, double* __restrict__ llf, double* __restrict__ llb,
                   T* __restrict__ costs, const Dims d) {
    extern __shared__ __align__(16) unsigned char ring_raw[];
    __shared__ double edge[2][32];
    lattice_body<T, MULTI, true>(lp2, xlen, ylen, alphas, betas, llf, llb, costs, d, ring_raw, edge);
}

// =================================================================================================
// Pass 2: dense gradient w.r.t. the logits, rows visited in reverse so the tail of pass 1 is met
// first in L2.
//   g_k = scale * ( e^{lp_k + alpha + beta - ll}
//                   - [k = blank, t < T-1]          e^{lp_k + alpha + beta(t+1,u) - ll}
//                   - [k = blank, t = T-1, u = U-1] e^{lp_k + alpha - ll}
//                   - [k = y_u,  u < U-1]           e^{lp_k + alpha + beta(t,u+1) - ll} )
// (reference gpu_rnnt_kernel.h:159-177), lp_k = (x_k - m) - lse.  The three per-row offsets are
// formed once per row in double and rounded (exp2 domain); per element the work is
// FADD (x-m), FFMA, MUFU.EX2 (+ FMUL when scale != 1).  The two special lanes (blank, label)
// are patched per VECTOR, not per element.  Padded rows are written as zeros here (no memset pass).
// =================================================================================================
// Per-row constants of the gradient: offsets in the exp2 domain (see the pass-2 header above).
template <typename T> struct RowGrad {
    T m, cA, cB, cL;
    int y;
};

// Gradient regularisers (include/rnnt.h rnntGradOptions), instantiated only in the REG = true kernels.
//   FastEmit(lambda): g_k = p_k (occ + lambda e_y) - [k = blank] e_b - [k = y] (1 + lambda) e_y, i.e. the dense
//   offset becomes cA' = log2(2^cA + lambda 2^(cL + log2 p_y)) and the label offset cL' = cL + log2(1 + lambda).
//   Both offsets carry -lse log2e, so 2^(cL + log2 p_y) = e_y e^-lse is normalised like 2^cA = occ e^-lse.
//   log2 p_y comes from the lattice factor lp2 of the cell (one 16-byte load per row), not from the logits.
//   clamp: the final per-utterance gradient is clipped to [-clamp, clamp] before grad_scale * grad_costs[b].
template <typename T> struct GradReg {
    const typename Lat<T>::fac* lp2;   // the cell's (blank, label) factors, diagonal-major (skew)
    T log2_lam;                        // log2(lambda); -inf when FastEmit is off
    T log2_1p_lam;                     // log2(1 + lambda)
    T clamp;                           // +inf when clamping is off
};
__device__ __forceinline__ float fac_label_log2(const float4 f) {
    float l;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(f.z));
    return (float)__float_as_int(f.w) + l;
}
__device__ __forceinline__ double fac_label_log2(const double2 f) { return f.y * Real<double>::kLog2e; }
__device__ __forceinline__ float log2_of(float x) {
    float l;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(x));
    return l;
}
__device__ __forceinline__ double log2_of(double x) { return ::log2(x); }
// per-row FastEmit fold of the offsets (before the 16-bit path's ZEROM fold of -m log2e)
template <typename T>
__device__ __forceinline__ void fastemit_fold(RowGrad<T>& g, const GradReg<T>& reg, uint32_t b, uint32_t t, uint32_t u,
                                              const Dims& d) {
    using R = Real<T>;
    if (g.y < 0 || !(reg.log2_lam > R::neg_inf())) return;
    const T c = g.cL + fac_label_log2(reg.lp2[skew(d, b, t, u)]) + reg.log2_lam;   // log2(lambda e_y e^-lse)
    const T mx = R::max(g.cA, c);
    if (mx > R::neg_inf()) g.cA = mx + log2_of(R::exp2(g.cA - mx) + R::exp2(c - mx));
    g.cL += reg.log2_1p_lam;
}
// delay penalty of the label offset (DESIGN.md §10), after fastemit_fold: FastEmit's log2 p_y comes from the
// stored, penalised factor, and adding it to the unpenalised cL gives exactly log2(e_y e^-lse) of the penalised
// lattice.  delay_log2 = lambda log2(e).  A row without a label keeps cL = -inf.
template <typename T>
__device__ __forceinline__ void delay_fold(RowGrad<T>& g, const T delay_log2, int Tb, uint32_t t) {
    g.cL += delay_log2 * delay_bracket<T>(Tb, t);
}
// clip to [-c, c]; a NaN gradient stays NaN (the c = +inf of "off" then leaves every value unchanged)
__device__ __forceinline__ float clip_grad(float g, float c) {
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(g), "f"(-c));
    asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(r), "f"(c));
    return r;
}
__device__ __forceinline__ double clip_grad(double g, double c) { return g > c ? c : (g < -c ? -c : g); }

// one vector of gradient from one vector of logits; k0 = index of its first element
// ZEROM: the caller has folded the row maximum into the offsets (rg.m is not read; 16-bit storage path)
// REG: clip to [-clamp, clamp] after the blank / label patch, before the scale
template <typename T, int VEC, bool SCALED, bool ZEROM = false, bool REG = false>
__device__ __forceinline__ VecT<T, VEC> grad_vec(const VecT<T, VEC>& x, const RowGrad<T>& rg, int k0,
                                                 int kb, T scale, T clamp = T(0)) {
    using R = Real<T>;
    VecT<T, VEC> g;
    T dl[VEC];
#pragma unroll
    for (int c = 0; c < VEC; ++c) {
        dl[c] = ZEROM ? x.v[c] : x.v[c] - rg.m;
        g.v[c] = R::exp2(fma(dl[c], (T)R::kLog2e, rg.cA));
    }
    // blank / label lanes: at most two vectors of the row take this branch
    if ((unsigned)(kb - k0) < (unsigned)VEC || (unsigned)(rg.y - k0) < (unsigned)VEC) {
#pragma unroll
        for (int c = 0; c < VEC; ++c) {
            if (k0 + c == kb) g.v[c] -= R::exp2(fma(dl[c], (T)R::kLog2e, rg.cB));
            if (k0 + c == rg.y) g.v[c] -= R::exp2(fma(dl[c], (T)R::kLog2e, rg.cL));
        }
    }
    if (REG) {
#pragma unroll
        for (int c = 0; c < VEC; ++c) g.v[c] = clip_grad(g.v[c], clamp);
    }
    if (SCALED) {
#pragma unroll
        for (int c = 0; c < VEC; ++c) g.v[c] *= scale;
    }
    return g;
}
// MOD (the modified topology, DESIGN.md §11): the label term reads beta(t+1,u+1), and on the last frame exists
// only at u = U-2, where beta(T,U-1) = 0; the blank term is the regular one.
// fp64: lattices are natural-log doubles
template <bool MOD = false>
__device__ __forceinline__ RowGrad<double> row_grad_setup(const Dims& d, uint32_t r, uint32_t b, uint32_t t,
                                                          uint32_t u, int Tb, int Ub,
                                                          const int* __restrict__ labels,
                                                          const double2* __restrict__ stat,
                                                          const double* __restrict__ alphas,
                                                          const double* __restrict__ betas,
                                                          const double* __restrict__ llf) {
    using R = Real<double>;
    RowGrad<double> g;
    const double2 st = __ldg(stat + r);
    const size_t q = skew(d, b, t, u);  // (t+1,u) is at q + maxU, (t,u+1) at q + maxU + 1
    const double occ = alphas[q] - __ldg(llf + b);
    g.m = st.x;
    g.cA = ((occ + betas[q]) - st.y) * R::kLog2e;
    g.cB = R::neg_inf();
    g.cL = R::neg_inf();
    if ((int)t < Tb - 1)
        g.cB = ((occ + betas[q + d.maxU]) - st.y) * R::kLog2e;
    else if ((int)u == Ub - 1)
        g.cB = (occ - st.y) * R::kLog2e;
    g.y = -1;
    if ((int)u < Ub - 1) {
        if (!MOD)
            g.cL = ((occ + betas[q + d.maxU + 1]) - st.y) * R::kLog2e;
        else if ((int)t < Tb - 1)
            g.cL = ((occ + betas[q + 2 * d.maxU + 1]) - st.y) * R::kLog2e;
        else if ((int)u == Ub - 2)
            g.cL = (occ - st.y) * R::kLog2e;
        g.y = __ldg(labels + (size_t)b * (d.maxU - 1) + u);
    }
    return g;
}
// fp32: lattices are LogVal {e, log2 v}: the offsets are formed in the exp2 domain from an exact integer
// part and a small float part - no conversions to double, no FP64 pipe
template <bool MOD = false>
__device__ __forceinline__ RowGrad<float> row_grad_setup(const Dims& d, uint32_t r, uint32_t b, uint32_t t,
                                                         uint32_t u, int Tb, int Ub,
                                                         const int* __restrict__ labels,
                                                         const float2* __restrict__ stat,
                                                         const LogVal* __restrict__ alphas,
                                                         const LogVal* __restrict__ betas,
                                                         const LogVal* __restrict__ llf) {
    using R = Real<float>;
    RowGrad<float> g;
    const float2 st = __ldg(stat + r);
    const size_t q = cell(d, b, t, u);   // (t+1,u) at q + maxU, (t,u+1) at q + 1
    const LogVal a = alphas[q], ll = llf[b], bq = betas[q];
    const int oe = a.e - ll.e;            // occupancy exponent alpha - ll (exact)
    const float ol = a.l - ll.l - st.y * R::kLog2e;
    g.m = st.x;
    g.cA = (float)(oe + bq.e) + (ol + bq.l);
    g.cB = R::neg_inf();
    g.cL = R::neg_inf();
    if ((int)t < Tb - 1) {
        const LogVal bn = betas[q + d.maxU];
        g.cB = (float)(oe + bn.e) + (ol + bn.l);
    } else if ((int)u == Ub - 1) {
        g.cB = (float)oe + ol;
    }
    g.y = -1;
    if ((int)u < Ub - 1) {
        if (!MOD) {
            const LogVal bn = betas[q + 1];
            g.cL = (float)(oe + bn.e) + (ol + bn.l);
        } else if ((int)t < Tb - 1) {
            const LogVal bn = betas[q + d.maxU + 1];
            g.cL = (float)(oe + bn.e) + (ol + bn.l);
        } else if ((int)u == Ub - 2) {
            g.cL = (float)oe + ol;
        }
        g.y = __ldg(labels + (size_t)b * (d.maxU - 1) + u);
    }
    return g;
}
// Same constants with every load issued unconditionally and at once (short rows: the row's scalars are
// the critical path of a chunk CTA, two dependent rounds of loads cost ~1 us).  Reads are in bounds for
// every (t,u) of the tensor: q + maxU (MOD: q + maxU + 1) stays inside the lattice arrays plus the slack carve() leaves.
template <bool MOD = false>
__device__ __forceinline__ RowGrad<float> row_grad_setup_spec(const Dims& d, uint32_t r, uint32_t b, uint32_t t,
                                                              uint32_t u, const int* __restrict__ xlen,
                                                              const int* __restrict__ ylen,
                                                              const int* __restrict__ labels,
                                                              const float2* __restrict__ stat,
                                                              const LogVal* __restrict__ alphas,
                                                              const LogVal* __restrict__ betas,
                                                              const LogVal* __restrict__ llf, int& Tb, int& Ub) {
    using R = Real<float>;
    const size_t q = cell(d, b, t, u);
    const int xl = __ldg(xlen + b), yl = __ldg(ylen + b);
    const float2 st = __ldg(stat + r);
    const LogVal a = alphas[q], ll = llf[b], bq = betas[q], bt = betas[q + d.maxU], bu = betas[q + (MOD ? d.maxU + 1 : 1)];
    const int lab = (int)u < d.maxU - 1 ? __ldg(labels + (size_t)b * (d.maxU - 1) + u) : 0;
    Tb = min(max(xl, 1), d.maxT);
    Ub = min(max(yl + 1, 1), d.maxU);
    RowGrad<float> g;
    const int oe = a.e - ll.e;
    const float ol = a.l - ll.l - st.y * R::kLog2e;
    g.m = st.x;
    g.cA = (float)(oe + bq.e) + (ol + bq.l);
    g.cB = R::neg_inf();
    if ((int)t < Tb - 1) g.cB = (float)(oe + bt.e) + (ol + bt.l);
    else if ((int)u == Ub - 1) g.cB = (float)oe + ol;
    g.cL = R::neg_inf();
    g.y = -1;
    if ((int)u < Ub - 1) {
        if (!MOD || (int)t < Tb - 1) g.cL = (float)(oe + bu.e) + (ol + bu.l);
        else if ((int)u == Ub - 2) g.cL = (float)oe + ol;
        g.y = lab;
    }
    return g;
}

// Pass 2, long rows: one CTA per row, non-persistent (same reasoning as rowstats_row_kernel).  All
// of a thread's loads are issued before the row's lattice constants are fetched, so both latencies
// overlap; measured shape of this loop (probe): 6.85 TB/s read+write at V = 5000.
#ifndef RNNT_GRAD_MINB
#define RNNT_GRAD_MINB 5
#endif
#ifndef RNNT_GRAD_MINB16
#define RNNT_GRAD_MINB16 8   // 16-bit rows are one trip of 128 threads: residency (bytes in flight) is what pays
#endif
template <typename T, int VEC, int NV, bool SCALED, typename IO, bool REG, bool PRUNED, bool DELAY, bool MOD = false>
__device__ __forceinline__ void grad_row(const IO* __restrict__ acts, IO* __restrict__ grads,
                                         const int* __restrict__ labels, const int* __restrict__ xlen,
                                         const int* __restrict__ ylen, const typename Real<T>::pair* __restrict__ stat,
                                         const typename Lat<T>::val* __restrict__ alphas,
                                         const typename Lat<T>::val* __restrict__ betas,
                                         const typename Lat<T>::val* __restrict__ llf, const T scale_in,
                                         const T* __restrict__ scale_vec, const Dims d, const GradReg<T> reg,
                                         const Prune p, const T delay_log2) {
    constexpr int kRowThreads = RowThreads<IO>::value;
    const uint32_t r = d.rows - 1 - blockIdx.x;
    uint32_t u, b, t;
    row_decode<PRUNED>(d, p, r, b, t, u);
    int Tb, Ub;
    utt_extent(d, xlen, ylen, b, Tb, Ub);
    const int nv = d.V / VEC;
    const int kb = d.blank;
    const IO* row = acts + (uint64_t)r * d.V;
    IO* grow = grads + (uint64_t)r * d.V;
    // per-utterance upstream gradient (autograd's grad_output) times the scalar factor
    const T scale = (SCALED && scale_vec) ? __ldg(scale_vec + b) * scale_in : scale_in;
    if (PRUNED ? pruned_grad_padding(t, u, Tb, Ub, llf, b)
               : MOD ? mod_grad_padding(t, u, Tb, Ub, llf, b) : (int)t >= Tb || (int)u >= Ub) {
        VecT<T, VEC> z;
#pragma unroll
        for (int c = 0; c < VEC; ++c) z.v[c] = 0;
        for (int i = threadIdx.x; i < nv; i += kRowThreads) st_stream<T, VEC>(grow + (size_t)i * VEC, z);
        return;
    }
    // the logits stay PACKED in registers until they are used (16-bit storage: 20 registers instead of 40)
    using P = typename Pack<sizeof(IO) * VEC>::type;
    P x[NV];
    auto load = [&](int base) {
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const int i = base + j * kRowThreads;
            if (i < nv) x[j] = __ldcs(reinterpret_cast<const P*>(row + (size_t)i * VEC));
        }
    };
    load(threadIdx.x);  // in flight before the lattice constants are fetched
    pdl_wait();         // (PDL) the logits were read ahead of the lattice kernel's completion; its output is not
    RowGrad<T> rg = row_grad_setup<MOD>(d, r, b, t, u, Tb, Ub, labels, stat, alphas, betas, llf);
    if constexpr (REG) fastemit_fold(rg, reg, b, t, u, d);
    if constexpr (DELAY) delay_fold(rg, delay_log2, Tb, t);
    // 16-bit storage: fold the row maximum into the three offsets, one FFMA per element instead of FADD + FFMA
    // (its rounding, |m| * 6e-8 in the exponent, is far below the 16-bit quantisation of input and output)
    constexpr bool ZEROM = sizeof(IO) == 2;
    if (ZEROM) {
        const T shift = -rg.m * (T)Real<T>::kLog2e;
        rg.cA += shift, rg.cB += shift, rg.cL += shift;
    }
    auto emit = [&](int base) {
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const int i = base + j * kRowThreads;
            if (i < nv)
                st_stream<T, VEC>(grow + (size_t)i * VEC,
                                  grad_vec<T, VEC, SCALED, ZEROM, REG>(unpack<T, VEC, IO, P>(x[j]), rg, i * VEC, kb,
                                                                       scale, reg.clamp));
        }
    };
    emit(threadIdx.x);
    for (int base = threadIdx.x + kRowThreads * NV; base < nv; base += kRowThreads * NV) {  // V > 256*NV*VEC only
        load(base);
        emit(base);
    }
}
template <typename T, int VEC, int NV, bool SCALED, typename IO, bool REG, bool PRUNED>
__global__ void __launch_bounds__(RowThreads<IO>::value, (sizeof(IO) >= 4 ? RNNT_GRAD_MINB : RNNT_GRAD_MINB16))
grad_row_kernel(const IO* __restrict__ acts, IO* __restrict__ grads, const int* __restrict__ labels,
                const int* __restrict__ xlen, const int* __restrict__ ylen,
                const typename Real<T>::pair* __restrict__ stat, const typename Lat<T>::val* __restrict__ alphas,
                const typename Lat<T>::val* __restrict__ betas, const typename Lat<T>::val* __restrict__ llf,
                const T scale_in, const T* __restrict__ scale_vec, const Dims d, const GradReg<T> reg,
                const Prune p) {
    grad_row<T, VEC, NV, SCALED, IO, REG, PRUNED, false>(acts, grads, labels, xlen, ylen, stat, alphas, betas, llf,
                                                         scale_in, scale_vec, d, reg, p, T(0));
}
template <typename T, int VEC, int NV, bool SCALED, typename IO, bool REG, bool PRUNED>
__global__ void __launch_bounds__(RowThreads<IO>::value, (sizeof(IO) >= 4 ? RNNT_GRAD_MINB : RNNT_GRAD_MINB16))
grad_row_delay_kernel(const IO* __restrict__ acts, IO* __restrict__ grads, const int* __restrict__ labels,
                      const int* __restrict__ xlen, const int* __restrict__ ylen,
                      const typename Real<T>::pair* __restrict__ stat, const typename Lat<T>::val* __restrict__ alphas,
                      const typename Lat<T>::val* __restrict__ betas, const typename Lat<T>::val* __restrict__ llf,
                      const T scale_in, const T* __restrict__ scale_vec, const Dims d, const GradReg<T> reg,
                      const Prune p, const T delay_log2) {
    grad_row<T, VEC, NV, SCALED, IO, REG, PRUNED, true>(acts, grads, labels, xlen, ylen, stat, alphas, betas, llf,
                                                        scale_in, scale_vec, d, reg, p, delay_log2);
}
// The modified topology (DESIGN.md §11).  Its twins take the upstream scale, the gradient options and the delay
// penalty as run-time values (scale 1, FastEmit off, clamp +inf and penalty 0 leave every value bitwise unchanged):
// one instantiation per shape and PRUNED instead of sixteen keeps the library's compile time near the parent's.
template <typename T, int VEC, int NV, typename IO, bool PRUNED>
__global__ void __launch_bounds__(RowThreads<IO>::value, (sizeof(IO) >= 4 ? RNNT_GRAD_MINB : RNNT_GRAD_MINB16))
grad_row_mod_kernel(const IO* __restrict__ acts, IO* __restrict__ grads, const int* __restrict__ labels,
                    const int* __restrict__ xlen, const int* __restrict__ ylen,
                    const typename Real<T>::pair* __restrict__ stat, const typename Lat<T>::val* __restrict__ alphas,
                    const typename Lat<T>::val* __restrict__ betas, const typename Lat<T>::val* __restrict__ llf,
                    const T scale_in, const T* __restrict__ scale_vec, const Dims d, const GradReg<T> reg,
                    const Prune p, const T delay_log2) {
    grad_row<T, VEC, NV, true, IO, true, PRUNED, true, true>(acts, grads, labels, xlen, ylen, stat, alphas, betas, llf,
                                                             scale_in, scale_vec, d, reg, p, delay_log2);
}

// Pass 2, short rows: same register tile as rowstats_tile_kernel.
template <typename T, int VEC, int LPR, bool SCALED, typename IO, bool REG, bool PRUNED, bool DELAY, bool MOD = false>
__device__ __forceinline__ void grad_tile(const IO* __restrict__ acts, IO* __restrict__ grads,
                                          const int* __restrict__ labels, const int* __restrict__ xlen,
                                          const int* __restrict__ ylen, const typename Real<T>::pair* __restrict__ stat,
                                          const typename Lat<T>::val* __restrict__ alphas,
                                          const typename Lat<T>::val* __restrict__ betas,
                                          const typename Lat<T>::val* __restrict__ llf, const T scale_in,
                                          const T* __restrict__ scale_vec, const Dims d, const GradReg<T> reg,
                                          const Prune p, const T delay_log2) {
    constexpr int RPW = kWarp / LPR;
    const int lane = threadIdx.x & 31;
    const int sub = lane / LPR, sl = lane % LPR;
    const uint64_t gw = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int nv = d.V / VEC;
    const int kb = d.blank;

    do {   // non-persistent: one tile of RPW rows per warp
        const uint64_t rr = gw * RPW + sub;
        if (rr >= d.rows) continue;
        const uint32_t r = d.rows - 1 - (uint32_t)rr;
        uint32_t u, b, t;
        row_decode<PRUNED>(d, p, r, b, t, u);
        int Tb, Ub;
        utt_extent(d, xlen, ylen, b, Tb, Ub);
        const IO* row = acts + (uint64_t)r * d.V;
        IO* grow = grads + (uint64_t)r * d.V;
        const T scale = (SCALED && scale_vec) ? __ldg(scale_vec + b) * scale_in : scale_in;
        if (PRUNED ? pruned_grad_padding(t, u, Tb, Ub, llf, b)
               : MOD ? mod_grad_padding(t, u, Tb, Ub, llf, b) : (int)t >= Tb || (int)u >= Ub) {
            VecT<T, VEC> z;
#pragma unroll
            for (int c = 0; c < VEC; ++c) z.v[c] = 0;
#pragma unroll
            for (int j = 0; j < kVPL; ++j) {
                const int i = sl + j * LPR;
                if (i < nv) st_stream<T, VEC>(grow + (size_t)i * VEC, z);
            }
            continue;
        }
        VecT<T, VEC> x[kVPL];
#pragma unroll
        for (int j = 0; j < kVPL; ++j) {
            const int i = sl + j * LPR;
            if (i < nv) x[j] = ld_stream<T, VEC>(row + (size_t)i * VEC);
        }
        pdl_wait();
        RowGrad<T> rg = row_grad_setup<MOD>(d, r, b, t, u, Tb, Ub, labels, stat, alphas, betas, llf);
        if constexpr (REG) fastemit_fold(rg, reg, b, t, u, d);
        if constexpr (DELAY) delay_fold(rg, delay_log2, Tb, t);
#pragma unroll
        for (int j = 0; j < kVPL; ++j) {
            const int i = sl + j * LPR;
            if (i < nv)
                st_stream<T, VEC>(grow + (size_t)i * VEC,
                                  grad_vec<T, VEC, SCALED, false, REG>(x[j], rg, i * VEC, kb, scale, reg.clamp));
        }
    } while (false);
}
template <typename T, int VEC, int LPR, bool SCALED, typename IO, bool REG, bool PRUNED>
__global__ void __launch_bounds__(256)
grad_tile_kernel(const IO* __restrict__ acts, IO* __restrict__ grads, const int* __restrict__ labels,
                 const int* __restrict__ xlen, const int* __restrict__ ylen,
                 const typename Real<T>::pair* __restrict__ stat, const typename Lat<T>::val* __restrict__ alphas,
                 const typename Lat<T>::val* __restrict__ betas, const typename Lat<T>::val* __restrict__ llf,
                 const T scale_in, const T* __restrict__ scale_vec, const Dims d, const GradReg<T> reg,
                 const Prune p) {
    grad_tile<T, VEC, LPR, SCALED, IO, REG, PRUNED, false>(acts, grads, labels, xlen, ylen, stat, alphas, betas, llf,
                                                           scale_in, scale_vec, d, reg, p, T(0));
}
template <typename T, int VEC, int LPR, bool SCALED, typename IO, bool REG, bool PRUNED>
__global__ void __launch_bounds__(256)
grad_tile_delay_kernel(const IO* __restrict__ acts, IO* __restrict__ grads, const int* __restrict__ labels,
                       const int* __restrict__ xlen, const int* __restrict__ ylen,
                       const typename Real<T>::pair* __restrict__ stat, const typename Lat<T>::val* __restrict__ alphas,
                       const typename Lat<T>::val* __restrict__ betas, const typename Lat<T>::val* __restrict__ llf,
                       const T scale_in, const T* __restrict__ scale_vec, const Dims d, const GradReg<T> reg,
                       const Prune p, const T delay_log2) {
    grad_tile<T, VEC, LPR, SCALED, IO, REG, PRUNED, true>(acts, grads, labels, xlen, ylen, stat, alphas, betas, llf,
                                                          scale_in, scale_vec, d, reg, p, delay_log2);
}
template <typename T, int VEC, int LPR, typename IO, bool PRUNED>
__global__ void __launch_bounds__(256)
grad_tile_mod_kernel(const IO* __restrict__ acts, IO* __restrict__ grads, const int* __restrict__ labels,
                     const int* __restrict__ xlen, const int* __restrict__ ylen,
                     const typename Real<T>::pair* __restrict__ stat, const typename Lat<T>::val* __restrict__ alphas,
                     const typename Lat<T>::val* __restrict__ betas, const typename Lat<T>::val* __restrict__ llf,
                     const T scale_in, const T* __restrict__ scale_vec, const Dims d, const GradReg<T> reg,
                     const Prune p, const T delay_log2) {
    grad_tile<T, VEC, LPR, true, IO, true, PRUNED, true, true>(acts, grads, labels, xlen, ylen, stat, alphas, betas,
                                                               llf, scale_in, scale_vec, d, reg, p, delay_log2);
}

}  // namespace b200rnnt
