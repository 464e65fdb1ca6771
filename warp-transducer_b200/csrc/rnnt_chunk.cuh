// rnnt_chunk.cuh — the two streaming passes for SHORT vocabulary rows (row <= 512 bytes: the README
// small-vocabulary shape V=28 and the long-utterance shape V=50).
//
// A row of 28 or 50 floats is far too short to be a unit of work: per-row index decoding, length
// checks, predicates on every vector slot and 8-byte loads (a 200-byte row is not 16-byte aligned)
// made the register-tile kernels issue-bound at ~19 instructions per element (ncu, round 1:
// smsp__issue_active 78 %, DRAM 75 %).  Here the unit is a CHUNK of R consecutive rows, which is
// one contiguous, 16-byte aligned run of R*V elements in the activation tensor:
//
//   * ONE thread moves the whole chunk global -> shared memory with a 1-D TMA bulk copy
//     (cp.async.bulk ... mbarrier::complete_tx, SASS UBLKCP): no per-element load instructions, no
//     alignment cases, the address generation is off the SM's issue slots.
//   * While the copy is in flight every thread decodes its row and fetches the per-row scalars.
//   * TPR threads share a row and walk it from shared memory element by element (pairs for even V); TPR
//     is the power of two dividing V (V=50 -> 2, V=28 -> 4).  Which lanes of a warp share a row is chosen
//     on the host per shape (ChunkMap below) so that a warp-wide access hits distinct banks: with adjacent
//     lanes sharing a row, V=50 puts lane (row 7, slice 1) on the banks of (row 0, slice 0) - every
//     access of the sweep took two wavefronts instead of one (ncu source page, round 2).
//   * Pass 2 overwrites the chunk in place with the gradient and ONE thread writes it back with a
//     bulk shared -> global copy.
//
// Replaces (for short rows) reference reduce.h:10-146 + gpu_rnnt_kernel.h:5-9 (pass 1) and
// gpu_rnnt.h:107-110 + gpu_rnnt_kernel.h:143-179 (pass 2).  Same outputs as the tile kernels in
// rnnt_kernels.cuh: stat[row] = (max, log sum exp), lp2[skew] = (lp_blank, lp_label), dense gradient
// with zeros on padded cells.  Short-lived CTAs on purpose (see rnnt_kernels.cuh).
#pragma once
#include "rnnt_kernels.cuh"

namespace b200rnnt {

// ---- mbarrier / bulk-copy PTX -------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Waiting threads SLEEP between probes (ns > 0: try_wait with a suspend-time hint, which compiles to
// SYNCS.TRYWAIT + NANOSLEEP ns) instead of spinning, so a CTA that waits for its chunk costs the SM no issue
// slots (pass 1 is issue-bound).  The sleep is a quantum, not an upper bound - a wait is rounded up to whole
// quanta - so it is a tuned value (RNNT_B200_CHUNK_WAIT_NS); ns = 0 spins on test_wait.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, uint32_t ns) {
    uint32_t done = 0;
    if (ns == 0) {
        while (!done)
            asm volatile("{ .reg .pred p; mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                         : "=r"(done)
                         : "r"(bar), "r"(parity)
                         : "memory");
        return;
    }
    while (!done) {
        asm volatile(
            "{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3; selp.u32 %0, 1, 0, p; }"
            : "=r"(done)
            : "r"(bar), "r"(parity), "r"(ns)
            : "memory");
    }
}
// global -> shared, completion counted in bytes on the mbarrier.  dst/src 16-B aligned, bytes % 16 == 0.
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
// shared -> global; the issuing thread waits until the source has been read before the CTA may exit
__device__ __forceinline__ void bulk_s2g_and_wait(void* dst, uint32_t src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

template <typename T> struct ChunkThreads { static constexpr int value = sizeof(T) >= 8 ? 128 : 256; };

// lane -> (row of the chunk, slice of the row).  slice-major (hmajor): lanes l, l + 32/TPR, ... share a
// row, so consecutive lanes walk consecutive rows; row-major: adjacent lanes share a row.
template <int TPR> struct ChunkMap {
    int row, slice, stride;   // stride: lane distance between the lanes of one row
    __device__ __forceinline__ ChunkMap(int hmajor) {
        constexpr int RPW = 32 / TPR;
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        const int il = hmajor ? lane % RPW : lane / TPR;
        slice = hmajor ? lane / RPW : lane % TPR;
        row = warp * RPW + il;
        stride = hmajor ? RPW : 1;
    }
};

// Stage rows [r0, r0+nrows) of the activation tensor into `tile`; returns after the data is visible
// to every thread of the CTA.  Thread 0 has already decided that the chunk is worth reading.
template <typename T>
__device__ __forceinline__ void chunk_issue(const T* __restrict__ acts, T* tile, uint32_t bar, uint32_t r0,
                                            uint32_t nrows, int V) {
    // called by thread 0 only, before the CTA-wide barrier that publishes the mbarrier
    const uint32_t bytes = nrows * (uint32_t)V * (uint32_t)sizeof(T);
    mbar_init(bar, 1);
    mbar_expect_tx(bar, bytes);
    bulk_g2s(smem_u32(tile), acts + (uint64_t)r0 * V, bytes, bar);
}

// =================================================================================================
// Pass 1 on a chunk: per row (max, log sum exp) and the lattice's transition factors.
//
// Per-row SCALAR work (index decoding, lengths, label, the statistics' logarithm, the factor split, the
// skewed store address) is done ROW-PARALLEL: thread r of the CTA owns row r's scalars, so that work runs
// on ROWS/32 fully populated warps instead of being repeated by (or idling) the TPR lanes that share a row.
// At small V it is most of the kernel (the loop is issue-bound).
// The element walk is group-parallel: TPR lanes per row, results handed over through shared memory.
// The CTA size NT is a template parameter (tuning hook RNNT_B200_CHUNK_NT; default 256).
// =================================================================================================
template <typename T, int TPR, int NT, bool PRUNED, bool DELAY>
__device__ __forceinline__ void rowstats_chunk(const T* __restrict__ acts, const int* __restrict__ labels,
                                               const int* __restrict__ xlen, const int* __restrict__ ylen,
                                               typename Real<T>::pair* __restrict__ stat,
                                               typename Lat<T>::fac* __restrict__ lp2, const Dims& d,
                                               const int hmajor, const uint32_t wait_ns, const Prune& p,
                                               const T delay, unsigned char* chunk_raw,
                                               unsigned long long* bar_store, typename Real<T>::pair* row_ms) {
    using R = Real<T>;
    using Pair = typename R::pair;
    constexpr int ROWS = NT / TPR;
    static_assert(TPR <= 32 && NT % 32 == 0, "the lanes of a row sit in one warp");
    T* tile = reinterpret_cast<T*>(chunk_raw);
    const uint32_t bar = smem_u32(bar_store);
    const uint32_t r0 = blockIdx.x * ROWS;
    const uint32_t nrows = min((uint32_t)ROWS, d.rows - r0);
    const int V = d.V;
    const bool bulk = ((nrows * (uint32_t)V * (uint32_t)sizeof(T)) & 15u) == 0;   // false only on a ragged last chunk
    // the copy goes out first: thread 0 needs nothing but the chunk index for it
    if (threadIdx.x == 0 && bulk) chunk_issue<T>(acts, tile, bar, r0, nrows, V);
    pdl_trigger();

    // row-parallel bookkeeping while the copy is in flight: thread r <-> row r0 + r
    bool valid = threadIdx.x < nrows;
    int y = -1;
    size_t q = 0;
    T pen = T(0);   // DELAY: the row's label penalty
    if (valid) {
        uint32_t u, b, t;
        int Tb, Ub;
        row_decode<PRUNED>(d, p, r0 + threadIdx.x, b, t, u);
        utt_extent(d, xlen, ylen, b, Tb, Ub);
        valid = !row_padding<PRUNED>(t, u, Tb, Ub);
        if (valid && (int)u < Ub - 1) y = __ldg(labels + (size_t)b * (d.maxU - 1) + u);
        q = skew(d, b, t, u);
        if constexpr (DELAY) pen = delay * delay_bracket<T>(Tb, t);
    }
    // one barrier: publishes the mbarrier to the waiters and tells whether any row of the chunk is a
    // real cell (a fully padded chunk - ragged batches only - costs one wasted read, nothing else)
    const bool any_valid = __syncthreads_or(valid);
    if (!any_valid) {
        if (bulk && threadIdx.x == 0) mbar_wait(bar, 0, wait_ns);   // shared memory must outlive the in-flight copy
        return;
    }
    if (bulk) {
        mbar_wait(bar, 0, wait_ns);
    } else {
        const T* src = acts + (uint64_t)r0 * V;
        for (uint32_t k = threadIdx.x; k < nrows * (uint32_t)V; k += NT) tile[k] = ld_scalar<T>(src + k);
        __syncthreads();
    }

    // group-parallel walk.  Even V: a row is walked as PAIRS (one 8/16-byte shared-memory access per two
    // elements); the row start is pair-aligned because V is even.  Rows past the chunk walk row 0.
    {
        const ChunkMap<TPR> map(hmajor);
        const int i = map.row, h = map.slice;
        const T* x = tile + (size_t)((uint32_t)i < nrows ? i : 0) * V;
        const Pair* x2 = reinterpret_cast<const Pair*>(x);
        const bool paired = (V & 1) == 0;
        T m = R::neg_inf();
        if (paired) {
#pragma unroll 4
            for (int j = h; j < (V >> 1); j += TPR) {
                const Pair v = x2[j];
                m = R::max(m, R::max(v.x, v.y));
            }
        } else {
#pragma unroll 4
            for (int k = h; k < V; k += TPR) m = R::max(m, x[k]);
        }
        const T M = group_max_strided<TPR>(m, map.stride);
        const ExpSum<T> es((M == R::neg_inf()) ? T(0) : M);
        T sum = 0;
        if (paired) {
#pragma unroll 4
            for (int j = h; j < (V >> 1); j += TPR) {
                const Pair v = x2[j];
                sum += es.term(v.x) + es.term(v.y);
            }
        } else {
#pragma unroll 4
            for (int k = h; k < V; k += TPR) sum += es.term(x[k]);
        }
        const T S = group_sum_strided<TPR>(sum, map.stride);
        if (h == 0) {
            Pair ms;
            ms.x = M;
            ms.y = S;
            row_ms[i] = ms;
        }
    }
    __syncthreads();
    // row-parallel epilogue: thread r finishes row r
    if (valid) {
        const Pair ms = row_ms[threadIdx.x];
        const T M = ms.x;
        const ExpSum<T> es((M == R::neg_inf()) ? T(0) : M);
        const T lse = es.log_of(ms.y);
        const T* x = tile + (size_t)threadIdx.x * V;
        Pair st;
        st.x = M;
        st.y = lse;
        stat[r0 + threadIdx.x] = st;
        if constexpr (DELAY)
            lp2[q] = Lat<T>::make((x[d.blank] - M) - lse, y >= 0 ? (x[y] - M) - lse + pen : T(0), y >= 0);
        else
            lp2[q] = Lat<T>::make((x[d.blank] - M) - lse, y >= 0 ? (x[y] - M) - lse : T(0), y >= 0);
    }
}
template <typename T, int TPR, int NT, bool PRUNED>
__global__ void __launch_bounds__(NT)
rowstats_chunk_kernel(const T* __restrict__ acts, const int* __restrict__ labels, const int* __restrict__ xlen,
                      const int* __restrict__ ylen, typename Real<T>::pair* __restrict__ stat,
                      typename Lat<T>::fac* __restrict__ lp2, const Dims d, const int hmajor, const uint32_t wait_ns,
                      const Prune p) {
    // shared memory: declared here, not in the body (in a device function the dynamic part would take the
    // 1024-byte alignment of the tensor-core kernels' and start elsewhere)
    extern __shared__ __align__(128) unsigned char chunk_raw[];
    __shared__ __align__(8) unsigned long long bar_store;
    __shared__ typename Real<T>::pair row_ms[NT / TPR];   // (max, sum of exponentials) per row, group leaders -> row owners
    rowstats_chunk<T, TPR, NT, PRUNED, false>(acts, labels, xlen, ylen, stat, lp2, d, hmajor, wait_ns, p, T(0), chunk_raw,
                                              &bar_store, row_ms);
}
template <typename T, int TPR, int NT, bool PRUNED>
__global__ void __launch_bounds__(NT)
rowstats_chunk_delay_kernel(const T* __restrict__ acts, const int* __restrict__ labels, const int* __restrict__ xlen,
                            const int* __restrict__ ylen, typename Real<T>::pair* __restrict__ stat,
                            typename Lat<T>::fac* __restrict__ lp2, const Dims d, const int hmajor,
                            const uint32_t wait_ns, const Prune p, const T delay) {
    // shared memory: declared here, not in the body (in a device function the dynamic part would take the
    // 1024-byte alignment of the tensor-core kernels' and start elsewhere)
    extern __shared__ __align__(128) unsigned char chunk_raw[];
    __shared__ __align__(8) unsigned long long bar_store;
    __shared__ typename Real<T>::pair row_ms[NT / TPR];   // (max, sum of exponentials) per row, group leaders -> row owners
    rowstats_chunk<T, TPR, NT, PRUNED, true>(acts, labels, xlen, ylen, stat, lp2, d, hmajor, wait_ns, p, delay, chunk_raw,
                                             &bar_store, row_ms);
}

// =================================================================================================
// Pass 2 on a chunk: gradient in place in shared memory, one bulk store.  Formula and per-row
// constants as grad_row_kernel (rnnt_kernels.cuh); the blank / label corrections are applied to the
// two affected words of the row after the sweep.  Each lane fetches its row's constants while the chunk is in
// flight (fp32: one round of loads).
// =================================================================================================
// a row's gradient constants (RowGrad), its upstream scale, and 1 / 0 / -1: valid / padding / past the tensor
template <typename T> struct ChunkRow {
    T m, cA, cB, cL;
    T scale;
    int y;
    int valid;
};

template <typename T, int TPR, int NT, bool SCALED, bool REG, bool PRUNED, bool DELAY, bool MOD = false>
__device__ __forceinline__ void grad_chunk(const T* __restrict__ acts, T* __restrict__ grads,
                                           const int* __restrict__ labels, const int* __restrict__ xlen,
                                           const int* __restrict__ ylen,
                                           const typename Real<T>::pair* __restrict__ stat,
                                           const typename Lat<T>::val* __restrict__ alphas,
                                           const typename Lat<T>::val* __restrict__ betas,
                                           const typename Lat<T>::val* __restrict__ llf, const T scale_in,
                                           const T* __restrict__ scale_vec, const Dims d, const int hmajor,
                                           const uint32_t wait_ns, const GradReg<T> reg, const Prune p,
                                           const T delay_log2, unsigned char* chunk_raw,
                                           unsigned long long* bar_store) {
    using R = Real<T>;
    using Pair = typename R::pair;
    constexpr int ROWS = NT / TPR;
    T* tile = reinterpret_cast<T*>(chunk_raw);
    const ChunkMap<TPR> map(hmajor);
    const uint32_t bar = smem_u32(bar_store);
    // chunks in reverse order: the tail of pass 1 is met first in L2
    const uint32_t nchunks = gridDim.x;
    const uint32_t r0 = (nchunks - 1 - blockIdx.x) * ROWS;
    const uint32_t nrows = min((uint32_t)ROWS, d.rows - r0);
    const int V = d.V;
    const uint32_t nelem = nrows * (uint32_t)V;
    const bool bulk = ((nelem * (uint32_t)sizeof(T)) & 15u) == 0;
    if (threadIdx.x == 0 && bulk) chunk_issue<T>(acts, tile, bar, r0, nrows, V);   // the copy goes out first
    T* gout = grads + (uint64_t)r0 * V;
    pdl_wait();   // (PDL) the chunk was requested ahead of the lattice kernel's completion; its output is read below

    // Row constants: every lane fetches its row's constants itself (lanes of a row hit the same addresses, so
    // the loads coalesce into one request per row).  Fetching them row-parallel and handing them over through
    // shared memory, as pass 1 does, costs more than the saved instructions at small V: the extra hop sits
    // behind the barrier, and the hand-over array costs resident CTAs per SM.
    auto fetch = [&](uint32_t row_in_chunk) {
        const bool inrange = row_in_chunk < nrows;
        const uint32_t r = r0 + (inrange ? row_in_chunk : 0);
        ChunkRow<T> c;
        c.scale = scale_in;
        uint32_t u, b, t;
        int Tb, Ub;
        row_decode<PRUNED>(d, p, r, b, t, u);
        RowGrad<T> rg;
        bool v;
        if constexpr (sizeof(T) == 4) {
            // every scalar of the row is requested in ONE round of loads, validity is sorted out afterwards
            // (addresses are in bounds for any t, u of the tensor: see the workspace slack in carve(); a pruned
            // row's u is clamped into the tensor for the addresses - the row is padding whenever that changes it)
            const uint32_t ua = PRUNED ? min(u, (uint32_t)d.maxU - 1) : u;
            rg = row_grad_setup_spec<MOD>(d, r, b, t, ua, xlen, ylen, labels, stat, alphas, betas, llf, Tb, Ub);
            if (SCALED && scale_vec) c.scale = __ldg(scale_vec + b) * scale_in;
            if constexpr (PRUNED) v = inrange && !pruned_grad_padding(t, u, Tb, Ub, llf, b);
            else if constexpr (MOD) v = inrange && !mod_grad_padding(t, u, Tb, Ub, llf, b);
            else v = inrange && (int)t < Tb && (int)u < Ub;
        } else {
            utt_extent(d, xlen, ylen, b, Tb, Ub);
            if constexpr (PRUNED) v = inrange && !pruned_grad_padding(t, u, Tb, Ub, llf, b);
            else if constexpr (MOD) v = inrange && !mod_grad_padding(t, u, Tb, Ub, llf, b);
            else v = inrange && (int)t < Tb && (int)u < Ub;
            rg.m = 0, rg.cA = 0, rg.cB = R::neg_inf(), rg.cL = R::neg_inf(), rg.y = -1;
            if (v) {
                rg = row_grad_setup<MOD>(d, r, b, t, u, Tb, Ub, labels, stat, alphas, betas, llf);
                if (SCALED && scale_vec) c.scale = __ldg(scale_vec + b) * scale_in;
            }
        }
        if constexpr (REG) {
            if (v) fastemit_fold(rg, reg, b, t, u, d);
        }
        if constexpr (DELAY) delay_fold(rg, delay_log2, Tb, t);
        c.m = rg.m, c.cA = rg.cA, c.cB = rg.cB, c.cL = rg.cL, c.y = rg.y;
        c.valid = v ? 1 : (inrange ? 0 : -1);   // -1: row does not exist (past the end of the tensor)
        return c;
    };
    const ChunkRow<T> g = fetch(map.row);
    // one barrier: publishes the mbarrier, and tells whether any row is a real cell
    const bool any_valid = __syncthreads_or(g.valid > 0);
    if (!any_valid) {   // the whole chunk is padding: zeros straight to global memory
        if (bulk) {
            constexpr int VEC = 16 / sizeof(T);
            VecT<T, VEC> z;
#pragma unroll
            for (int c = 0; c < VEC; ++c) z.v[c] = 0;
            for (uint32_t k = threadIdx.x; k < nelem / VEC; k += NT) st_stream<T, VEC>(gout + (size_t)k * VEC, z);
            if (threadIdx.x == 0) mbar_wait(bar, 0, wait_ns);   // shared memory must outlive the in-flight copy
        } else {
            for (uint32_t k = threadIdx.x; k < nelem; k += NT) gout[k] = T(0);
        }
        return;
    }
    if (bulk) {
        mbar_wait(bar, 0, wait_ns);
    } else {
        const T* src = acts + (uint64_t)r0 * V;
        for (uint32_t k = threadIdx.x; k < nelem; k += NT) tile[k] = ld_scalar<T>(src + k);
        __syncthreads();
    }

    // Lanes sharing a row sit in one warp (TPR divides 32), so warp-level barriers order the reads of
    // the two special logits, the in-place sweep and the corrections.
    const int i = map.row, h = map.slice;
    const bool rvalid = g.valid > 0, inrange = g.valid >= 0;
    T* x = tile + (size_t)(inrange ? i : 0) * V;
    T xb = 0, xy = 0;
    if (rvalid) {
        xb = x[d.blank];
        xy = x[g.y >= 0 ? g.y : 0];
    }
    __syncwarp();
    Pair* x2 = reinterpret_cast<Pair*>(x);
    if (rvalid) {
        if ((V & 1) == 0) {   // pairs: one shared-memory load and one store per two elements
#pragma unroll 4
            for (int j = h; j < (V >> 1); j += TPR) {
                Pair v = x2[j];
                v.x = R::exp2(fma(v.x - g.m, (T)R::kLog2e, g.cA));
                v.y = R::exp2(fma(v.y - g.m, (T)R::kLog2e, g.cA));
                if (REG) v.x = clip_grad(v.x, reg.clamp), v.y = clip_grad(v.y, reg.clamp);
                if (SCALED) v.x *= g.scale, v.y *= g.scale;
                x2[j] = v;
            }
        } else {
#pragma unroll 4
            for (int k = h; k < V; k += TPR) {
                T e = R::exp2(fma(x[k] - g.m, (T)R::kLog2e, g.cA));
                if (REG) e = clip_grad(e, reg.clamp);
                if (SCALED) e *= g.scale;
                x[k] = e;
            }
        }
    } else if (inrange) {
        for (int k = h; k < V; k += TPR) x[k] = T(0);
    }
    __syncwarp();
    if (rvalid && h == 0) {
        if constexpr (REG) {
            // the sweep stored clip(dense) at the blank and label words; the clip belongs to the corrected
            // value, so both words are rewritten from the dense term minus their corrections
            T gb = R::exp2(fma(xb - g.m, (T)R::kLog2e, g.cA)) - R::exp2(fma(xb - g.m, (T)R::kLog2e, g.cB));
            if (g.y == d.blank) gb -= R::exp2(fma(xy - g.m, (T)R::kLog2e, g.cL));
            gb = clip_grad(gb, reg.clamp);
            if (SCALED) gb *= g.scale;
            x[d.blank] = gb;
            if (g.y >= 0 && g.y != d.blank) {
                T gl = R::exp2(fma(xy - g.m, (T)R::kLog2e, g.cA)) - R::exp2(fma(xy - g.m, (T)R::kLog2e, g.cL));
                gl = clip_grad(gl, reg.clamp);
                if (SCALED) gl *= g.scale;
                x[g.y] = gl;
            }
        } else {
            T gb = R::exp2(fma(xb - g.m, (T)R::kLog2e, g.cB));
            if (SCALED) gb *= g.scale;
            x[d.blank] -= gb;
            if (g.y >= 0) {
                T gl = R::exp2(fma(xy - g.m, (T)R::kLog2e, g.cL));
                if (SCALED) gl *= g.scale;
                x[g.y] -= gl;
            }
        }
    }
    if (bulk) {
        fence_async_smem();   // generic-proxy writes -> visible to the bulk copy engine
        __syncthreads();
        if (threadIdx.x == 0) bulk_s2g_and_wait(gout, smem_u32(tile), nelem * (uint32_t)sizeof(T));
    } else {
        __syncthreads();
        for (uint32_t k = threadIdx.x; k < nelem; k += NT) gout[k] = tile[k];
    }
}
template <typename T, int TPR, int NT, bool SCALED, bool REG, bool PRUNED>
__global__ void __launch_bounds__(NT)
grad_chunk_kernel(const T* __restrict__ acts, T* __restrict__ grads, const int* __restrict__ labels,
                  const int* __restrict__ xlen, const int* __restrict__ ylen,
                  const typename Real<T>::pair* __restrict__ stat, const typename Lat<T>::val* __restrict__ alphas,
                  const typename Lat<T>::val* __restrict__ betas, const typename Lat<T>::val* __restrict__ llf,
                  const T scale_in, const T* __restrict__ scale_vec, const Dims d, const int hmajor,
                  const uint32_t wait_ns, const GradReg<T> reg, const Prune p) {
    extern __shared__ __align__(128) unsigned char chunk_raw[];   // declared here: see rowstats_chunk_kernel
    __shared__ __align__(8) unsigned long long bar_store;
    grad_chunk<T, TPR, NT, SCALED, REG, PRUNED, false>(acts, grads, labels, xlen, ylen, stat, alphas, betas, llf,
                                                       scale_in, scale_vec, d, hmajor, wait_ns, reg, p, T(0), chunk_raw,
                                                       &bar_store);
}
template <typename T, int TPR, int NT, bool SCALED, bool REG, bool PRUNED>
__global__ void __launch_bounds__(NT)
grad_chunk_delay_kernel(const T* __restrict__ acts, T* __restrict__ grads, const int* __restrict__ labels,
                        const int* __restrict__ xlen, const int* __restrict__ ylen,
                        const typename Real<T>::pair* __restrict__ stat,
                        const typename Lat<T>::val* __restrict__ alphas, const typename Lat<T>::val* __restrict__ betas,
                        const typename Lat<T>::val* __restrict__ llf, const T scale_in,
                        const T* __restrict__ scale_vec, const Dims d, const int hmajor, const uint32_t wait_ns,
                        const GradReg<T> reg, const Prune p, const T delay_log2) {
    extern __shared__ __align__(128) unsigned char chunk_raw[];   // declared here: see rowstats_chunk_kernel
    __shared__ __align__(8) unsigned long long bar_store;
    grad_chunk<T, TPR, NT, SCALED, REG, PRUNED, true>(acts, grads, labels, xlen, ylen, stat, alphas, betas, llf,
                                                      scale_in, scale_vec, d, hmajor, wait_ns, reg, p, delay_log2,
                                                      chunk_raw, &bar_store);
}
// the modified topology (DESIGN.md §11); scale, gradient options and delay penalty at run time, as grad_row_mod_kernel
template <typename T, int TPR, int NT, bool PRUNED>
__global__ void __launch_bounds__(NT)
grad_chunk_mod_kernel(const T* __restrict__ acts, T* __restrict__ grads, const int* __restrict__ labels,
                      const int* __restrict__ xlen, const int* __restrict__ ylen,
                      const typename Real<T>::pair* __restrict__ stat,
                      const typename Lat<T>::val* __restrict__ alphas, const typename Lat<T>::val* __restrict__ betas,
                      const typename Lat<T>::val* __restrict__ llf, const T scale_in,
                      const T* __restrict__ scale_vec, const Dims d, const int hmajor, const uint32_t wait_ns,
                      const GradReg<T> reg, const Prune p, const T delay_log2) {
    extern __shared__ __align__(128) unsigned char chunk_raw[];   // declared here: see rowstats_chunk_kernel
    __shared__ __align__(8) unsigned long long bar_store;
    grad_chunk<T, TPR, NT, true, true, PRUNED, true, true>(acts, grads, labels, xlen, ylen, stat, alphas, betas, llf,
                                                           scale_in, scale_vec, d, hmajor, wait_ns, reg, p, delay_log2,
                                                           chunk_raw, &bar_store);
}

}  // namespace b200rnnt
