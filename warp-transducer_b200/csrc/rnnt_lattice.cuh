// rnnt_lattice.cuh — fp32 alpha/beta wavefronts in the LINEAR domain with an explicit exponent.
//
// The log-domain recurrence (lattice_kernel in rnnt_kernels.cuh, kept for fp64) puts
// SHFL -> DADD -> DADD -> F2F -> FMUL -> MUFU.EX2 -> FADD -> MUFU.LG2 -> FMUL -> F2F -> DADD on the
// dependent chain of every anti-diagonal, and that chain, not the batch, sets the time per diagonal.  Here a lattice value is  v * 2^e  with v a float in [1,2) and e an
// int, and a transition probability is  m * 2^k  (m in [0.71,1.42], k int), both prepared by pass 1:
//
//   product   v*m, e+k                                         FMUL || IADD          (4 cycles)
//   sum       E = max(e1,e2);  v = v1*2^(e1-E) + v2*2^(e2-E)   VIMNMX, IADD, VIMNMX, IMAD, FMUL/FFMA
//   renorm    e = E + exponent(v) - 127;  v = mantissa(v)      SHF, IADD3 || LOP3
//
// no MUFU, no conversions and no FP64 on the chain (~60 cycles + the shuffle).  "log zero" is
// (1, kEZero): alignment shifts are clamped to 2^-120, so such a term can never contribute and no
// -inf special cases are needed.  Values are stored as LogVal {e, log2 v} (8 B, the same size as the
// double the fp64 path stores); the gradient kernels consume them in the exp2 domain directly.
//
// Warps of one utterance are DECOUPLED: each thread fetches only its own column's factors (cp.async
// ring, completion counted per thread), the u-1 / u+1 neighbour inside a warp comes by shuffle, and
// across warps through a small tagged ring in shared memory (producer lane publishes {v,e,tag}, the
// consumer lane prefetches one step ahead and spins only if the tag is not there yet).  A downstream
// warp therefore settles a step or two behind its upstream neighbour and the shared-memory round trip
// leaves the dependent chain; there is no __syncthreads in the step loop.
//
// Layouts: the factors are read diagonal-major (one 16-byte cp.async per lane and step, contiguous across
// the lanes); alpha / beta are written CELL-major [b][t][u] for the gradient pass (rnnt_kernels.cuh: cell()),
// directly by single-warp wavefronts and through a per-lane delay line by multi-warp ones (see the body).
//
// Replaces reference compute_alphas_kernel / compute_betas_kernel (gpu_rnnt_kernel.h:11-47,79-113)
// and log_sum_exp (rnnt_helper.h:16-24) for fp32.
#pragma once
#include "rnnt_kernels.cuh"

namespace b200rnnt {

// v1*2^e1 + v2*2^e2, normalised
__device__ __forceinline__ void lin_add(float v1, int e1, float v2, int e2, float& v, int& e) {
    const int E = max(e1, e2);
    const int d1 = min(E - e1, 120), d2 = min(E - e2, 120);
    const float s1 = __int_as_float(0x3f800000 - (d1 << 23));
    const float s2 = __int_as_float(0x3f800000 - (d2 << 23));
    const float w = fmaf(v2, s2, v1 * s1);
    const int bits = __float_as_int(w);
    e = max(E + (bits >> 23) - 127, kEZero);
    v = __int_as_float((bits & 0x007fffff) | 0x3f800000);
}
constexpr int kLinRing = 8;    // the step loop is unrolled by this; the factor ring holds RD = 8, 16 or 32 diagonals per thread
constexpr int kEdge = 16;      // slots of the cross-warp exchange ring (multiple of kLinRing, power of two)
constexpr int kEdgeWarps = 32;
constexpr int kLinStaticSmem = kEdgeWarps * kEdge * 16 + kEdgeWarps * 4 + 16;

// ---- shared memory by 32-bit shared-space address (no generic->shared conversion in the step loop) ----
__device__ __forceinline__ void cp_async16_s(uint32_t dst, const void* gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
// ---- cross-warp exchange.  One 16-byte slot = {v bits, tag, e, tag}: each 8-byte half carries the tag,
// so a torn slot shows mismatching tags.  The producer's ONE publishing lane stores (predicated, no
// branch); the consumer warp reads the slot with ALL lanes (same address: a broadcast), so the "is it
// there yet" test and the spin are warp-uniform and the shuffles around them stay convergent. ----------
__device__ __forceinline__ void edge_publish(uint32_t slot, float v, int e, int tag, bool pred) {
    asm volatile(
        "{ .reg .pred p; setp.ne.b32 p, %5, 0; @p st.volatile.shared.v4.b32 [%0], {%1, %2, %3, %2}; }" ::"r"(slot),
        "r"(__float_as_int(v)), "r"(tag), "r"(e), "r"(0), "r"((int)pred)
        : "memory");
}
__device__ __forceinline__ bool edge_read(uint32_t slot, int tag, float& v, int& e) {
    int a, b, c, d;
    asm volatile("ld.volatile.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"(slot) : "memory");
    v = __int_as_float(a);
    e = c;
    return b == tag && d == tag;
}
__device__ __forceinline__ int lds_volatile(uint32_t addr) {
    int v;
    asm volatile("ld.volatile.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void sts_volatile(uint32_t addr, int v) {
    asm volatile("st.volatile.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

// =================================================================================================
// grid = (N, 1 or 2): blockIdx.y 0 -> alpha, 1 -> beta.  Every lane owns COLS ADJACENT columns
// (u = (thread * COLS) + c), a warp 32*COLS of them; blockDim = ceil(maxU / (32*COLS)) warps.
// Step s = 0..last visits anti-diagonal n = s (alpha) or n = last - s (beta); column u owns cell (n-u, u).
//
// Why several columns per lane: the neighbour of a lane's inner columns is the lane's own adjacent
// column from the previous step (a register), only the first (alpha) / last (beta) column's neighbour
// crosses lanes - ONE shuffle pair per step serves COLS cells, the COLS cell updates are independent
// (ILP), and a wavefront of U columns needs U/(32*COLS) warps instead of U/32: with two columns per
// lane 33..64 labels are a single warp with no cross-warp exchange at all.
// (See lattice_cols() for when that pays and when it does not.)
// =================================================================================================
//
// MOD: the modified topology (DESIGN.md §11), one transition per frame.  The label term of cell (t,u) comes from
// (t-1,u-1) (alpha) / (t+1,u+1) (beta), which the neighbouring column held two diagonals before, so the offer
// that crosses columns is the one of the previous step: ov2 / sv2 below, one step behind ov / sv.  Alpha runs one
// diagonal further, to the virtual cell (T, U-1), whose value is the log-likelihood.
template <int COLS, bool MULTI, bool BACKWARD, int RD, bool MOD = false>
__device__ __forceinline__ void lattice_lin_body(const float4* __restrict__ fac, const int* __restrict__ xlen,
                                                 const int* __restrict__ ylen, LogVal* __restrict__ out,
                                                 LogVal* __restrict__ llout, float* __restrict__ costs,
                                                 const Dims& d, uint32_t ring_base, uint32_t edge_base,
                                                 uint32_t prog_base, uint32_t delay_base, int* bad_any) {
    constexpr int DIR = BACKWARD ? -1 : 1;
    static_assert(RD % kLinRing == 0 && RD >= kLinRing, "ring depth: a multiple of the unroll factor");
    static_assert(!(MULTI && COLS > 1), "the store delay line below is written for one column per lane");
    static_assert(kLinRing == 8, "delay line depth = unroll factor = 8");
    const int b = blockIdx.x;
    const int tid = threadIdx.x;
    const int NT = blockDim.x;
    const int lane = tid & 31;
    // broadcast from lane 0 so the compiler treats the warp index (and everything derived from it:
    // has_src / has_dst, the exchange addresses) as warp-uniform - no divergence handling in the step loop
    const int warp = MULTI ? __shfl_sync(0xffffffffu, tid >> 5, 0) : 0;
    const int u0 = tid * COLS;             // first column of this lane
    int Tb, Ub;
    utt_extent(d, xlen, ylen, b, Tb, Ub);
    const size_t base = (size_t)b * lattice_block(d);
    const int last = Tb + Ub - 2 + (MOD && !BACKWARD ? 1 : 0);
    const int mU = d.maxU;
    const int nactive = (Ub + 32 * COLS - 1) / (32 * COLS);   // warps that own at least one column
    if (MULTI && warp >= nactive) return;                     // no column of this warp exists in this utterance

    unsigned width[COLS];                  // column c is active on diagonals n with (unsigned)(n - u0 - c) < width[c]
#pragma unroll
    for (int c = 0; c < COLS; ++c) width[c] = u0 + c < Ub ? (unsigned)Tb : 0u;
    const uint32_t step_bytes = NT * COLS * 16;
    uint32_t ring_u = ring_base + tid * (COLS * 16);     // this thread's COLS records of a ring slot
    asm volatile("" : "+r"(ring_u));                     // opaque: keep it in a register, do not rematerialise the cvta
    const int dstep = DIR * mU;                          // pointer step per diagonal in step order
    const int n0 = BACKWARD ? last : 0;
    const float4* gp = fac + base + u0 + (ptrdiff_t)n0 * mU;  // column u0's record of the next diagonal to fetch
    // lattice values go out CELL-MAJOR (see cell() in rnnt_kernels.cuh): cell (n-u, u) = n*mU - u*(mU-1)
    ptrdiff_t si = (ptrdiff_t)b * d.maxT * mU + (ptrdiff_t)n0 * mU - (ptrdiff_t)u0 * (mU - 1);
    // Multi-warp wavefronts: a step's 32 cells of a warp lie in 32 different rows t - written directly, every
    // warp-store is 32 sectors, and ten warps of one CTA saturate the SM's store path (measured: 0.40 -> 0.69 ms
    // at U = 301).  Each lane therefore DELAYS its store by kd steps through a private 8-deep line in shared
    // memory, kd = 7 - u%8 (alpha) / u%8 (beta): the 8 lanes of a group then store the same row t at the same
    // step - 64 contiguous bytes per group, 2-3 sectors instead of 8.
    const int kd = MULTI ? (BACKWARD ? (u0 & 7) : 7 - (u0 & 7)) : 0;
    const uint32_t delay_u = delay_base + (uint32_t)(tid >> 5) * 2048u + (uint32_t)lane * 8u;   // [8][32] x 8 B per warp
    const int kdn = (8 - kd) & 7;        // row of step s - kd  =  (s + kdn) & 7
    si -= (ptrdiff_t)kd * DIR * mU;
    int nu = n0 - u0;                                    // (current diagonal) - u0
    // Ring slots that no copy will fill hold NEUTRAL factors {1, 0, 1, log zero}: the step body below runs
    // unconditionally - a column that is not active yet keeps its "log zero" unchanged (and beta's virtual
    // beta(T,U-1) = 1 in column U-1 cannot leak into column U-2: in MOD it reaches U-2 one step later, through
    // that column's own, real label factor of (T-1,U-2)), a column that has finished computes values nobody
    // reads - and only the lattice STORE is predicated.
    auto neutral = [](uint32_t addr) {
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %1, %3};" ::"r"(addr), "r"(0x3f800000), "r"(0), "r"(kEZero) : "memory");
    };
#pragma unroll
    for (int k = 0; k < RD; ++k) {
#pragma unroll
        for (int c = 0; c < COLS; ++c) {
            const bool act = (unsigned)(nu - c + k * DIR) < width[c];
            const uint32_t slot = ring_u + k * step_bytes + c * 16;
            if (k < RD - 1 && act) cp_async16_s(slot, gp + c);
            else if (k < RD - 1 || !act) neutral(slot);   // (the last slot is step 0's refill target)
        }
        if (k < RD - 1) {
            cp_async_commit();
            gp += dstep;
        }
    }
    uint32_t roff = 0;   // byte offset of the ring slot of step s0 (always 0 when the ring is one unroll group deep)
    // running values.  alpha: (sv,se) = alpha(t,u) p_blank(t,u) offered to (t+1,u), (ov,oe) = alpha(t,u)
    // p_label(t,u) offered to (t,u+1).  beta: (sv,se) = beta(t+1,u).
    // MOD: (ov2,oe2) / (sv2,se2) = the value (ov,oe) / (sv,se) had one step earlier.  (fv,fe) = alpha's virtual
    // cell (T, U-1), taken from the last step.
    float sv[COLS], ov[COLS], ov2[COLS], sv2[COLS], fv[COLS];
    int se[COLS], oe[COLS], oe2[COLS], se2[COLS], fe[COLS];
#pragma unroll
    for (int c = 0; c < COLS; ++c) {
        sv[c] = ov[c] = 1.0f;
        se[c] = oe[c] = kEZero;
        if (MOD) sv2[c] = ov2[c] = fv[c] = 1.0f, se2[c] = oe2[c] = fe[c] = kEZero;
        if (!BACKWARD && u0 + c == 0) se[c] = 0;        // alpha(0,0) = 1 enters as the "stay" term of step 0
        if (BACKWARD && u0 + c == Ub - 1) se[c] = 0;    // virtual beta(T, U-1) = 1
    }
    float nansum = 0.0f;                                 // NaN factor anywhere -> NaN here
    // cross-warp neighbour (warp-uniform): alpha reads warp-1's lane 31, beta reads warp+1's lane 0
    const bool has_src = MULTI && (BACKWARD ? warp + 1 < nactive : warp > 0);
    const bool has_dst = MULTI && (BACKWARD ? warp > 0 : warp + 1 < nactive);
    const bool edge_lane = BACKWARD ? lane == 31 : lane == 0;   // the lane without a neighbour inside the warp
    const bool pub_lane = BACKWARD ? lane == 0 : lane == 31;    // the lane whose value the next warp needs
    const int edge_bias = edge_lane ? kEZero : 0;
    const uint32_t src_edge = edge_base + (BACKWARD ? warp + 1 : warp - 1) * (kEdge * 16);
    const uint32_t my_edge = edge_base + warp * (kEdge * 16);
    const uint32_t dst_prog = prog_base + (BACKWARD ? warp - 1 : warp + 1) * 4;
    float pv = 1.0f;   // cross-warp value for the coming step (prefetched)
    int pe = kEZero;
    bool pok = true;

    for (int s0 = 0; s0 <= last; s0 += kLinRing) {
        const uint32_t eoff = (uint32_t)(s0 & (kEdge - 1)) * 16;
        if (MULTI && has_dst) {
            // do not lap the consumer: this pass writes slots that hold the steps of one pass ago
            while (lds_volatile(dst_prog) < s0 - kLinRing) {}
        }
#pragma unroll
        for (int j = 0; j < kLinRing; ++j) {
            const int s = s0 + j;
            if (s > last) break;
            cp_async_wait<RD - 2>();   // this thread's factors of the current diagonal have landed
            // refill the slot of the previous step (private to this thread, already consumed)
            uint32_t prev;
            if (RD == kLinRing) prev = ring_u + ((j + kLinRing - 1) % kLinRing) * step_bytes;
            else if (j > 0) prev = ring_u + roff + (j - 1) * step_bytes;
            else prev = ring_u + (roff == 0 ? RD * step_bytes : roff) - step_bytes;
#pragma unroll
            for (int c = 0; c < COLS; ++c)
                if ((unsigned)(nu - c + (RD - 1) * DIR) < width[c]) cp_async16_s(prev + c * 16, gp + c);
            cp_async_commit();
            gp += dstep;
            float4 f[COLS];   // neutral / stale factors where a column is not active
#pragma unroll
            for (int c = 0; c < COLS; ++c) f[c] = lds128(ring_u + (RD == kLinRing ? 0u : roff) + j * step_bytes + c * 16);

            // the one neighbour value that crosses lanes, from the previous step
            float nv;
            int ne;
            if (BACKWARD) {
                nv = __shfl_down_sync(0xffffffffu, MOD ? sv2[0] : sv[0], 1);
                ne = __shfl_down_sync(0xffffffffu, MOD ? se2[0] : se[0], 1);
            } else {
                nv = __shfl_up_sync(0xffffffffu, MOD ? ov2[COLS - 1] : ov[COLS - 1], 1);
                ne = __shfl_up_sync(0xffffffffu, MOD ? oe2[COLS - 1] : oe[COLS - 1], 1);
            }
            if (MULTI && has_src) {
                // value of step s-1 (tag s) from the neighbouring warp; at s == 0 nothing beside is active
                const uint32_t slot = src_edge + ((eoff + (uint32_t)(j + kEdge - 1) * 16) & (kEdge * 16 - 1));
                if (s > 0)
                    while (!pok) pok = __all_sync(0xffffffffu, edge_read(slot, s, pv, pe));
                if (edge_lane) nv = pv, ne = pe;
            } else {
                ne += edge_bias;   // the lane without a neighbour: push its (own, shuffled-back) value to log zero
            }
            float v[COLS];
            int e[COLS];
            if (BACKWARD) {
                // beta(t,u) = beta(t+1,u) p_blank(t,u) + beta(t,u+1) p_label(t,u);  (t,u+1): the next column of
                // this lane (previous step's value), or the next lane's first column for the last one
                // (MOD: beta(t,u) = beta(t+1,u) p_blank(t,u) + beta(t+1,u+1) p_label(t,u), the next column's value
                // of two steps ago)
#pragma unroll
                for (int c = 0; c < COLS; ++c) {
                    const int cn = c + 1 < COLS ? c + 1 : c;
                    const float rv = c + 1 < COLS ? (MOD ? sv2[cn] : sv[cn]) : nv;
                    const int re = c + 1 < COLS ? (MOD ? se2[cn] : se[cn]) : ne;
                    lin_add(sv[c] * f[c].x, se[c] + __float_as_int(f[c].y), rv * f[c].z, re + __float_as_int(f[c].w), v[c], e[c]);
                }
#pragma unroll
                for (int c = 0; c < COLS; ++c) {
                    if (MOD) sv2[c] = sv[c], se2[c] = se[c];
                    sv[c] = v[c], se[c] = e[c];
                }
            } else {
                // alpha(t,u) = [alpha(t-1,u) p_blank(t-1,u)] + [alpha(t,u-1) p_label(t,u-1)];  (t,u-1): the previous
                // column of this lane (previous step's offer), or the previous lane's last column for the first one
                // (MOD: alpha(t,u) = [alpha(t-1,u) p_blank(t-1,u)] + [alpha(t-1,u-1) p_label(t-1,u-1)], the previous
                // column's offer of two steps ago)
#pragma unroll
                for (int c = 0; c < COLS; ++c) {
                    const int cp = c > 0 ? c - 1 : 0;
                    const float lv = c > 0 ? (MOD ? ov2[cp] : ov[cp]) : nv;
                    const int le = c > 0 ? (MOD ? oe2[cp] : oe[cp]) : ne;
                    lin_add(sv[c], se[c], lv, le, v[c], e[c]);
                }
#pragma unroll
                for (int c = 0; c < COLS; ++c) {
                    if (MOD) {
                        ov2[c] = ov[c], oe2[c] = oe[c];
                        if (s == last) fv[c] = v[c], fe[c] = e[c];   // the virtual cell (T, U-1) in column U-1
                    }
                    sv[c] = v[c] * f[c].x, se[c] = e[c] + __float_as_int(f[c].y);   // offered to (t+1, u)
                    ov[c] = v[c] * f[c].z, oe[c] = e[c] + __float_as_int(f[c].w);   // offered to (t, u+1)
                }
            }
#pragma unroll
            for (int c = 0; c < COLS; ++c) {
                nansum = fmaf(f[c].x, f[c].z, nansum);
                if (!MULTI) {
                    if ((unsigned)(nu - c) < width[c]) out[si - c * (mU - 1)] = to_logval(v[c], e[c]);
                } else {
                    const LogVal now = to_logval(v[c], e[c]);
                    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(delay_u + (uint32_t)(j & 7) * 256u), "r"(now.e),
                                 "r"(__float_as_int(now.l)) : "memory");
                    LogVal old;
                    int ol;
                    asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(old.e), "=r"(ol)
                                 : "r"(delay_u + (uint32_t)((j + kdn) & 7) * 256u) : "memory");
                    old.l = __int_as_float(ol);
                    if ((unsigned)(nu - kd * DIR) < width[c]) out[si] = old;   // the value of kd steps ago
                }
            }
            si += dstep;
            nu += DIR;
            if (MULTI) {
                const uint32_t slot_off = (eoff + (uint32_t)j * 16) & (kEdge * 16 - 1);
                if (has_dst)
                    edge_publish(my_edge + slot_off, BACKWARD ? (MOD ? sv2[0] : sv[0]) : (MOD ? ov2[COLS - 1] : ov[COLS - 1]),
                                 BACKWARD ? (MOD ? se2[0] : se[0]) : (MOD ? oe2[COLS - 1] : oe[COLS - 1]), s + 1, pub_lane);
                if (has_src) {
                    sts_volatile(prog_base + warp * 4, s);   // every lane, same value: progress of this warp
                    pok = __all_sync(0xffffffffu, edge_read(src_edge + slot_off, s + 1, pv, pe));   // prefetch for the next step
                }
            }
        }
        if (RD != kLinRing) {
            roff += kLinRing * step_bytes;
            if (roff == RD * step_bytes) roff = 0;
        }
    }
    cp_async_wait<0>();
    if (MULTI) {
        // drain the delay lines: the values of the last kd steps are still to be stored
        for (int s = last + 1; s <= last + 7; ++s) {
            LogVal old;
            int ol;
            asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(old.e), "=r"(ol)
                         : "r"(delay_u + (uint32_t)((s + kdn) & 7) * 256u) : "memory");
            old.l = __int_as_float(ol);
            if (s - kd <= last && (unsigned)(nu - kd * DIR) < width[0]) out[si] = old;
            si += dstep;
            nu += DIR;
        }
    }

    // NaN anywhere in this utterance's factors -> NaN cost (the reference propagates it through log_plus)
    bool bad = nansum != nansum;
    if (MULTI) {
        if (bad) atomicOr(bad_any, 1);
        asm volatile("bar.sync 1, %0;" ::"r"(nactive * 32) : "memory");
        bad = *(volatile int*)bad_any != 0;
    } else {
        bad = __any_sync(0xffffffffu, bad);
    }
    if (!BACKWARD) {
        // (sv, se) of column U-1 = alpha(T-1,U-1) p_blank(T-1,U-1) after the last step (MOD: (fv, fe) = alpha(T,U-1))
        if ((Ub - 1) / COLS == tid) {
            float llv = MOD ? fv[0] : sv[0];
            int lle = MOD ? fe[0] : se[0];
#pragma unroll
            for (int c = 1; c < COLS; ++c)
                if ((Ub - 1) % COLS == c) llv = MOD ? fv[c] : sv[c], lle = MOD ? fe[c] : se[c];
            LogVal ll = to_logval(llv, lle);
            float cost = -(logval_log2(ll) * 0.6931471805599453f);
            if (lle < kEDead) cost = INFINITY;
            if (bad) {
                cost = __int_as_float(0x7fc00000);
                ll.l = cost;
            }
            llout[b] = ll;
            costs[b] = cost;
        }
    } else if (tid == 0) {
        LogVal ll = to_logval(sv[0], se[0]);
        if (bad) ll.l = __int_as_float(0x7fc00000);
        llout[b] = ll;
    }
}

// The kernels' shared memory is declared in the kernels themselves (see rowstats_chunk_kernel) and handed in here.
template <int COLS, bool MULTI, int RD, bool MOD>
__device__ __forceinline__ void lattice_lin_run(const float4* __restrict__ fac, const int* __restrict__ xlen,
                                                const int* __restrict__ ylen, LogVal* __restrict__ alphas,
                                                LogVal* __restrict__ betas, LogVal* __restrict__ llf,
                                                LogVal* __restrict__ llb, float* __restrict__ costs, const Dims& d,
                                                unsigned char* ring_raw, int4* edge, int* prog, int* bad_any) {
    if (MULTI) {
        // tags start at 0 (= nothing published), progress at -1
        for (int i = threadIdx.x; i < kEdgeWarps * kEdge; i += blockDim.x) edge[i] = make_int4(0, 0, 0, 0);
        if (threadIdx.x < kEdgeWarps) prog[threadIdx.x] = -1;
        if (threadIdx.x == 0) *bad_any = 0;
        __syncthreads();
    }
    const uint32_t ring_base = smem_u32(ring_raw), edge_base = smem_u32(edge), prog_base = smem_u32(prog);
    const uint32_t delay_base = ring_base + (uint32_t)RD * blockDim.x * COLS * 16u;   // MULTI only: [warps][8][32] x 8 B
    pdl_trigger();   // the gradient kernel may launch and read the logits while the wavefront runs
    pdl_wait();      // pass 1's factors are complete and visible
    if (blockIdx.y == 0)
        lattice_lin_body<COLS, MULTI, false, RD, MOD>(fac, xlen, ylen, alphas, llf, costs, d, ring_base, edge_base, prog_base, delay_base, bad_any);
    else
        lattice_lin_body<COLS, MULTI, true, RD, MOD>(fac, xlen, ylen, betas, llb, costs, d, ring_base, edge_base, prog_base, delay_base, bad_any);
}
template <int COLS, bool MULTI, int RD>
__global__ void __launch_bounds__(MULTI ? 1024 / COLS : 32)
lattice_lin_kernel(const float4* __restrict__ fac, const int* __restrict__ xlen, const int* __restrict__ ylen,
                   LogVal* __restrict__ alphas, LogVal* __restrict__ betas, LogVal* __restrict__ llf,
                   LogVal* __restrict__ llb, float* __restrict__ costs, const Dims d) {
    extern __shared__ __align__(16) unsigned char ring_raw[];   // [RD][blockDim.x][COLS] float4, thread-private
    __shared__ __align__(16) int4 edge[MULTI ? kEdgeWarps * kEdge : 1];
    __shared__ int prog[MULTI ? kEdgeWarps : 1];
    __shared__ int bad_any;
    lattice_lin_run<COLS, MULTI, RD, false>(fac, xlen, ylen, alphas, betas, llf, llb, costs, d, ring_raw, edge, prog,
                                            &bad_any);
}
// the modified topology (DESIGN.md §11)
template <int COLS, bool MULTI, int RD>
__global__ void __launch_bounds__(MULTI ? 1024 / COLS : 32)
lattice_lin_mod_kernel(const float4* __restrict__ fac, const int* __restrict__ xlen, const int* __restrict__ ylen,
                       LogVal* __restrict__ alphas, LogVal* __restrict__ betas, LogVal* __restrict__ llf,
                       LogVal* __restrict__ llb, float* __restrict__ costs, const Dims d) {
    extern __shared__ __align__(16) unsigned char ring_raw[];
    __shared__ __align__(16) int4 edge[MULTI ? kEdgeWarps * kEdge : 1];
    __shared__ int prog[MULTI ? kEdgeWarps : 1];
    __shared__ int bad_any;
    lattice_lin_run<COLS, MULTI, RD, true>(fac, xlen, ylen, alphas, betas, llf, llb, costs, d, ring_raw, edge, prog,
                                           &bad_any);
}

// Columns per lane for a label extent.  A lone warp issues about one instruction every few cycles whatever
// the instruction-level parallelism, so a warp-step costs in proportion to its instruction count: two columns
// per lane win where they remove the cross-warp exchange, while fewer, fatter warps lose at large U.
// -> two columns per lane exactly where that saves the exchange (33..64 labels), one column otherwise.
inline int lattice_cols(int maxU) { return maxU > 32 && maxU <= 64 ? 2 : 1; }
inline int lattice_threads(int maxU) {
    const int per_warp = 32 * lattice_cols(maxU);
    return (maxU + per_warp - 1) / per_warp * 32;
}
// Diagonals of factors each thread keeps in flight.  8 covers the DRAM latency of an otherwise idle GPU
// (8 steps x ~220 ns); next to the streaming passes of other batch groups the loaded latency is several
// microseconds and the multi-warp wavefront starves, so there the ring is as deep as ~100 KB allow.
// forced = 8 | 16 | 32 (tuning hook RNNT_B200_LAT_RING) overrides it where the ring fits.
inline int lattice_ring_depth(int maxU, bool co_running, int forced) {
    if (maxU <= 64) return 8;
    const size_t per_slot = (size_t)lattice_threads(maxU) * lattice_cols(maxU) * 16;
    int depth = 8;
    if (co_running)
        while (depth < 32 && per_slot * depth * 2 <= 100 * 1024) depth *= 2;
    if ((forced == 8 || forced == 16 || forced == 32) && per_slot * forced + kLinStaticSmem <= 200 * 1024) depth = forced;
    return depth;
}
// dynamic shared memory: the factor ring, plus (multi-warp kernels) one 2 KB store delay line per warp
inline size_t lattice_ring_bytes(int maxU, int depth) {
    const size_t threads = lattice_threads(maxU);
    return (size_t)depth * threads * lattice_cols(maxU) * 16 + (maxU > 64 ? threads * 64 : 0);
}

}  // namespace b200rnnt
