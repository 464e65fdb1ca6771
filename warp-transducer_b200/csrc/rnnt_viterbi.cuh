// rnnt_viterbi.cuh — forced alignment (DESIGN.md §12): the best path through the lattice pass 1 left in the
// workspace, and the frame at which it emits each label.
//
// One CTA per utterance, one thread per label column u (blockDim = ceil(maxU/32) warps).  Step s of the
// wavefront computes, in every column, the max-product recurrence
//
//   regular   step s = anti-diagonal n:  cell (s-u, u),   a = max( a(t-1,u) p_blank(t-1,u),  a(t,u-1) p_label(t,u-1) )
//   modified  step s = frame t:          cell (s, u),     a = max( a(t-1,u) p_blank(t-1,u),  a(t-1,u-1) p_label(t-1,u-1) )
//
// Both read the same two offers of the previous step: the column's own blank offer ("stay") and the label offer of
// column u-1 ("left"), which comes by shuffle inside a warp and through shared memory across warps (one
// __syncthreads per step, as lattice_kernel does).  The modified recurrence only looks one frame back, so it steps
// frame by frame; its column reads the factors of cell (t,u) at (t+u)*maxU + u of the diagonal-major array, the
// regular one reads one anti-diagonal per step.  A cp.async ring holds the next kRing - 1 steps' factors.
//
// Decision: "label" exactly when the label offer is strictly greater, so equal partial paths emit their labels as
// early as possible.  Every warp stores __ballot_sync of its 32 decisions as one word: dec[b][s][u/32].  After the
// last step one warp walks the decisions back from the final cell; each step of the walk goes back exactly one step
// s and u drops by at most one, so the 32 steps ahead lie in the column window [u-31, u] of the next 32 words'
// rows.  Lane k loads the (at most two) words of step s-k covering that window - one round trip per 32 steps - and
// the warp then resolves the 32 steps with shuffles.
//
// Values: fp32 (and the 16-bit storage types) keep the linear domain with an explicit exponent, v * 2^e with
// v in [1,2), as rnnt_lattice.cuh does; a product is one FMUL and a renormalisation, and the max of two
// normalised values is exact.  The only rounding is one per factor product, so the score's relative error in
// probability is about (T_b + U_b) 2^-24 whatever its magnitude.  fp64 adds natural-log probabilities.
#pragma once
#include "rnnt_kernels.cuh"

namespace b200rnnt {

// fp32 lattice: v * 2^e, log zero = exponents at kEZero (clamped there, as lin_add does)
struct LinVit {
    using fac = float4;   // {m_blank, k_blank, m_label, k_label}
    using out = float;
    struct V {
        float v;
        int e;
    };
    static __device__ __forceinline__ V zero() { return V{1.0f, kEZero}; }
    static __device__ __forceinline__ V one() { return V{1.0f, 0}; }
    static __device__ __forceinline__ V mul(V a, float m, float kbits) {
        const int bits = __float_as_int(a.v * m);   // in [0.71, 2.84): a positive normal float
        V r;
        r.e = max(a.e + __float_as_int(kbits) + (bits >> 23) - 127, kEZero);
        r.v = __int_as_float((bits & 0x007fffff) | 0x3f800000);
        return r;
    }
    static __device__ __forceinline__ V blank(V a, const fac& f) { return mul(a, f.x, f.y); }
    static __device__ __forceinline__ V label(V a, const fac& f) { return mul(a, f.z, f.w); }
    static __device__ __forceinline__ bool greater(V x, V y) { return x.e > y.e || (x.e == y.e && x.v > y.v); }
    static __device__ __forceinline__ bool nan_in(const fac& f) { return f.x != f.x || f.z != f.z; }
    static __device__ __forceinline__ V shfl_up(V a) {
        return V{__shfl_up_sync(0xffffffffu, a.v, 1), __shfl_up_sync(0xffffffffu, a.e, 1)};
    }
    static __device__ __forceinline__ bool alive(V a) { return a.e >= kEDead; }
    static __device__ __forceinline__ float score(V a) {
        return alive(a) ? (float)(((double)a.e + (double)log2f(a.v)) * 0.6931471805599453) : -INFINITY;
    }
};
// fp64 lattice: natural-log probabilities, max-plus
struct LogVit {
    using fac = double2;   // {lp_blank, lp_label}; lp_label is 0 where the cell has no label
    using out = double;
    using V = double;
    static __device__ __forceinline__ V zero() { return -(double)INFINITY; }
    static __device__ __forceinline__ V one() { return 0.0; }
    static __device__ __forceinline__ V blank(V a, const fac& f) { return a + f.x; }
    static __device__ __forceinline__ V label(V a, const fac& f) { return a + f.y; }
    static __device__ __forceinline__ bool greater(V x, V y) { return x > y; }
    static __device__ __forceinline__ bool nan_in(const fac& f) { return f.x != f.x || f.y != f.y; }
    static __device__ __forceinline__ V shfl_up(V a) { return __shfl_up_sync(0xffffffffu, a, 1); }
    static __device__ __forceinline__ bool alive(V a) { return a > -(double)INFINITY; }
    static __device__ __forceinline__ double score(V a) { return a; }
};

// words of the decision array per step, and steps per utterance (the regular lattice has at most maxT + maxU - 1)
__host__ __device__ __forceinline__ int viterbi_words(int maxU) { return (maxU + 31) / 32; }
__host__ __device__ __forceinline__ size_t viterbi_dec_block(const Dims& d) {
    return (size_t)(d.maxT + d.maxU) * viterbi_words(d.maxU);
}

template <typename Ops, bool MULTI, bool MOD>
__device__ __forceinline__ void viterbi_body(const typename Ops::fac* __restrict__ lp2, const int* __restrict__ xlen,
                                             const int* __restrict__ ylen, uint32_t* __restrict__ dec,
                                             int* __restrict__ frames, typename Ops::out* __restrict__ scores,
                                             const Dims& d, unsigned char* ring_raw, typename Ops::V (*edge)[32],
                                             int* alive_flag) {
    using P = typename Ops::fac;
    using V = typename Ops::V;
    P* ring = reinterpret_cast<P*>(ring_raw);   // [kRing][blockDim.x], one slot per thread and step
    const int b = blockIdx.x;
    const int u = threadIdx.x;
    const int NT = blockDim.x;
    const int lane = u & 31, warp = u >> 5;
    const int mU = d.maxU;
    const int W = viterbi_words(mU);
    int Tb, Ub;
    utt_extent(d, xlen, ylen, b, Tb, Ub);
    int* fr = frames + (size_t)b * (mU - 1);
    for (int j = u; j < mU - 1; j += NT) fr[j] = -1;   // padding, and every label of an utterance without a path
    const int last = MOD ? Tb : Tb + Ub - 2;            // MOD: step T_b is the virtual cell (T_b, U_b - 1)
    const unsigned width = u < Ub ? (unsigned)Tb : 0u;  // cell of step s exists iff (unsigned)t(s) < width
    uint32_t* db = dec + (size_t)b * viterbi_dec_block(d);
    const P* gp = lp2 + (size_t)b * lattice_block(d) + u + (MOD ? (size_t)u * mU : 0);   // factors of step 0
    P* ring_u = ring + u;
    int fs = 0;   // next step to fetch; step s lives in slot s % kRing
#pragma unroll
    for (int k = 0; k < kRing - 1; ++k) {
        if ((unsigned)(MOD ? fs : fs - u) < width) cp_async<sizeof(P)>(ring_u + k * NT, gp);
        cp_async_commit();
        gp += mU;
        ++fs;
    }
    V stay = u == 0 ? Ops::one() : Ops::zero();   // a(t-1,u) p_blank(t-1,u): the path enters at (0,0) with 1
    V off = Ops::zero();                          // a p_label of this column's previous cell, offered to u+1
    V fin = Ops::zero();                          // MOD: the virtual cell (T_b, U_b - 1), the last step's value
    bool bad = false;                             // a NaN factor in this utterance
    const bool has_label = u < Ub - 1;
    uint32_t* dp = db + warp;                     // this warp's decision word of the current step
    // unrolled by the ring depth, so that every ring slot is a constant offset; the step body has no branch
    for (int s0 = 0; s0 <= last; s0 += kRing) {
#pragma unroll
        for (int j = 0; j < kRing; ++j) {
            const int s = s0 + j;
            if (s > last) break;
            cp_async_wait<kRing - 2>();   // this thread's factors of step s have landed
            if (MULTI) {
                if (lane == 31) edge[j & 1][warp] = off;
                __syncthreads();
            }
            // refill the slot of step s-1 (private to this thread, already read)
            if ((unsigned)(MOD ? fs : fs - u) < width) cp_async<sizeof(P)>(ring_u + ((j + kRing - 1) % kRing) * NT, gp);
            cp_async_commit();
            gp += mU;
            ++fs;
            const P f = ring_u[j * NT];   // stale where the cell does not exist: every use below is masked
            V left = Ops::shfl_up(off);
            if (MULTI && lane == 0 && warp > 0) left = edge[j & 1][warp - 1];
            if (u == 0) left = Ops::zero();
            const bool take_label = Ops::greater(left, stay);
            const V a = take_label ? left : stay;
            const unsigned word = __ballot_sync(0xffffffffu, take_label);
            if (lane == 0) *dp = word;
            dp += W;
            const bool on = (unsigned)(MOD ? s : s - u) < width;
            bad |= on && Ops::nan_in(f);
            const V sb = Ops::blank(a, f), sl = Ops::label(a, f);
            stay = on ? sb : Ops::zero();
            off = on && has_label ? sl : Ops::zero();
            if (MOD) fin = a;
        }
    }
    cp_async_wait<0>();
    bad = __syncthreads_or(bad);
    // regular: the path leaves with the blank of (T_b-1, U_b-1), the stay offer column U_b-1 made at the last step
    if (u == Ub - 1) {
        const V best = MOD ? fin : stay;
        scores[b] = bad ? (typename Ops::out)NAN : Ops::score(best);
        *alive_flag = !bad && Ops::alive(best);
    }
    __syncthreads();   // every warp's decision words and the flag are visible
    if (warp != 0 || !*alive_flag) return;

    // backtrace from the final cell: step s, column cu; a label decision at (s, cu) means label cu-1 was emitted
    // at frame s - cu (regular, from (t, cu-1)) / s - 1 (modified, from (t-1, cu-1))
    int s = last, cu = Ub - 1;
    while (s > 0) {
        const int sk = s - lane;   // this lane's step
        const int wb = cu >> 5;
        uint32_t hi = 0, lo = 0;
        if (sk > 0) {
            hi = __ldcg(db + (size_t)sk * W + wb);
            if (wb > 0) lo = __ldcg(db + (size_t)sk * W + wb - 1);
        }
        // bit i of win: column cu - 31 + i of step sk
        const uint32_t win = (uint32_t)((((uint64_t)hi << 32) | lo) >> ((cu & 31) + 1));
        const int cu0 = cu;
        const int steps = min(s, 32);
        for (int k = 0; k < steps; ++k) {
            const uint32_t wk = __shfl_sync(0xffffffffu, win, k);
            if ((wk >> (cu - cu0 + 31)) & 1u) {
                if (lane == 0) fr[cu - 1] = MOD ? s - k - 1 : s - k - cu;
                --cu;
            }
        }
        s -= steps;
    }
}

template <bool MULTI>
__global__ void __launch_bounds__(1024)
viterbi_lin_kernel(const float4* __restrict__ lp2, const int* __restrict__ xlen, const int* __restrict__ ylen,
                   uint32_t* __restrict__ dec, int* __restrict__ frames, float* __restrict__ scores, const Dims d) {
    extern __shared__ __align__(16) unsigned char ring_raw[];
    __shared__ LinVit::V edge[2][32];
    __shared__ int alive_flag;
    viterbi_body<LinVit, MULTI, false>(lp2, xlen, ylen, dec, frames, scores, d, ring_raw, edge, &alive_flag);
}
template <bool MULTI>
__global__ void __launch_bounds__(1024)
viterbi_lin_mod_kernel(const float4* __restrict__ lp2, const int* __restrict__ xlen, const int* __restrict__ ylen,
                       uint32_t* __restrict__ dec, int* __restrict__ frames, float* __restrict__ scores, const Dims d) {
    extern __shared__ __align__(16) unsigned char ring_raw[];
    __shared__ LinVit::V edge[2][32];
    __shared__ int alive_flag;
    viterbi_body<LinVit, MULTI, true>(lp2, xlen, ylen, dec, frames, scores, d, ring_raw, edge, &alive_flag);
}
template <bool MULTI>
__global__ void __launch_bounds__(1024)
viterbi_kernel(const double2* __restrict__ lp2, const int* __restrict__ xlen, const int* __restrict__ ylen,
               uint32_t* __restrict__ dec, int* __restrict__ frames, double* __restrict__ scores, const Dims d) {
    extern __shared__ __align__(16) unsigned char ring_raw[];
    __shared__ double edge[2][32];
    __shared__ int alive_flag;
    viterbi_body<LogVit, MULTI, false>(lp2, xlen, ylen, dec, frames, scores, d, ring_raw, edge, &alive_flag);
}
template <bool MULTI>
__global__ void __launch_bounds__(1024)
viterbi_mod_kernel(const double2* __restrict__ lp2, const int* __restrict__ xlen, const int* __restrict__ ylen,
                   uint32_t* __restrict__ dec, int* __restrict__ frames, double* __restrict__ scores, const Dims d) {
    extern __shared__ __align__(16) unsigned char ring_raw[];
    __shared__ double edge[2][32];
    __shared__ int alive_flag;
    viterbi_body<LogVit, MULTI, true>(lp2, xlen, ylen, dec, frames, scores, d, ring_raw, edge, &alive_flag);
}

}  // namespace b200rnnt
