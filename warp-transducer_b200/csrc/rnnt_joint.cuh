// rnnt_joint.cuh — RNN-T loss for the ADDITIVE joint network, logits never materialised
// (SURVEY.md §8(f).2; the reference's own timing script builds its logits this way,
// pytorch_binding/test/test_time.py:73: acts = trans.unsqueeze(2) + pred.unsqueeze(1); the
// gradients w.r.t. the two factors are docs/rnnt_notes.tex:147-153).
//
//   h[b,t,u,k] = f[b,t,k] + g[b,u,k]
//
// Because exp(f+g) = exp(f)·exp(g), every V-length reduction of the standard path factorises:
//   S(t,u)   = sum_k e^{f_tk - mf_t} e^{g_uk - mg_u}            = (Ef · Eg^T)[t,u]
//   lse(t,u) = mf_t + mg_u + log S(t,u)
//   dL/df_tk = Ef_tk · sum_u Wm(t,u) Eg_uk  - (blank / label terms),   Wm = e^{alpha+beta-ll} / S
//   dL/dg_uk = Eg_uk · sum_t Wm(t,u) Ef_tk  - (blank / label terms)
// i.e. three small batched fp32 GEMMs around the SAME lattice kernel, and HBM traffic of
// O(N (T+U) V) instead of O(N T U V): 0.44 GB instead of 24 GB on the README large-vocabulary shape.
// fp32 FMA GEMMs, not tensor cores: the sums feed a logarithm and need ~1e-6 relative accuracy,
// and the whole contraction is only 3 x 2 GFMA.
// Limitation (documented in DESIGN.md): the factor-wise maxima bound the terms by 1 but not from
// below; if max_k(f+g) is more than ~85 nats under mf+mg the fp32 sum underflows.
#pragma once
#include <float.h>
#include "rnnt_kernels.cuh"
#include "rnnt_lattice.cuh"
#include "rnnt_wgmma.cuh"

namespace b200rnnt {

struct JointDims {
    int N, T, U, V, blank;
};

// ---- J1: per row of a factor: max and exp(x - max) ------------------------------------------------
// Rows come R per utterance (R = T for f, U for g); row r of utterance b is valid iff r < clamp(len[b] + add, 1, R)
// (len = xlen, add = 0 for f; len = ylen, add = 1 for g).  A padded row is never read: its exponentials, max and
// sum are written as 0, so whatever the caller left there (NaN, inf) cannot reach a contraction as 0 * NaN.
__device__ __forceinline__ bool joint_row_valid(const int* __restrict__ len, int add, int R, int row) {
    const int b = row / R;
    return row - b * R < min(max(__ldg(len + b) + add, 1), R);
}

// one warp per row of V elements (rows = N*T for f, N*U for g)
// SUM (smoothing, DESIGN.md §9): also sum[row] = sum_k e_k * wv[k] (wv NULL: 1) from the exponentials in registers
template <bool SUM = false>
__global__ void __launch_bounds__(256)
joint_prep_kernel(const float* __restrict__ x, float* __restrict__ e, float* __restrict__ mx, int rows, int V,
                  const int* __restrict__ len, int add, int R, const float* __restrict__ wv, float* __restrict__ sum) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    if (!joint_row_valid(len, add, R, row)) {
        float* q = e + (size_t)row * V;
        for (int k = lane; k < V; k += 32) q[k] = 0.0f;
        if (lane == 0) {
            mx[row] = 0.0f;
            if (SUM) sum[row] = 0.0f;
        }
        return;
    }
    const float* p = x + (size_t)row * V;
    float m = -INFINITY;
    for (int k = lane; k < V; k += 32) m = fmaxf(m, __ldg(p + k));
    m = group_max<32>(m);
    const float mz = (m == -INFINITY) ? 0.0f : m;
    float* q = e + (size_t)row * V;
    if (!SUM) {
        for (int k = lane; k < V; k += 32) q[k] = Real<float>::exp(__ldg(p + k) - mz);
    } else {
        float sm = 0.0f;
        for (int k = lane; k < V; k += 32) {
            const float ek = Real<float>::exp(__ldg(p + k) - mz);
            q[k] = ek;
            sm = wv ? fmaf(ek, __ldg(wv + k), sm) : sm + ek;
        }
        sm = group_sum<32>(sm);
        if (lane == 0) sum[row] = sm;
    }
    if (lane == 0) mx[row] = m;
}

// Same, one CTA per row with the whole row in registers (V % 4 == 0, V <= 256*4*NV): the factor is read
// ONCE (16-byte loads, all in flight before first use) and its exponentials written once with 16-byte
// stores - the streaming shape of rowstats_row_kernel.
template <int NV, bool SUM = false>
__global__ void __launch_bounds__(256)
joint_prep_row_kernel(const float* __restrict__ x, float* __restrict__ e, float* __restrict__ mx, int V,
                      const int* __restrict__ len, int add, int R, const float* __restrict__ wv,
                      float* __restrict__ sum) {
    __shared__ float sh[8];
    const int row = blockIdx.x, nv = V >> 2;
    if (!joint_row_valid(len, add, R, row)) {   // the whole CTA takes this branch
        float4* q = reinterpret_cast<float4*>(e + (size_t)row * V);
        for (int i = threadIdx.x; i < nv; i += 256) q[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (threadIdx.x == 0) {
            mx[row] = 0.0f;
            if (SUM) sum[row] = 0.0f;
        }
        return;
    }
    const float4* p = reinterpret_cast<const float4*>(x + (size_t)row * V);
    float4 v[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        const int i = threadIdx.x + j * 256;
        v[j] = i < nv ? __ldg(p + i) : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    }
    float m = -INFINITY;
#pragma unroll
    for (int j = 0; j < NV; ++j) m = fmaxf(m, fmaxf(fmaxf(v[j].x, v[j].y), fmaxf(v[j].z, v[j].w)));
    m = group_max<32>(m);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = m;
    __syncthreads();
    m = sh[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) m = fmaxf(m, sh[w]);
    const float mz = (m == -INFINITY) ? 0.0f : m;
    float4* q = reinterpret_cast<float4*>(e + (size_t)row * V);
    float sm = 0.0f;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        const int i = threadIdx.x + j * 256;
        if (i < nv) {
            float4 o;
            o.x = Real<float>::exp(v[j].x - mz);
            o.y = Real<float>::exp(v[j].y - mz);
            o.z = Real<float>::exp(v[j].z - mz);
            o.w = Real<float>::exp(v[j].w - mz);
            q[i] = o;
            if (SUM) {
                if (wv) {
                    const float4 c = __ldg(reinterpret_cast<const float4*>(wv) + i);
                    sm = fmaf(o.x, c.x, fmaf(o.y, c.y, fmaf(o.z, c.z, fmaf(o.w, c.w, sm))));
                } else {
                    sm += (o.x + o.y) + (o.z + o.w);
                }
            }
        }
    }
    if (SUM) {   // fixed-order block sum (deterministic)
        __shared__ float ss[8];
        sm = group_sum<32>(sm);
        if ((threadIdx.x & 31) == 0) ss[threadIdx.x >> 5] = sm;
        __syncthreads();
        if (threadIdx.x == 0) {
            float t = ss[0];
#pragma unroll
            for (int w = 1; w < 8; ++w) t += ss[w];
            sum[row] = t;
        }
    }
    if (threadIdx.x == 0) mx[row] = m;
}

// ---- generic batched fp32 GEMM  C[b](m,n) = sum_k A[b](m,k) * B[b](k,n), strided operands ----------
// 64x64 tile, 16-deep k-chunks through shared memory, 256 threads x (4x4) outputs.  Epilogue
// functor Epi(b, m, n, acc) writes the result.
struct Operand {
    const float* p;
    size_t batch;  // elements between batches
    int s_outer;   // stride of the m (A) / n (B) index
    int s_k;       // stride of the k index
};

template <typename Epi, int TN = 64, int KC = 16>
__global__ void __launch_bounds__(256)
joint_gemm_kernel(Operand A, Operand B, int M, int Nn, int Kfull, int slices, Epi epi) {
    // 64 x TN output tile (TN = 32 for skinny right-hand sides), KC-deep k-chunks
    constexpr int PN = TN / 16;  // output columns per thread
    __shared__ float sa[KC][64 + 1], sb[KC][TN + 1];
    // blockIdx.z = batch * slices + k-slice; each slice covers a KC-aligned range of K
    const int b = blockIdx.z / slices, ks = blockIdx.z - b * slices;
    const int kper = ((Kfull + slices - 1) / slices + KC - 1) / KC * KC;
    const int kbeg = ks * kper;
    const int K = min(Kfull, kbeg + kper);
    const int m0 = blockIdx.y * 64, n0 = blockIdx.x * TN;
    const float* a = A.p + (size_t)b * A.batch;
    const float* bb = B.p + (size_t)b * B.batch;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;  // 16 x 16 threads, 4 x PN outputs each
    float acc[4][PN] = {};
    for (int k0 = kbeg; k0 < K; k0 += KC) {
        // cooperative loads; the index order follows whichever stride is 1 so reads coalesce
        for (int i = threadIdx.x; i < 64 * KC; i += 256) {
            int r, kk;
            if (A.s_k == 1) { kk = i % KC; r = i / KC; } else { r = i & 63; kk = i >> 6; }
            const int m = m0 + r, k = k0 + kk;
            sa[kk][r] = (m < M && k < K) ? __ldg(a + (size_t)m * A.s_outer + (size_t)k * A.s_k) : 0.0f;
        }
        for (int i = threadIdx.x; i < TN * KC; i += 256) {
            int r, kk;
            if (B.s_k == 1) { kk = i % KC; r = i / KC; } else { r = i % TN; kk = i / TN; }
            const int n = n0 + r, k = k0 + kk;
            sb[kk][r] = (n < Nn && k < K) ? __ldg(bb + (size_t)n * B.s_outer + (size_t)k * B.s_k) : 0.0f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < KC; ++kk) {
            float av[4], bv[PN];
#pragma unroll
            for (int i = 0; i < 4; ++i) av[i] = sa[kk][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < PN; ++j) bv[j] = sb[kk][tx * PN + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < PN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < PN; ++j) {
            const int m = m0 + ty * 4 + i, n = n0 + tx * PN + j;
            if (m < M && n < Nn) epi(blockIdx.z, m, n, acc[i][j]);
        }
}

// ---- J2: split-K partial sums (deterministic: one slab per K-slice, summed in fixed order) ---------
struct EpiPartial {
    float* part;  // [slices][N,T,U]
    size_t cells; // N*T*U
    int T, U, slices;
    __device__ void operator()(int bz, int t, int u, float acc) const {
        const int b = bz / slices, ks = bz - b * slices;
        part[(size_t)ks * cells + ((size_t)b * T + t) * U + u] = acc;
    }
};

// ---- J2 epilogue: S -> lse, lattice log-prob pair (diagonal-major), keep 1/S -----------------------
// SMOOTH (DESIGN.md §9): each factor is  c lp_c + lml lp_l + lma lp_a  (a term with scale 0 is left out), with
//   lp_c = f_k + g_k - lse,  lp_l = g_k - mg - log sg,  lp_a = f_k + log ug_k - mf - log A.
// DELAY (DESIGN.md §10): the label factor gains  delay ((T_b - 1)/2 - t)  after the smoothing interpolation, as in
// k2; joint_stats_delay_kernel runs it.  Everything downstream reads the penalised factors from lp2.
template <bool SMOOTH = false, bool DELAY = false>
struct EpiStats {
    const float *f, *g, *mf, *mg;
    const int *labels, *xlen, *ylen;
    float* inv_s;  // [N,T,U]
    float4* lp2;   // diagonal-major lattice factors (Lat<float>::fac)
    JointDims jd;
    Dims d;        // lattice geometry (maxT = T, maxU = U)
    const float *sg, *A, *lug;   // SMOOTH: [N,U] row sums of Eg, [N,T] Ef . ug, [V] log ug
    float c, lml, lma;           // SMOOTH: the three scales
    float delay;                 // DELAY: lambda
    __device__ float mix(const float* fr, const float* gr, int k, float lse, float Lg, float La) const {
        const float fk = __ldg(fr + k), gk = __ldg(gr + k);
        float lp = 0.0f;
        if (c != 0.0f) lp = c * ((fk + gk) - lse);
        if (lml != 0.0f) lp = fmaf(lml, gk - Lg, lp);
        if (lma != 0.0f) lp = fmaf(lma, (fk + __ldg(lug + k)) - La, lp);
        return lp;
    }
    __device__ void operator()(int b, int t, int u, float S) const {
        int Tb, Ub;
        utt_extent(d, xlen, ylen, b, Tb, Ub);
        const size_t cell = ((size_t)b * jd.T + t) * jd.U + u;
        if (t >= Tb || u >= Ub) {
            inv_s[cell] = 0.0f;
            return;
        }
        const float mft = mf[(size_t)b * jd.T + t], mgu = mg[(size_t)b * jd.U + u];
        const float lse = mft + mgu + logf(S);
        inv_s[cell] = 1.0f / S;
        const float* fr = f + ((size_t)b * jd.T + t) * jd.V;
        const float* gr = g + ((size_t)b * jd.U + u) * jd.V;
        const bool has_label = u < Ub - 1;
        if (SMOOTH) {
            const float Lg = mgu + logf(__ldg(sg + (size_t)b * jd.U + u));
            const float La = lma != 0.0f ? mft + logf(__ldg(A + (size_t)b * jd.T + t)) : 0.0f;
            const float lpb = mix(fr, gr, jd.blank, lse, Lg, La);
            float lpl = 0.0f;
            if (has_label) lpl = mix(fr, gr, __ldg(labels + (size_t)b * (jd.U > 1 ? jd.U - 1 : 0) + u), lse, Lg, La);
            if (DELAY && has_label) lpl += delay * delay_bracket<float>(Tb, (uint32_t)t);
            lp2[skew(d, b, t, u)] = make_fac(lpb, lpl, has_label);
            return;
        }
        const float lpb = (__ldg(fr + jd.blank) + __ldg(gr + jd.blank)) - lse;
        float lpl = 0.0f;
        if (has_label) {
            const int y = __ldg(labels + (size_t)b * (jd.U > 1 ? jd.U - 1 : 0) + u);
            lpl = (__ldg(fr + y) + __ldg(gr + y)) - lse;
            if (DELAY) lpl += delay * delay_bracket<float>(Tb, (uint32_t)t);
        }
        lp2[skew(d, b, t, u)] = make_fac(lpb, lpl, has_label);
    }
};

template <typename Epi>
__device__ __forceinline__ void joint_stats(const float* __restrict__ part, int slices, const Epi& epi) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= epi.d.rows) return;
    uint32_t bt, u, b, t;
    epi.d.divU.divmod(r, bt, u);
    epi.d.divT.divmod(bt, b, t);
    float S = 0.0f;
    for (int ks = 0; ks < slices; ++ks) S += part[(size_t)ks * epi.d.rows + r];
    epi((int)b, (int)t, (int)u, S);
}
template <bool SMOOTH = false>
__global__ void __launch_bounds__(256)
joint_stats_kernel(const float* __restrict__ part, int slices, const EpiStats<SMOOTH> epi) {
    joint_stats(part, slices, epi);
}
template <bool SMOOTH = false>
__global__ void __launch_bounds__(256)
joint_stats_delay_kernel(const float* __restrict__ part, int slices, const EpiStats<SMOOTH, true> epi) {
    joint_stats(part, slices, epi);
}

// ---- J3: per cell weights from the lattices ---------------------------------------------------------
//   Wm = e^{alpha+beta-ll} / S ;  Bk = blank-transition occupancy ;  Lb = label-transition occupancy
// REG (FastEmit, rnnt_kernels.cuh GradReg): Wm += lambda Lb / S and Lb *= 1 + lambda.
// SMOOTH (DESIGN.md §9): Wm carries the scale c of the full-joint term; Bk / Lb stay the factor gradients.
// MOD (the modified topology, DESIGN.md §11): Lb reads beta(t+1,u+1) (on the last frame only u = U-2 has a label
// transition, into the virtual beta(T,U-1) = log 1), and an utterance without a path gets zero weights.
template <bool REG, bool SMOOTH, bool MOD>
__device__ __forceinline__ void joint_weights(const float4* __restrict__ lp2, const LogVal* __restrict__ alphas,
                                              const LogVal* __restrict__ betas, const LogVal* __restrict__ llf,
                                              const float* __restrict__ inv_s, const int* __restrict__ xlen,
                                              const int* __restrict__ ylen, float* __restrict__ Wm,
                                              float* __restrict__ Bk, float* __restrict__ Lb, const float scale_in,
                                              const float* __restrict__ scale_vec, const Dims& d, const int wm_pitch,
                                              const float lam, const float c) {
    // Wm rows have `wm_pitch` >= maxU entries (zero beyond maxU: the tensor-core kernel fetches them as aligned
    // float4 rows); Bk / Lb / inv_s are [N,T,maxU].  One thread per Wm entry.
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= (uint32_t)d.N * d.maxT * wm_pitch) return;
    const uint32_t bt = q / (uint32_t)wm_pitch, u = q % (uint32_t)wm_pitch;
    if (u >= (uint32_t)d.maxU) {
        Wm[q] = 0.0f;
        return;
    }
    const uint32_t r = bt * d.maxU + u;
    uint32_t b, t;
    d.divT.divmod(bt, b, t);
    int Tb, Ub;
    utt_extent(d, xlen, ylen, b, Tb, Ub);
    float w = 0.0f, bk = 0.0f, lb = 0.0f;
    const float scale = scale_vec ? scale_in * __ldg(scale_vec + b) : scale_in;
    if ((int)t < Tb && (int)u < Ub && !(MOD && ll_dead(llf, b))) {
        // everything in the exp2 domain: log2 occupancy = exact integer part + small float part
        const float4 fc = lp2[skew(d, b, t, u)];
        const size_t q = cell(d, b, t, u);
        const LogVal a = alphas[q], ll = llf[b], bq = betas[q];
        const int oe = a.e - ll.e;
        const float ol = a.l - ll.l;
        const float lpb2 = (float)__float_as_int(fc.y) + log2f(fc.x);   // log2 p_blank
        w = scale * exp2f((float)(oe + bq.e) + (ol + bq.l)) * inv_s[r];
        if ((int)t < Tb - 1) {
            const LogVal bn = betas[q + d.maxU];
            bk = scale * exp2f((float)(oe + bn.e) + (ol + bn.l) + lpb2);
        } else if ((int)u == Ub - 1) {
            bk = scale * exp2f((float)oe + ol + lpb2);
        }
        if ((int)u < Ub - 1 && (!MOD || (int)t < Tb - 1 || (int)u == Ub - 2)) {
            // MOD on the last frame: the virtual beta(T,U-1), log 0 = 0, is LogVal {0, 0}
            const bool term = MOD && (int)t == Tb - 1;
            const LogVal bn = term ? LogVal{0, 0.0f} : betas[q + (MOD ? d.maxU + 1 : 1)];
            const float lpl2 = (float)__float_as_int(fc.w) + log2f(fc.z);
            lb = scale * exp2f((float)(oe + bn.e) + (ol + bn.l) + lpl2);
            if (REG) {
                w = fmaf(lam * lb, inv_s[r], w);
                lb *= 1.0f + lam;
            }
        }
        if (SMOOTH) w *= c;
    }
    Wm[q] = w;
    Bk[r] = bk;
    Lb[r] = lb;
}
template <bool REG = false, bool SMOOTH = false>
__global__ void __launch_bounds__(256)
joint_weights_kernel(const float4* __restrict__ lp2, const LogVal* __restrict__ alphas,
                     const LogVal* __restrict__ betas, const LogVal* __restrict__ llf,
                     const float* __restrict__ inv_s, const int* __restrict__ xlen,
                     const int* __restrict__ ylen, float* __restrict__ Wm, float* __restrict__ Bk,
                     float* __restrict__ Lb, const float scale_in, const float* __restrict__ scale_vec,
                     const Dims d, const int wm_pitch, const float lam, const float c) {
    joint_weights<REG, SMOOTH, false>(lp2, alphas, betas, llf, inv_s, xlen, ylen, Wm, Bk, Lb, scale_in, scale_vec, d,
                                      wm_pitch, lam, c);
}
template <bool REG = false, bool SMOOTH = false>
__global__ void __launch_bounds__(256)
joint_weights_mod_kernel(const float4* __restrict__ lp2, const LogVal* __restrict__ alphas,
                         const LogVal* __restrict__ betas, const LogVal* __restrict__ llf,
                         const float* __restrict__ inv_s, const int* __restrict__ xlen,
                         const int* __restrict__ ylen, float* __restrict__ Wm, float* __restrict__ Bk,
                         float* __restrict__ Lb, const float scale_in, const float* __restrict__ scale_vec,
                         const Dims d, const int wm_pitch, const float lam, const float c) {
    joint_weights<REG, SMOOTH, true>(lp2, alphas, betas, llf, inv_s, xlen, ylen, Wm, Bk, Lb, scale_in, scale_vec, d,
                                     wm_pitch, lam, c);
}

// ---- pruning ranges (DESIGN.md §8) from the lattice a forward with beta left in the workspace ---------------
// With E = max(U_b - R, 0) and the occupancies  e_b(t,u) = exp(alpha(t,u) + lp_blank(t,u) + beta(t+1,u) - ll),
// e_y(t,u) = exp(alpha(t,u) + lp_y(t,u) + beta(t,u+1) - ll):
//   1. 0 < t < T_b - 1: s[t] = the smallest a in [0, E] maximising
//      sum_{u=a}^{min(a+R,U_b)-1} e_b(t,u) - [a>0] e_y(t,a-1)
//   2. s[0] = 0; s[T_b-1] = E if T_b > 1; s[t] = E for t >= T_b
//   3. t = T_b-2 down to 0: s[t] = min(max(s[t], s[t+1] - (R-1)), s[t+1])
// One CTA per utterance.  A warp takes a frame at a time: the frame's occupancies go to the warp's shared-memory
// rows, lane l scores the starts a = l, l+32, ... (strict > keeps its smallest best) and a shuffle argmax keeps the
// smallest a on ties.  Thread 0 then runs the sweep over the frame starts in shared memory.
// MOD (DESIGN.md §11): e_y(t,u) = exp(alpha(t,u) + lp_y(t,u) + beta(t+1,u+1) - ll); an utterance without a path
// scores every start 0 (so step 1 picks a = 0).
constexpr int kRangeWarps = 4;
inline size_t prune_ranges_smem(int maxT, int maxU) {
    return (size_t)kRangeWarps * 2 * maxU * sizeof(float) + (size_t)maxT * sizeof(int);
}
template <bool MOD>
__device__ __forceinline__ void joint_prune_ranges(const float4* __restrict__ lp2, const LogVal* __restrict__ alphas,
                                                   const LogVal* __restrict__ betas, const LogVal* __restrict__ llf,
                                                   const int* __restrict__ xlen, const int* __restrict__ ylen,
                                                   int* __restrict__ ranges, const Dims& d, const int R,
                                                   float* range_smem) {
    // range_smem: [kRangeWarps][2][maxU] occupancies, then [maxT] window starts
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int Tb, Ub;
    utt_extent(d, xlen, ylen, b, Tb, Ub);
    const int E = max(Ub - R, 0);
    float* eb = range_smem + (size_t)warp * 2 * d.maxU;
    float* ey = eb + d.maxU;
    int* s = reinterpret_cast<int*>(range_smem + (size_t)kRangeWarps * 2 * d.maxU);
    const LogVal ll = llf[b];
    const bool dead = MOD && ll_dead(llf, b);
    for (int t = 1 + warp; t < Tb - 1; t += kRangeWarps) {
        for (int u = lane; u < Ub; u += 32) {
            if (dead) {
                eb[u] = ey[u] = 0.0f;
                continue;
            }
            // exp2 domain, as joint_weights_kernel: exact integer exponent + small float part
            const float4 fc = lp2[skew(d, b, t, u)];
            const size_t q = cell(d, b, t, u);
            const LogVal a = alphas[q], bn = betas[q + d.maxU];
            const int oe = a.e - ll.e;
            const float ol = a.l - ll.l;
            eb[u] = exp2f((float)(oe + bn.e) + (ol + bn.l) + ((float)__float_as_int(fc.y) + log2f(fc.x)));
            if (u < Ub - 1) {
                const LogVal bl = betas[q + (MOD ? d.maxU + 1 : 1)];
                ey[u] = exp2f((float)(oe + bl.e) + (ol + bl.l) + ((float)__float_as_int(fc.w) + log2f(fc.z)));
            }
        }
        __syncwarp();
        float best = -INFINITY;
        int best_a = E;
        for (int a = lane; a <= E; a += 32) {
            float sc = 0.0f;
            const int end = min(a + R, Ub);
            for (int u = a; u < end; ++u) sc += eb[u];
            if (a > 0) sc -= ey[a - 1];
            if (sc > best) best = sc, best_a = a;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oa = __shfl_xor_sync(0xffffffffu, best_a, o);
            if (ob > best || (ob == best && oa < best_a)) best = ob, best_a = oa;
        }
        if (lane == 0) s[t] = best_a;
        __syncwarp();   // the rows are rewritten for the warp's next frame
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        s[0] = 0;
        if (Tb > 1) s[Tb - 1] = E;
        for (int t = Tb - 2; t >= 0; --t) s[t] = min(max(s[t], s[t + 1] - (R - 1)), s[t + 1]);
    }
    __syncthreads();
    for (int t = threadIdx.x; t < d.maxT; t += blockDim.x) ranges[(size_t)b * d.maxT + t] = t < Tb ? s[t] : E;
}
__global__ void __launch_bounds__(kRangeWarps * 32)
joint_prune_ranges_kernel(const float4* __restrict__ lp2, const LogVal* __restrict__ alphas,
                          const LogVal* __restrict__ betas, const LogVal* __restrict__ llf,
                          const int* __restrict__ xlen, const int* __restrict__ ylen, int* __restrict__ ranges,
                          const Dims d, const int R) {
    extern __shared__ float range_smem[];
    joint_prune_ranges<false>(lp2, alphas, betas, llf, xlen, ylen, ranges, d, R, range_smem);
}
__global__ void __launch_bounds__(kRangeWarps * 32)
joint_prune_ranges_mod_kernel(const float4* __restrict__ lp2, const LogVal* __restrict__ alphas,
                              const LogVal* __restrict__ betas, const LogVal* __restrict__ llf,
                              const int* __restrict__ xlen, const int* __restrict__ ylen, int* __restrict__ ranges,
                              const Dims d, const int R) {
    extern __shared__ float range_smem[];
    joint_prune_ranges<true>(lp2, alphas, betas, llf, xlen, ylen, ranges, d, R, range_smem);
}

// ---- J4/J5: out[b,r,v] = Eout[b,r,v] * sum_s W(r,s) * Ein[b,s,v]  (thin contraction over s) ----------
//   dF: r = t, s = u, W(r,s) = Wm[b,t,u], Ein = Eg, Eout = Ef
//   dG: r = u, s = t, W(r,s) = Wm[b,t,u] (transposed access), Ein = Ef, Eout = Eg
// One thread per vocabulary column (coalesced over v), RT output rows per block held in registers,
// the W tile broadcast from shared memory: RT FMAs per 4-byte load of Ein.
// SMOOTH (DESIGN.md §9): out = Eout * (acc + coef[b,r].x + coef[b,r].y * wv[v])   (wv NULL: no last term; coef
// NULL: no smoothing term on this product)
constexpr int kJointRT = 16, kJointSC = 64;
template <bool SMOOTH = false>
__global__ void __launch_bounds__(256)
joint_thin_kernel(const float* __restrict__ Wm, int w_stride_r, int w_stride_s, size_t w_batch,
                  const float* __restrict__ Ein, const float* __restrict__ Eout, float* __restrict__ out,
                  int R, int S, int V, const float2* __restrict__ coef, const float* __restrict__ wv) {
    __shared__ float sw[kJointSC][kJointRT];
    const int b = blockIdx.z, r0 = blockIdx.y * kJointRT;
    const int v = blockIdx.x * 256 + threadIdx.x;
    const float* w = Wm + (size_t)b * w_batch;
    const float* ein = Ein + (size_t)b * S * V;
    float acc[kJointRT];
#pragma unroll
    for (int i = 0; i < kJointRT; ++i) acc[i] = 0.0f;
    for (int s0 = 0; s0 < S; s0 += kJointSC) {
        for (int i = threadIdx.x; i < kJointSC * kJointRT; i += 256) {
            const int ss = i / kJointRT, rr = i % kJointRT;
            const int s = s0 + ss, r = r0 + rr;
            sw[ss][rr] = (s < S && r < R) ? __ldg(w + (size_t)r * w_stride_r + (size_t)s * w_stride_s) : 0.0f;
        }
        __syncthreads();
        if (v < V) {
            const int smax = min(kJointSC, S - s0);
            for (int ss = 0; ss < smax; ++ss) {
                const float e = __ldg(ein + (size_t)(s0 + ss) * V + v);
#pragma unroll
                for (int i = 0; i < kJointRT; ++i) acc[i] = fmaf(sw[ss][i], e, acc[i]);
            }
        }
        __syncthreads();
    }
    if (v < V) {
#pragma unroll
        for (int i = 0; i < kJointRT; ++i) {
            const int r = r0 + i;
            if (r < R) {
                const size_t o = ((size_t)b * R + r) * V + v;
                float x = acc[i];
                if (SMOOTH && coef) {
                    const float2 cf = __ldg(coef + (size_t)b * R + r);
                    x += cf.x;
                    if (wv) x = fmaf(cf.y, __ldg(wv + v), x);
                }
                out[o] = __ldg(Eout + o) * x;
            }
        }
    }
}

// generic-GEMM form of the same products, used when V is too short to give every thread a column
template <bool SMOOTH = false>
struct EpiGrad {
    const float* e;  // Ef [N,T,V] (or Eg [N,U,V])
    float* out;      // dF (or dG), same shape
    int rows, V;     // rows per batch (T or U)
    const float2* coef;   // SMOOTH: as joint_thin_kernel
    const float* wv;
    __device__ void operator()(int b, int m, int n, float acc) const {
        const size_t i = ((size_t)b * rows + m) * V + n;
        if (SMOOTH && coef) {
            const float2 cf = __ldg(coef + (size_t)b * rows + m);
            acc += cf.x;
            if (wv) acc = fmaf(cf.y, __ldg(wv + n), acc);
        }
        out[i] = e[i] * acc;
    }
};

// ---- J6: the blank / label terms (sparse in k) -------------------------------------------------------
// One WARP per (b,t) row of dF and per (b,u) row of dG.  The blank term is a warp sum; the label terms are
// one read-modify-write per distinct label: lanes holding the same label are found with a warp match, the
// lowest of them adds the group's values in lane order (deterministic, no atomics) and updates the row.
// Chunks of 32 labels are processed in order with a warp barrier between them.
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// row[key] -= sum of val over the lanes with this key (lanes with key < 0 hold nothing); whole warp calls
__device__ __forceinline__ void warp_scatter_sub(float* row, int key, float val) {
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    const int lane = threadIdx.x & 31;
    const int leader = __ffs(peers) - 1;
    float acc = 0.0f;
    // every lane walks its own peer set in lane order; shuffles are executed by the whole warp
    for (int src = 0; src < 32; ++src) {
        const float v = __shfl_sync(0xffffffffu, val, src);
        if ((peers >> src) & 1u) acc += v;
    }
    if (key >= 0 && lane == leader) row[key] -= acc;
}

// SMOOTH (DESIGN.md §9): the subtracted terms carry the factor k (c + lma on dF, c + lml on dG)
template <bool SMOOTH = false>
__global__ void __launch_bounds__(128)
joint_sparse_f_kernel(float* __restrict__ dF, const float* __restrict__ Bk, const float* __restrict__ Lb,
                      const int* __restrict__ labels, const int* __restrict__ ylen, const JointDims jd,
                      const float k) {
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;   // (b,t)
    const int lane = threadIdx.x & 31;
    if (i >= jd.N * jd.T) return;
    const int b = i / jd.T;
    const int Ub = min(max(__ldg(ylen + b) + 1, 1), jd.U);
    float* row = dF + (size_t)i * jd.V;
    const float* bk = Bk + (size_t)i * jd.U;
    const float* lb = Lb + (size_t)i * jd.U;
    float sb = 0.0f;
    for (int u = lane; u < Ub; u += 32) sb += bk[u];
    sb = warp_sum(sb);
    if (lane == 0) row[jd.blank] -= SMOOTH ? k * sb : sb;
    for (int u0 = 0; u0 < Ub - 1; u0 += 32) {
        __syncwarp();
        const int u = u0 + lane;
        const bool has = u < Ub - 1;
        warp_scatter_sub(row, has ? __ldg(labels + (size_t)b * (jd.U - 1) + u) : -1,
                         has ? (SMOOTH ? k * lb[u] : lb[u]) : 0.0f);
    }
}

template <bool SMOOTH = false>
__global__ void __launch_bounds__(128)
joint_sparse_g_kernel(float* __restrict__ dG, const float* __restrict__ Bk, const float* __restrict__ Lb,
                      const int* __restrict__ labels, const int* __restrict__ xlen,
                      const int* __restrict__ ylen, const JointDims jd, const float k) {
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;   // (b,u)
    const int lane = threadIdx.x & 31;
    if (i >= jd.N * jd.U) return;
    const int b = i / jd.U, u = i % jd.U;
    const int Tb = min(max(__ldg(xlen + b), 1), jd.T);
    const int Ub = min(max(__ldg(ylen + b) + 1, 1), jd.U);
    if (u >= Ub) return;
    float* row = dG + (size_t)i * jd.V;
    float sb = 0.0f, sl = 0.0f;
    for (int t = lane; t < Tb; t += 32) {
        const size_t c = ((size_t)b * jd.T + t) * jd.U + u;
        sb += Bk[c];
        sl += Lb[c];
    }
    sb = warp_sum(sb);
    sl = warp_sum(sl);
    if (SMOOTH) {
        sb *= k;
        sl *= k;
    }
    if (lane == 0) {
        row[jd.blank] -= sb;
        if (u < Ub - 1) row[__ldg(labels + (size_t)b * (jd.U - 1) + u)] -= sl;
    }
}

// ---- smoothing (DESIGN.md §9): the batch-wide quantities of the lm-only / am-only terms -------------------
// Every reduction has a fixed order (fixed row chunks, fixed shuffle trees, partials summed in chunk order) and
// no floating-point atomics, so a second call gives the same bits.
constexpr int kSmoothChunks = 128;   // max row chunks of a column sum
// Row chunks of a column sum over `rows` rows: at most kSmoothChunks, at least 32 rows each where there are enough,
// and none empty (chunk c covers rows [c*per, min(rows, (c+1)*per)) with per = ceil(rows / chunks)).
inline int smooth_chunks(int rows) {
    const int target = rows >= 32 * kSmoothChunks ? kSmoothChunks : rows > 32 ? (rows + 31) / 32 : 1;
    const int per = (rows + target - 1) / target;
    return (rows + per - 1) / per;
}

// part[c][v] = sum over the VALID rows q = (b, r) of chunk c of  w(q) * E[q, v],  w(q) = INV ? 1 / wr[q] : wr[q].
// Row r of utterance b is valid iff r < clamp(len[b] + add, 1, R); other rows are never read.  The sums are fp64:
// the gradient through ug takes the difference h[v] - hbar of two such sums (joint_smooth_g_kernel).
template <bool INV>
__global__ void __launch_bounds__(256)
joint_colsum_kernel(const float* __restrict__ E, const float* __restrict__ wr, const int* __restrict__ len, int add,
                    int N, int R, int V, int chunks, double* __restrict__ part) {
    const int v = blockIdx.x * 256 + threadIdx.x, c = blockIdx.y;
    const int rows = N * R, per = (rows + chunks - 1) / chunks;
    const int q0 = c * per, q1 = min(rows, q0 + per);
    double acc = 0.0;
    if (v >= V) return;
    if (q0 < q1) {   // smooth_chunks leaves no chunk empty; the guard keeps len[] in bounds regardless
        int b = q0 / R, r = q0 - b * R, lim = min(max(__ldg(len + b) + add, 1), R);
        for (int q = q0; q < q1; ++q) {
            if (r < lim) {
                const float x = __ldg(wr + q);
                acc += (double)((INV ? 1.0f / x : x) * __ldg(E + (size_t)q * V + v));
            }
            if (++r == R && q + 1 < q1) {
                r = 0;
                lim = min(max(__ldg(len + ++b) + add, 1), R);
            }
        }
    }
    part[(size_t)c * V + v] = acc;
}

// number of valid pred rows M = sum_b U_b (an integer sum: exact in any order)
__device__ __forceinline__ int valid_pred_rows(const int* __restrict__ ylen, int N, int U) {
    __shared__ int m;
    if (threadIdx.x == 0) m = 0;
    __syncthreads();
    int s = 0;
    for (int b = threadIdx.x; b < N; b += blockDim.x) s += min(max(__ldg(ylen + b) + 1, 1), U);
    atomicAdd(&m, s);
    __syncthreads();
    return m;
}

// ug[v] = (1/M) sum_{valid (b,u)} Eg[b,u,v] / sg[b,u] + FLT_MIN, lug = log ug; msum[0] = M
__global__ void __launch_bounds__(256)
joint_unigram_kernel(const double* __restrict__ part, int chunks, const int* __restrict__ ylen, int N, int U, int V,
                     float* __restrict__ ug, float* __restrict__ lug, float* __restrict__ msum) {
    const float M = (float)valid_pred_rows(ylen, N, U);
    const int v = blockIdx.x * 256 + threadIdx.x;
    if (blockIdx.x == 0 && threadIdx.x == 0) msum[0] = M;
    if (v >= V) return;
    double s = 0.0;
    for (int c = 0; c < chunks; ++c) s += part[(size_t)c * V + v];
    const float x = (float)(s / M) + FLT_MIN;
    ug[v] = x;
    lug[v] = logf(x);
}

// Row totals of the factor gradients, per frame and per label position, and the dF epilogue coefficients; one warp
// per row (fixed shuffle tree: deterministic):
//   (b,t):  O_t = sum_u (Bk + Lb),  coefF = (0, lma O_t / A),  amw = O_t / A        (zero for t >= T_b)
//   (b,u):  Bu = sum_t Bk,  Lu = sum_t Lb,  Ou = Bu + Lu                          (zero for u >= U_b)
__global__ void __launch_bounds__(256)
joint_smooth_rows_kernel(const float* __restrict__ Bk, const float* __restrict__ Lb, const float* __restrict__ A,
                         const int* __restrict__ xlen, const int* __restrict__ ylen, const JointDims jd,
                         const float lma, float2* __restrict__ coefF, float* __restrict__ amw,
                         float* __restrict__ Ou, float* __restrict__ Bu, float* __restrict__ Lu) {
    const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int NT = jd.N * jd.T;
    if (q >= NT + jd.N * jd.U) return;
    if (q < NT) {
        const int b = q / jd.T, t = q - b * jd.T;
        const int Tb = min(max(__ldg(xlen + b), 1), jd.T), Ub = min(max(__ldg(ylen + b) + 1, 1), jd.U);
        float o = 0.0f, w = 0.0f;
        if (t < Tb) {
            const size_t c0 = (size_t)q * jd.U;
            for (int u = lane; u < Ub; u += 32) o += Bk[c0 + u] + Lb[c0 + u];
            o = warp_sum(o);
            if (lma != 0.0f) w = o / __ldg(A + q);
        }
        if (lane == 0) {
            coefF[q] = make_float2(0.0f, lma * w);
            amw[q] = w;
        }
    } else {
        const int i = q - NT, b = i / jd.U, u = i - b * jd.U;
        const int Tb = min(max(__ldg(xlen + b), 1), jd.T), Ub = min(max(__ldg(ylen + b) + 1, 1), jd.U);
        float sb = 0.0f, sl = 0.0f;
        if (u < Ub) {
            for (int t = lane; t < Tb; t += 32) {
                const size_t c = ((size_t)b * jd.T + t) * jd.U + u;
                sb += Bk[c];
                sl += Lb[c];
            }
            sb = warp_sum(sb);
            sl = warp_sum(sl);
        }
        if (lane == 0) {
            Bu[i] = sb;
            Lu[i] = sl;
            Ou[i] = sb + sl;
        }
    }
}

// h[v] = lma (sum_{b,t} amw Ef[b,t,v] - Z[v] / ug[v] - K),  Z[v] = [v = blank] sum Bu + sum_{(b,u): y_u = v} Lu,
// K = sum_{b,u} (Bu + Lu).  dG only sees h[v] - hbar_u, which a constant leaves unchanged; without K every column
// that is no label would hold nearly the same large value, and fp32 would lose the small differences that matter.
// The (b,u) items pass through shared memory in tiles, every thread scans them all in the same order.
__global__ void __launch_bounds__(256)
joint_unigram_grad_kernel(const double* __restrict__ part, int chunks, const float* __restrict__ ug,
                          const float* __restrict__ Bu, const float* __restrict__ Lu, const int* __restrict__ labels,
                          const int* __restrict__ ylen, const JointDims jd, const float lma, float* __restrict__ h) {
    __shared__ int sy[256];
    __shared__ float sb[256], sl[256];
    const int v = blockIdx.x * 256 + threadIdx.x;
    const int items = jd.N * jd.U;
    double z = 0.0, K = 0.0;
    for (int i0 = 0; i0 < items; i0 += 256) {
        const int i = i0 + threadIdx.x;
        int y = -1;
        float bb = 0.0f, ll = 0.0f;
        if (i < items) {
            const int b = i / jd.U, u = i - b * jd.U;
            const int Ub = min(max(__ldg(ylen + b) + 1, 1), jd.U);
            if (u < Ub) {
                bb = Bu[i];
                if (u < Ub - 1) {
                    y = __ldg(labels + (size_t)b * (jd.U - 1) + u);
                    ll = Lu[i];
                }
            }
        }
        __syncthreads();   // the previous tile has been read
        sy[threadIdx.x] = y;
        sb[threadIdx.x] = bb;
        sl[threadIdx.x] = ll;
        __syncthreads();
        const int n = min(256, items - i0);
        if (v == jd.blank)
            for (int j = 0; j < n; ++j) z += sb[j];
        for (int j = 0; j < n; ++j) {
            K += (double)sb[j] + (double)sl[j];
            if (sy[j] == v) z += sl[j];
        }
    }
    if (v >= jd.V) return;
    double s = 0.0;
    for (int c = 0; c < chunks; ++c) s += part[(size_t)c * jd.V + v];
    h[v] = (float)(lma * (s - z / ug[v] - K));
}

// dG epilogue coefficients, one warp per (b,u):  coefG = (lml Ou / sg - hbar / (M sg), 1 / (M sg)) with
// hbar = sum_v Eg h / sg;  without h (lma = 0): (lml Ou / sg, 0).  Zero for u >= U_b (Eg not read there).
__global__ void __launch_bounds__(256)
joint_smooth_g_kernel(const float* __restrict__ eg, const float* __restrict__ sg, const float* __restrict__ h,
                      const float* __restrict__ Ou, const float* __restrict__ msum, const int* __restrict__ ylen,
                      const JointDims jd, const float lml, float2* __restrict__ coefG) {
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= jd.N * jd.U) return;
    const int b = i / jd.U, u = i - b * jd.U;
    const int Ub = min(max(__ldg(ylen + b) + 1, 1), jd.U);
    float2 cf = make_float2(0.0f, 0.0f);
    if (u < Ub) {
        const float s = __ldg(sg + i);
        cf.x = lml * Ou[i] / s;
        if (h) {
            const float* row = eg + (size_t)i * jd.V;
            double hb = 0.0;
            for (int v = lane; v < jd.V; v += 32) hb += (double)__ldg(row + v) * (double)__ldg(h + v);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) hb += __shfl_xor_sync(0xffffffffu, hb, o);
            const float inv = 1.0f / (__ldg(msum) * s);
            cf.x -= (float)(hb / s) * inv;
            cf.y = inv;
        }
    }
    if (lane == 0) coefG[i] = cf;
}

}  // namespace b200rnnt
