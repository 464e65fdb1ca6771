// rnnt_common.cuh — small device/host helpers shared by the sm_90a RNN-T kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace b200rnnt {

constexpr int kWarp = 32;

// ---------------------------------------------------------------------------------------------
// Division by a runtime constant without the ~30-instruction 32-bit divide: q = umulhi(n, mul) >> shr.
// Exact for 0 <= n < 2^31 (the cell index space; the entry point rejects larger lattices).
// ---------------------------------------------------------------------------------------------
struct FastDiv {
    uint32_t d, mul, shr;
    __host__ __device__ FastDiv() : d(1), mul(0), shr(0) {}
    explicit FastDiv(uint32_t div) : d(div) {
        if (div <= 1) {
            mul = 0;
            shr = 0;
        } else {
            uint32_t lg = 0;
            while ((1ull << lg) < div) ++lg;
            const uint32_t p = 31 + lg;
            mul = (uint32_t)(((1ull << p) + div - 1) / div);
            shr = p - 32;
        }
    }
    __device__ __forceinline__ uint32_t div(uint32_t n) const {
        return d == 1 ? n : (__umulhi(n, mul) >> shr);
    }
    __device__ __forceinline__ void divmod(uint32_t n, uint32_t& q, uint32_t& r) const {
        q = div(n);
        r = n - q * d;
    }
};

// ---------------------------------------------------------------------------------------------
// Element-type traits: vector-of-2 storage used for the per-cell (rowmax, logsumexp) and
// (blank, label) log-prob pairs, plus the math the kernels need in each precision.
// ---------------------------------------------------------------------------------------------
template <typename T> struct Real;
template <> struct Real<float> {
    using pair = float2;
    static __device__ __forceinline__ float neg_inf() { return -INFINITY; }
    // e^x via the MUFU ex2 unit: one FMUL + MUFU.EX2, rel. error ~2^-22 (fine against the 1e-4 budget)
    static __device__ __forceinline__ float exp(float x) {
        float y;
        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x * 1.4426950408889634f));
        return y;
    }
    // 2^x directly (caller pre-multiplied by log2 e)
    static __device__ __forceinline__ float exp2(float x) {
        float y;
        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
        return y;
    }
    static __device__ __forceinline__ float log(float x) { return logf(x); }
    static __device__ __forceinline__ float max(float a, float b) { return fmaxf(a, b); }  // one FMNMX
    static constexpr float kLog2e = 1.4426950408889634f;
};
template <> struct Real<double> {
    using pair = double2;
    static __device__ __forceinline__ double neg_inf() { return -(double)INFINITY; }
    static __device__ __forceinline__ double exp(double x) { return ::exp(x); }
    static __device__ __forceinline__ double exp2(double x) { return ::exp2(x); }
    static __device__ __forceinline__ double log(double x) { return ::log(x); }
    static __device__ __forceinline__ double max(double a, double b) { return fmax(a, b); }
    static constexpr double kLog2e = 1.4426950408889634;
};

// ---------------------------------------------------------------------------------------------
// sum_k exp(x_k - M) for a known row maximum M, and the log of the sum.
// float: one FFMA + MUFU.EX2 per element, 2^(x*log2e - fl(M*log2e)); the rounding of the product
// M*log2e is recovered exactly with one FMA per row (comp) and folded into the logarithm, so the
// result equals the (x - M) form to fp32 rounding even for |M| ~ 1e3.  double: plain exp/log.
// ---------------------------------------------------------------------------------------------
template <typename T> struct ExpSum;
template <> struct ExpSum<float> {
    float negML, comp;
    __device__ __forceinline__ explicit ExpSum(float M) {
        const float ML = M * Real<float>::kLog2e;
        negML = -ML;
        comp = fmaf(M, Real<float>::kLog2e, negML);  // M*log2e - fl(M*log2e), exact
    }
    __device__ __forceinline__ float term(float x) const {
        return Real<float>::exp2(fmaf(x, Real<float>::kLog2e, negML));
    }
    __device__ __forceinline__ float log_of(float S) const {
        float l;
        asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(S));
        return (l - comp) * 0.6931471805599453f;
    }
};
template <> struct ExpSum<double> {
    double M;
    __device__ __forceinline__ explicit ExpSum(double m) : M(m) {}
    __device__ __forceinline__ double term(double x) const { return ::exp(x - M); }
    __device__ __forceinline__ double log_of(double S) const { return ::log(S); }
};

// ---------------------------------------------------------------------------------------------
// Vectorised global access with cache policy.  BYTES in {4, 8, 16}.
//   ld_keep   : read-only path, normal L2 residency (first pass over the logits: on shapes that fit
//               the 50 MB L2 the second pass then hits)
//   ld_stream : evict-first (second/last pass over the logits)
//   st_stream : evict-first store (gradients are never re-read by this library)
// ---------------------------------------------------------------------------------------------
template <int BYTES> struct Pack;
template <> struct Pack<2> { using type = unsigned short; };
template <> struct Pack<4> { using type = int; };
template <> struct Pack<8> { using type = int2; };
template <> struct Pack<16> { using type = int4; };

template <typename T, int VEC> struct alignas(sizeof(T) * VEC) VecT {
    T v[VEC];
};

// Storage (IO) type -> arithmetic type.  float/double compute in themselves; the 16-bit storage
// types (bf16 / fp16 logits and gradients, SURVEY.md 8(f).3) compute in float.
template <typename IO> struct ComputeOf { using type = IO; };
template <> struct ComputeOf<__nv_bfloat16> { using type = float; };
template <> struct ComputeOf<__half> { using type = float; };

template <typename T, typename IO> __device__ __forceinline__ T to_compute(IO v) { return (T)v; }
template <> __device__ __forceinline__ float to_compute<float, __nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_compute<float, __half>(__half v) { return __half2float(v); }
template <typename IO, typename T> __device__ __forceinline__ IO from_compute(T v) { return (IO)v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_compute<__nv_bfloat16, float>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_compute<__half, float>(float v) { return __float2half_rn(v); }

// VEC storage elements -> VEC arithmetic values (identity when IO == T)
template <typename T, int VEC, typename IO, typename P>
__device__ __forceinline__ VecT<T, VEC> unpack(P raw) {
    union {
        P raw;
        VecT<IO, VEC> val;
    } x;
    x.raw = raw;
    VecT<T, VEC> out;
#pragma unroll
    for (int c = 0; c < VEC; ++c) out.v[c] = to_compute<T, IO>(x.val.v[c]);
    return out;
}

template <typename T, int VEC, typename IO> __device__ __forceinline__ VecT<T, VEC> ld_keep(const IO* p) {
    using P = typename Pack<sizeof(IO) * VEC>::type;
    return unpack<T, VEC, IO, P>(__ldg(reinterpret_cast<const P*>(p)));
}
template <typename T, int VEC, typename IO> __device__ __forceinline__ VecT<T, VEC> ld_stream(const IO* p) {
    using P = typename Pack<sizeof(IO) * VEC>::type;
    return unpack<T, VEC, IO, P>(__ldcs(reinterpret_cast<const P*>(p)));
}
template <typename T, int VEC, typename IO>
__device__ __forceinline__ void st_stream(IO* p, const VecT<T, VEC>& v) {
    using P = typename Pack<sizeof(IO) * VEC>::type;
    union {
        P raw;
        VecT<IO, VEC> val;
    } x;
#pragma unroll
    for (int c = 0; c < VEC; ++c) x.val.v[c] = from_compute<IO, T>(v.v[c]);
    __stcs(reinterpret_cast<P*>(p), x.raw);
}
// one element through the read-only path
template <typename T, typename IO> __device__ __forceinline__ T ld_scalar(const IO* p) {
    using P = typename Pack<sizeof(IO)>::type;
    union {
        P raw;
        IO val;
    } x;
    x.raw = __ldg(reinterpret_cast<const P*>(p));
    return to_compute<T, IO>(x.val);
}

// ---------------------------------------------------------------------------------------------
// 16-bit storage, two elements per 32-bit word: maximum on the packed word (HMNMX2 - one instruction
// per two elements, no conversion) and conversion of a word to two floats (bf16: a shift and a mask).
// ---------------------------------------------------------------------------------------------
template <typename IO> struct Packed16;
template <> struct Packed16<__nv_bfloat16> {
    static constexpr unsigned kNegInf2 = 0xFF80FF80u;
    static __device__ __forceinline__ unsigned max2(unsigned a, unsigned b) {
        union { unsigned u; __nv_bfloat162 h; } x, y, z;
        x.u = a, y.u = b;
        z.h = __hmax2(x.h, y.h);
        return z.u;
    }
    static __device__ __forceinline__ void to_floats(unsigned w, float& lo, float& hi) {
        lo = __uint_as_float(w << 16);
        hi = __uint_as_float(w & 0xffff0000u);
    }
};
template <> struct Packed16<__half> {
    static constexpr unsigned kNegInf2 = 0xFC00FC00u;
    static __device__ __forceinline__ unsigned max2(unsigned a, unsigned b) {
        union { unsigned u; __half2 h; } x, y, z;
        x.u = a, y.u = b;
        z.h = __hmax2(x.h, y.h);
        return z.u;
    }
    static __device__ __forceinline__ void to_floats(unsigned w, float& lo, float& hi) {
        union { unsigned u; __half2 h; } x;
        x.u = w;
        const float2 f = __half22float2(x.h);
        lo = f.x, hi = f.y;
    }
};

// ---------------------------------------------------------------------------------------------
// Reductions over an aligned group of LPR lanes (LPR a power of two <= 32) by xor-shuffle.
// Every lane of the warp must call these (full mask).
// ---------------------------------------------------------------------------------------------
template <int LPR, typename T> __device__ __forceinline__ T group_max(T v) {
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) {
        T w = __shfl_xor_sync(0xffffffffu, v, o);
        v = Real<T>::max(v, w);
    }
    return v;
}
template <int LPR, typename T> __device__ __forceinline__ T group_sum(T v) {
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// same with the group's lanes `stride` apart (stride 1: adjacent lanes, as above)
template <int LPR, typename T> __device__ __forceinline__ T group_max_strided(T v, int stride) {
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) {
        T w = __shfl_xor_sync(0xffffffffu, v, o * stride);
        v = Real<T>::max(v, w);
    }
    return v;
}
template <int LPR, typename T> __device__ __forceinline__ T group_sum_strided(T v, int stride) {
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o * stride);
    return v;
}

// ---------------------------------------------------------------------------------------------
// Lattice-space log-sum-exp.  The running alpha/beta values are kept in double (they reach
// |x| ~ 1e3..1e4 on the README shapes, where an fp32 ulp is 1e-4..1e-3 and would dominate the
// gradient error); only the bounded correction term log(1 + e^-d) in (0, ln 2] is evaluated
// in the caller's precision: two MUFU ops on the dependent chain for float.
// Same -inf short-circuits as the reference (include/detail/rnnt_helper.h:16-24).
// ---------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ double lse_step(double a, double b) {
    const double mx = fmax(a, b), mn = fmin(a, b);
    if (mx == -(double)INFINITY) return mx;
    if (sizeof(T) == 4) {
        const float d = (float)(mn - mx);  // <= 0, -inf allowed (-> correction 0)
        const float e = Real<float>::exp(d);
        return mx + (double)(__logf(1.0f + e));
    } else {
        return mx + log1p(::exp(mn - mx));
    }
}

// ---------------------------------------------------------------------------------------------
// fp32 lattice storage (rnnt_lattice.cuh): values v * 2^e, transition factors m * 2^k.
// ---------------------------------------------------------------------------------------------
constexpr int kEZero = -(1 << 29);        // exponent of "log zero"
constexpr int kEDead = -(1 << 28);        // anything below this is reported as -inf
constexpr float kMinLog2 = -65536.0f;     // transition log2-probabilities are clamped here (2^-65536 == 0)

// log2 of a lattice value = e + l
struct __align__(8) LogVal {
    int e;
    float l;
};
__device__ __forceinline__ float logval_log2(const LogVal a) { return (float)a.e + a.l; }

// (m, k) with m * 2^k = e^lp, by round-to-nearest of lp*log2(e) with the 1.5*2^23 trick: FMA/ALU
// pipes only.  NaN becomes m = NaN (the lattice kernel turns it into a NaN cost).
__device__ __forceinline__ void split_prob(float lp, float& m, int& k) {
    const float y = lp * 1.4426950408889634f;
    const float yc = fmaxf(y, kMinLog2);
    const float yk = yc + 12582912.0f;
    k = __float_as_int(yk) - 0x4B400000;
    const float f = yc - (yk - 12582912.0f);   // in [-0.5, 0.5]
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(m) : "f"(f));
    if (!(y > kMinLog2)) m = 1.0f, k = kEZero;   // probability zero (lp = -inf included)
    if (lp != lp) m = lp;
}
// lattice factors of one cell: {m_blank, k_blank, m_label, k_label}; no label (u = U-1) -> log zero
__device__ __forceinline__ float4 make_fac(float lp_blank, float lp_label, bool has_label) {
    float mb, ml = 1.0f;
    int kb, kl = kEZero;
    split_prob(lp_blank, mb, kb);
    if (has_label) split_prob(lp_label, ml, kl);
    return make_float4(mb, __int_as_float(kb), ml, __int_as_float(kl));
}
// natural-log probabilities back from the factors (additive-joint weights kernel)
__device__ __forceinline__ float fac_logp(float m, float kbits) {
    float l;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(m));
    return ((float)__float_as_int(kbits) + l) * 0.6931471805599453f;
}

__device__ __forceinline__ LogVal to_logval(float v, int e) {
    LogVal a;
    a.e = e;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(a.l) : "f"(v));
    return a;
}


// Programmatic dependent launch (PDL).  pdl_trigger(): this CTA no longer holds back the launch of the
// next kernel in the stream; pdl_wait(): everything the previous kernel wrote is complete and visible.
// Both are no-ops for a kernel launched without the programmatic-serialization attribute.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Per-type lattice storage: what pass 1 writes per cell (`fac`) and what the wavefront stores (`val`).
//   float : fac = {m_blank, k_blank, m_label, k_label} (16 B), val = LogVal {e, log2 v}
//   double: fac = (lp_blank, lp_label) natural logs (16 B),    val = double natural log
template <typename T> struct Lat;
template <> struct Lat<float> {
    using fac = float4;
    using val = LogVal;
    static __device__ __forceinline__ fac make(float lp_blank, float lp_label, bool has_label) {
        return make_fac(lp_blank, lp_label, has_label);
    }
};
template <> struct Lat<double> {
    using fac = double2;
    using val = double;
    static __device__ __forceinline__ fac make(double lp_blank, double lp_label, bool has_label) {
        return make_double2(lp_blank, has_label ? lp_label : 0.0);
    }
};

}  // namespace b200rnnt
