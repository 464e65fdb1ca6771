// rnnt_wgmma.cuh — batched fp32-accurate GEMM on Hopper's warpgroup tensor cores (wgmma.mma_async, tf32
// inputs, fp32 accumulators in registers) for the three contractions of the additive-joint RNN-T loss
// (rnnt_joint.cuh):
//
//   S [t,u]  = sum_v Ef[t,v] Eg[u,v]          M = t tile, N = u,      K = v (split over CTAs)
//   P [v,t]  = sum_u Eg[u,v] Wm[t,u]          M = v tile, N = t,      K = u      dF[t,v] = Ef[t,v] P[v,t]
//   Q [v,u]  = sum_t Ef[t,v] Wm[t,u]          M = v tile, N = u,      K = t      dG[u,v] = Eg[u,v] Q[v,u]
//
// In P and Q the VOCABULARY index is the M dimension: in the accumulator fragment the eight lanes of a
// quad column hold eight consecutive rows, so the epilogue's global accesses are 32-byte sectors.
//
// fp32 accuracy on tf32 tensor cores: every operand element x is split by the producer threads into
// hi = tf32(x) (truncated) and lo = x - hi (exact in fp32; the tensor core keeps its top 11 bits), and
// each k-step issues three MMAs into the same accumulator: hi*hi + hi*lo + lo*hi.  The dropped lo*lo
// term is 2^-20 relative; the sums feed a logarithm (S) and gradients checked to 1e-4 (P, Q).  The tensor
// core's accumulation rounds toward zero, up to an ulp per MMA in one direction: S, whose bias every lattice
// cell sees, therefore accumulates stage-wise (Stagewise below); P and Q keep one accumulator.
//
// Operands are staged global -> registers (split) -> shared memory in the canonical K-major NO-SWIZZLE
// ("interleave") layout of the wgmma matrix descriptor (tf32 operands must be K-major), in units of
// 16-byte core-matrix rows:
//   ((8,n),2):((1,SBO),LBO)     element (mn,k) at (mn%8)*16 + (mn/8)*SBO + (k/4)*LBO + (k%4)*4
// LBO is the distance between the two 16-byte k-chunks of an 8-row core matrix pair, SBO the distance
// between 8-row groups.  The chunk stride is padded (144 B instead of 128 B) so that the scalar stores
// of a warp hit 32 different banks.
//
// One CTA = 256 threads = 2 warpgroups; warpgroup w owns accumulator rows [64w, 64w + 64) of the 128-row
// M tile.  All threads produce the k-stages (one shared-memory stage buffer, the next stage's loads in
// flight in registers); each warpgroup then issues its MMAs of the stage (wgmma, asynchronous) and waits
// for them before the buffer is refilled.  gemm_kernel is the generic form (S, and dF / dG beyond 32
// label positions); grad_fused_kernel computes P and Q in one pass over Ef (see there).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>

namespace b200rnnt {
namespace wg {

// ---- PTX wrappers -------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// generic-proxy shared-memory stores -> visible to the tensor core's async proxy
__device__ __forceinline__ void fence_smem_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// warpgroup-collective: order this thread's register / shared-memory accesses before the next wgmma
__device__ __forceinline__ void mma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void mma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void mma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, tf32 inputs from shared-memory descriptors, fp32 accumulators in
// registers (thread fragment: element i is row 16*(warp%4) + lane/4 + 8*((i/2)%2), column 8*(i/4) + 2*(lane%4) + i%2).
// accumulate == 0 overwrites D.  Issued by all 128 threads of a warpgroup.
template <int N> struct Mma;
template <> struct Mma<32> {
    static __device__ __forceinline__ void run(float (&d)[16], uint64_t a, uint64_t b, int accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
            "}, %16, %17, p, 1, 1;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(a), "l"(b), "r"(accumulate)
            : "memory");
    }
};
template <> struct Mma<64> {
    static __device__ __forceinline__ void run(float (&d)[32], uint64_t a, uint64_t b, int accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
            "}, %32, %33, p, 1, 1;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(a), "l"(b), "r"(accumulate)
            : "memory");
    }
};
template <> struct Mma<128> {
    static __device__ __forceinline__ void run(float (&d)[64], uint64_t a, uint64_t b, int accumulate) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
            "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
            "}, %64, %65, p, 1, 1;\n\t}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(a), "l"(b), "r"(accumulate)
            : "memory");
    }
};

// ---- shared-memory matrix descriptor (wgmma) ------------------------------------------------------
// no swizzle: start[0,14) LBO[16,30) SBO[32,46) (all >> 4), base offset 0, layout type 0 at [62,64)
__host__ __device__ constexpr uint64_t smem_desc(uint32_t start_bytes, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((start_bytes >> 4) & 0x3fff) | ((uint64_t)((lbo_bytes >> 4) & 0x3fff) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32);
}

constexpr int kPad = 144;   // padded stride between the 16-byte k-chunks of a row group: 8 chunks (128 B) + 16 B

// Geometry of one operand tile [MN x KS] in shared memory: K-major, no swizzle.  Chunk (mn/8, k/4) holds
// 8 rows x 16 B; the k-chunks of a row group are kPad apart (LBO), row groups (KS/4)*kPad apart (SBO).
// (wgmma takes tf32 operands K-major only, so operands that are MN-contiguous in global memory are
//  transposed on their way into shared memory.)
struct TileGeom {
    static __host__ __device__ constexpr uint32_t lbo() { return kPad; }
    // row-group stride: the k-chunks of a group plus a pad that makes it 16 (mod 128) bytes, so that 16-byte
    // stores of 8 lanes to rows 4 apart in consecutive row groups (StageT4) fall on 8 different bank groups
    static __host__ __device__ constexpr uint32_t sbo(int KS) {
        return (uint32_t)(KS / 4) * kPad + (16u + 128u - ((uint32_t)(KS / 4) * kPad) % 128u) % 128u;
    }
    static __host__ __device__ constexpr uint32_t bytes(int MN, int KS) { return (uint32_t)(MN / 8) * sbo(KS); }
    static __device__ __forceinline__ uint32_t off(int mn, int k, int KS) {
        return (uint32_t)(mn & 7) * 16 + (uint32_t)(mn >> 3) * sbo(KS) + (uint32_t)(k >> 2) * kPad + (uint32_t)(k & 3) * 4;
    }
    // descriptor start offset of k-step j (8 values of k = two 16-byte chunks)
    static __host__ __device__ constexpr uint32_t kstep(int j) { return (uint32_t)(2 * j) * kPad; }
};

// element (mn, k) of batch b lives at p + b*batch + mn*s_mn + k*s_k (one of the two strides is 1);
// rows mn >= mn_valid and columns k >= the slice end read as 0
struct Operand {
    const float* p;
    long long batch;
    int s_mn, s_k;
    int mn_valid;
};

// hi = x truncated to tf32 (one LOP3; cvt.rna.tf32 is a multi-instruction sequence and the staging
// loops are issue-bound), lo = x - hi exactly; the tensor core then drops at most 2^-20 |x| from lo.
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
    hi = __uint_as_float(__float_as_uint(x) & 0xffffe000u);
    lo = x - hi;
}

// One operand's share of a k-stage, staged through registers.  init() fixes, once per CTA, this
// thread's first element (global pointer, shared-memory offset) - every further element of the thread is a
// COMPILE-TIME step away in shared memory and a constant stride away in global memory, so the stage loop
// carries no index arithmetic.  load() issues all of the thread's global loads for the stage at k0 (they
// stay in flight while the previous stage is multiplied), store() splits into hi / lo and writes the two
// shared-memory copies.
//  MODE 2 (k-contiguous, 16-byte aligned rows): float4 loads, one 16-byte chunk per store (KS in {8,16,32,64}).
//  MODE 1 (k-contiguous, unaligned rows, KS <= 32): scalar; lane = k, warp = row.
//  MODE 0 (mn-contiguous): scalar; a warp covers 8 consecutive mn x 4 consecutive k - four full 32-byte
//         sectors per load instruction, 32 different banks per store (the transposition happens here).
//  MODE 3 (mn-contiguous, 16-byte aligned rows): float4 loads of 4 consecutive mn at one k; a warp covers
//         16 mn x 8 k (eight 64-byte row pieces per load instruction); the four values go to four
//         consecutive 16-byte chunks of the K-major layout (immediate offsets), bank-conflict free at KS=24.
// Rows beyond mn_valid are neither loaded nor stored: a row of D depends on its own row of A only (and a
// column on its own row of B), and the epilogue never reads those rows/columns - so M tiles with few real
// rows (T=150: the second tile has 22) cost what their real rows cost.  The k padding IS zero-filled.
constexpr int kThreads = 256;   // 8 warps: two per accumulator lane quarter (they split the columns in the epilogue)
template <int MODE, int MN, int KS> struct StageRegs {
    static constexpr int CH = KS / 4;                 // 16-byte chunks per row
    static constexpr int RP = kThreads / (CH > 0 ? CH : 1);   // MODE 2: rows per pass
    static constexpr int MB = MN / 8;                 // MODE 0: 8-row blocks per k-group
    static constexpr int Q = MB >= 8 ? MB / 8 : 1;    // MODE 0, MB >= 8: passes over mn per k-group
    static constexpr int KB_STEP = MB >= 8 ? 1 : 8 / MB;   // MODE 0: k-groups advanced per pass (MB < 8: several at once)
    static constexpr int MT = MN / 16 > 0 ? MN / 16 : 1;   // MODE 3: 16-row tiles along mn
    static constexpr int KT = KS / 8;                     // MODE 3: 8-wide tiles along k
    static constexpr int PER = MODE == 2   ? (MN + RP - 1) / RP
                               : MODE == 1 ? MN / 8
                               : MODE == 3 ? (MT * KT + 7) / 8
                               : MB >= 8   ? Q * CH
                                           : (CH + KB_STEP - 1) / KB_STEP;
    static_assert(MODE != 3 || (MN % 16 == 0 && (MT >= 8 ? MT % 8 == 0 : 8 % MT == 0)), "MODE 3 needs MN in {16..128} or a multiple of 128");
    static_assert(MODE != 2 || (kThreads % CH == 0 && RP % 8 == 0), "MODE 2 needs KS in {8,16,32,64}");
    static_assert(MODE != 1 || KS <= 32, "MODE 1 needs KS <= 32");
    static_assert(MODE != 0 || (MB >= 8 ? MB % 8 == 0 : 8 % MB == 0), "MODE 0 needs MN in {8,16,32,64} or a multiple of 64");

    float4 v4[(MODE == 2 || MODE == 3) ? PER : 1];
    float v1[(MODE == 2 || MODE == 3) ? 1 : PER];
    const float* g0;      // this thread's element 0 at k0 = 0
    int g_mn, g_k;        // global strides (elements) along mn / k; offsets inside one batch item fit 32 bits
    uint32_t o0;          // shared-memory offset of element 0
    int mn_first, k_first, mn_lim;

    __device__ __forceinline__ void init(const Operand& op, const float* base, int mn0) {
        const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
        g_mn = op.s_mn, g_k = op.s_k;
        if (MODE == 2) {
            mn_first = tid / CH;
            k_first = 4 * (tid % CH);
        } else if (MODE == 1) {
            mn_first = w;
            k_first = lane;
        } else if (MODE == 3) {
            // warp tile = 16 mn x 8 k; tile index of pass j: w + 8j -> (mt, kt) = (ti % MT, ti / MT)
            mn_first = (MT >= 8 ? w : w % MT) * 16 + (tid & 3) * 4;
            k_first = (MT >= 8 ? 0 : w / MT) * 8 + ((tid >> 2) & 7);
        } else {
            const int mm = tid & 7, kk = (tid >> 3) & 3;
            mn_first = (MB >= 8 ? w : w % MB) * 8 + mm;
            k_first = (MB >= 8 ? 0 : w / MB) * 4 + kk;
        }
        o0 = TileGeom::off(mn_first, k_first, KS);
        g0 = base + ((mn0 + mn_first) * g_mn + k_first * g_k);
        mn_lim = op.mn_valid - mn0 - mn_first;   // element j is a real row iff its mn step < mn_lim
    }
    // (mn step, k step) of element j relative to element 0 - compile-time
    static __device__ __forceinline__ constexpr int dmn(int j) {
        return MODE == 2 ? j * RP : MODE == 1 ? 8 * j : MODE == 3 ? (MT >= 8 ? 128 * (j % (MT / 8)) : 0)
                                                      : MB >= 8   ? 64 * (j % Q)
                                                                  : 0;
    }
    static __device__ __forceinline__ constexpr int dk(int j) {
        return MODE == 2 ? 0 : MODE == 1 ? 0 : MODE == 3 ? (MT >= 8 ? 8 * (j / (MT / 8)) : 8 * (8 / MT) * j)
                                                      : MB >= 8   ? 4 * (j / Q)
                                                                  : 4 * KB_STEP * j;
    }
    __device__ __forceinline__ void load(int k0, int k_end) {
        const float* g = g0 + k0 * g_k;
        if (MODE == 2 && k0 + KS <= k_end) {
            // every stage but the last of a k range: no k raggedness - one predicated 16-byte load per row
            // (CTA-uniform branch; the general form below costs ~3x the instructions in an issue-bound loop)
#pragma unroll
            for (int j = 0; j < PER; ++j) {
                const bool in = dmn(j) < mn_lim && mn_first + dmn(j) < MN;
                v4[j] = in ? __ldg(reinterpret_cast<const float4*>(g + dmn(j) * g_mn)) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            return;
        }
#pragma unroll
        for (int j = 0; j < PER; ++j) {
            const int kj = k0 + k_first + dk(j);
            const bool in = dmn(j) < mn_lim && kj < k_end && (MODE != 1 || k_first < KS) &&
                            (MODE == 2 ? mn_first + dmn(j) < MN : k_first + dk(j) < KS);
            const float* p = g + (dmn(j) * g_mn + dk(j) * g_k);
            if (MODE == 3) {
                v4[j] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (in) {
                    if (dmn(j) + 3 < mn_lim) {
                        v4[j] = __ldg(reinterpret_cast<const float4*>(p));
                    } else {   // ragged end of the mn range
                        v4[j].x = __ldg(p);
                        if (dmn(j) + 1 < mn_lim) v4[j].y = __ldg(p + 1);
                        if (dmn(j) + 2 < mn_lim) v4[j].z = __ldg(p + 2);
                    }
                }
            } else if (MODE == 2) {
                v4[j] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (in) {
                    if (kj + 3 < k_end) {
                        v4[j] = __ldg(reinterpret_cast<const float4*>(p));
                    } else {   // ragged end of the k range
                        v4[j].x = __ldg(p);
                        if (kj + 1 < k_end) v4[j].y = __ldg(p + 1);
                        if (kj + 2 < k_end) v4[j].z = __ldg(p + 2);
                    }
                }
            } else {
                v1[j] = in ? __ldg(p) : 0.0f;
            }
        }
    }
    __device__ __forceinline__ void store(unsigned char* hi, unsigned char* lo) const {
#pragma unroll
        for (int j = 0; j < PER; ++j) {
            // offset step of element j: row groups are SBO apart, k-chunks kPad apart (compile-time)
            const uint32_t o = o0 + (uint32_t)(dmn(j) / 8) * TileGeom::sbo(KS) + (uint32_t)(dk(j) / 4) * kPad;
            // rows past mn_valid are skipped (see above); the k padding of real rows is written as zeros
            const bool slot = (MODE == 2 ? mn_first + dmn(j) < MN : k_first + dk(j) < KS) && (MODE != 1 || k_first < KS) &&
                              dmn(j) < mn_lim;
            if (slot) {
                if (MODE == 3) {
                    const float xs[4] = {v4[j].x, v4[j].y, v4[j].z, v4[j].w};
#pragma unroll
                    for (int c = 0; c < 4; ++c) {   // mn + c sits one 16-byte chunk further (same 8-row group)
                        float h, l;
                        split_tf32(xs[c], h, l);
                        *reinterpret_cast<float*>(hi + o + 16 * c) = h;
                        *reinterpret_cast<float*>(lo + o + 16 * c) = l;
                    }
                } else if (MODE == 2) {
                    float4 h, l;
                    split_tf32(v4[j].x, h.x, l.x);
                    split_tf32(v4[j].y, h.y, l.y);
                    split_tf32(v4[j].z, h.z, l.z);
                    split_tf32(v4[j].w, h.w, l.w);
                    *reinterpret_cast<float4*>(hi + o) = h;
                    *reinterpret_cast<float4*>(lo + o) = l;
                } else {
                    float h, l;
                    split_tf32(v1[j], h, l);
                    *reinterpret_cast<float*>(hi + o) = h;
                    *reinterpret_cast<float*>(lo + o) = l;
                }
            }
        }
    }
};

// MN-contiguous operand with 16-byte aligned rows, transposed IN REGISTERS: a thread fetches a 4 (k) x 4 (mn)
// block as four float4 loads (a warp: 32 adjacent blocks of one k group = four fully coalesced 512-byte row
// pieces), and writes it as four 16-byte chunks per copy (one per mn: the four k values of a K-major chunk) -
// 8 STS.128 instead of the 32 scalar stores of StageRegs MODE 3.  The hi / lo split here truncates
// (hi = x & ~0x1fff, lo = x - hi, exact): one LOP3 instead of the four-instruction cvt.rna sequence; the
// tensor core then drops at most 2^-20 of x from lo, instead of 2^-21 with rounding.
// Same interface as StageRegs.
template <int MN, int KS> struct StageT4 {
    static constexpr int MG = MN / 4, KG = KS / 4, UNITS = MG * KG;
    static constexpr int PER = (UNITS + kThreads - 1) / kThreads;
    static_assert(MN % 128 == 0 || MN == 32 || MN == 64, "a warp covers 32 adjacent blocks of one k group");
    float4 v[PER][4];
    const float* g0;
    int g_k;
    uint32_t o0;
    int mn_lim, k_first;
    bool active;
    __device__ __forceinline__ void init(const Operand& op, const float* base, int mn0) {
        const int tid = threadIdx.x;
        const int mg = tid % MG, kg = tid / MG;
        g_k = op.s_k;
        k_first = 4 * kg;
        active = tid < UNITS || PER > 1;
        o0 = TileGeom::off(4 * mg, 4 * kg, KS);
        g0 = base + (mn0 + 4 * mg + k_first * g_k);
        mn_lim = op.mn_valid - mn0 - 4 * mg;   // > 0: the block's four rows exist (mn_valid is a multiple of 4)
    }
    __device__ __forceinline__ void load(int k0, int k_end) {
#pragma unroll
        for (int p = 0; p < PER; ++p) {
            const int kk = k_first + p * 4 * (kThreads / MG);
            const float* gp = g0 + (k0 + p * 4 * (kThreads / MG)) * g_k;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const bool in = active && mn_lim > 0 && kk < KS && k0 + kk + j < k_end;
                v[p][j] = in ? __ldg(reinterpret_cast<const float4*>(gp + j * g_k)) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
    }
    static __device__ __forceinline__ void split(float x, float& hi, float& lo) {
        hi = __uint_as_float(__float_as_uint(x) & 0xffffe000u);
        lo = x - hi;
    }
    __device__ __forceinline__ void store(unsigned char* hi, unsigned char* lo) const {
#pragma unroll
        for (int p = 0; p < PER; ++p) {
            const int kk = k_first + p * 4 * (kThreads / MG);
            if (!(active && mn_lim > 0 && kk < KS)) continue;
            const uint32_t o = o0 + (uint32_t)(p * (kThreads / MG)) * kPad;
            const float xs[4][4] = {{v[p][0].x, v[p][1].x, v[p][2].x, v[p][3].x},
                                    {v[p][0].y, v[p][1].y, v[p][2].y, v[p][3].y},
                                    {v[p][0].z, v[p][1].z, v[p][2].z, v[p][3].z},
                                    {v[p][0].w, v[p][1].w, v[p][2].w, v[p][3].w}};
#pragma unroll
            for (int c = 0; c < 4; ++c) {   // row mn + c: one 16-byte chunk further inside the 8-row group
                float4 h, l;
                split(xs[c][0], h.x, l.x);
                split(xs[c][1], h.y, l.y);
                split(xs[c][2], h.z, l.z);
                split(xs[c][3], h.w, l.w);
                *reinterpret_cast<float4*>(hi + o + 16 * c) = h;
                *reinterpret_cast<float4*>(lo + o + 16 * c) = l;
            }
        }
    }
};

// What the epilogue does with accumulator element (m, n) of batch b, k slice `slice`:
//   out[slice*out_s + b*out_b + m*out_m + n*out_n] = acc * (in ? in[b*in_b + m*in_m + n*in_n] : 1)
struct Epilogue {
    const float* in;
    long long in_b;
    int in_m, in_n;      // strides inside one batch item: 32-bit
    float* out;
    long long out_s, out_b;
    int out_m, out_n;
};

// Smoothing terms of a gradient epilogue (DESIGN.md §9), for accumulator row m (vocabulary) and column n (t or u):
//   acc -> acc + coef[b*coef_b + n].x + coef[b*coef_b + n].y * w[m]      (w NULL: no last term; coef NULL: acc)
struct Smooth {
    const float2* coef;
    int coef_b;
    const float* w;
};
template <bool SMOOTH>
__device__ __forceinline__ float smooth_acc(float acc, const Smooth& sm, int b, int m, int n) {
    if (!SMOOTH || !sm.coef) return acc;
    const float2 cf = __ldg(sm.coef + (b * sm.coef_b + n));
    acc += cf.x;
    return sm.w ? fmaf(cf.y, __ldg(sm.w + m), acc) : acc;
}
// Stage-wise accumulation (gemm_kernel's trailing parameter, the S contraction): the tensor core accumulates in fp32
// rounding toward zero, so with all-positive terms every MMA into an accumulator loses up to an ulp of the running
// sum, in the same direction - 189 MMAs over K = 500 made S ~1.5e-5 too small.  Stagewise restarts the accumulator
// every k-stage, issues the stage's hi*lo and lo*hi MMAs before its hi*hi ones (while the running sum is ~2^-10 of
// the stage's, their truncations are that much smaller), and adds the stage into an fp32 register total with
// round-to-nearest: KS / 8 biased roundings per stage instead of 3 KS / 8 per stage for the whole slab.
struct Stagewise {};
template <typename... Sm> struct IsStagewise : std::false_type {};
template <> struct IsStagewise<Stagewise> : std::true_type {};

// gemm_kernel's form: the smoothing terms come as an optional trailing parameter (none: the plain epilogue)
__device__ __forceinline__ float smooth_acc_opt(float acc, int, int, int) { return acc; }
__device__ __forceinline__ float smooth_acc_opt(float acc, int b, int m, int n, const Smooth& sm) {
    return smooth_acc<true>(acc, sm, b, m, n);
}
__device__ __forceinline__ float smooth_acc_opt(float acc, int, int, int, const Stagewise&) { return acc; }

// Accumulator fragment of this thread (see Mma): row and column of element i relative to the warpgroup's tile
__device__ __forceinline__ constexpr int frag_row(int i) { return 8 * ((i >> 1) & 1); }
__device__ __forceinline__ constexpr int frag_col(int i) { return 8 * (i >> 2) + (i & 1); }

// D[128 x N] = sum_{k in slice} A[m0+m][k] * B[n0+n][k]   for batch blockIdx.z, M tile blockIdx.y, and
// blockIdx.x = k slice + slices * N tile.  A_MODE / B_MODE: how the operand is fetched (StageRegs).
// One shared-memory stage buffer per CTA: the footprint stays small, so several CTAs are resident per SM
// and cover each other's load -> split -> multiply chains; within a CTA the global loads of stage s+1 are in
// flight in registers while stage s is multiplied.  Elements with m >= A.mn_valid or n >= B.mn_valid are skipped.
// Sm: empty (the plain kernel, named gemm_kernel<A_MODE, B_MODE, N, KS>), one Smooth, whose terms the epilogue
// adds (the smoothed joint's dF / dG, DESIGN.md §9), or Stagewise (S: the accumulation above; its register total
// needs N / 2 more registers per thread, so at most 64 columns, and two CTAs per SM at 64).
template <int A_MODE, int B_MODE, int N, int KS, typename... Sm>
__global__ void __launch_bounds__(kThreads, N <= 32 || (N <= 64 && !IsStagewise<Sm...>::value) ? 3 : 2)
gemm_kernel(const Operand A, const Operand B, int K, int slices, const Epilogue epi, Sm... sm) {
    static_assert(sizeof...(Sm) <= 1, "at most one set of smoothing terms");
    constexpr bool STAGEWISE = IsStagewise<Sm...>::value;
    static_assert(!STAGEWISE || N <= 64, "the stage-wise total fits the register budget up to 64 columns");
    static_assert(N % 32 == 0 && N >= 32 && N <= 128 && KS % 8 == 0, "wgmma shape");
    constexpr uint32_t A_BYTES = TileGeom::bytes(128, KS), B_BYTES = TileGeom::bytes(N, KS);
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char* a_hi = smem;
    unsigned char* a_lo = a_hi + A_BYTES;
    unsigned char* b_hi = a_lo + A_BYTES;
    unsigned char* b_lo = b_hi + B_BYTES;

    const int b = blockIdx.z, m0 = blockIdx.y * 128, slice = blockIdx.x % slices, n0 = (blockIdx.x / slices) * N;
    const int kper = ((K + slices - 1) / slices + KS - 1) / KS * KS;
    const int kbeg = slice * kper, kend = min(K, kbeg + kper);
    const int nstages = kbeg < kend ? (kend - kbeg + KS - 1) / KS : 0;
    const int warp = threadIdx.x >> 5, group = threadIdx.x >> 7;

    StageRegs<A_MODE, 128, KS> ra;
    StageRegs<B_MODE, N, KS> rb;
    ra.init(A, A.p + (long long)b * A.batch, m0);
    rb.init(B, B.p + (long long)b * B.batch, n0);
    if (nstages > 0) {   // first stage's loads go out before anything else
        ra.load(kbeg, kend);
        rb.load(kbeg, kend);
    }
    float acc[N / 2];
    float total[STAGEWISE ? N / 2 : 1];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.0f;
#pragma unroll
    for (int i = 0; i < (STAGEWISE ? N / 2 : 1); ++i) total[i] = 0.0f;
    // this warpgroup's 64 rows of A start 8 row groups into the tile
    const uint32_t a_off = (uint32_t)group * 8 * TileGeom::sbo(KS);

    for (int s = 0; s < nstages; ++s) {
        if (s > 0) __syncthreads();   // both warpgroups' MMAs of stage s-1 have finished reading the buffer
        ra.store(a_hi, a_lo);
        rb.store(b_hi, b_lo);
        if (s + 1 < nstages) {   // next stage's loads fly during the barrier and the MMAs
            ra.load(kbeg + (s + 1) * KS, kend);
            rb.load(kbeg + (s + 1) * KS, kend);
        }
        fence_smem_async();
        __syncthreads();
        mma_fence();
#pragma unroll
        for (int j = 0; j < KS / 8; ++j) {
            const uint64_t ah = smem_desc(s32(a_hi) + a_off + TileGeom::kstep(j), TileGeom::lbo(), TileGeom::sbo(KS));
            const uint64_t al = smem_desc(s32(a_lo) + a_off + TileGeom::kstep(j), TileGeom::lbo(), TileGeom::sbo(KS));
            const uint64_t bh = smem_desc(s32(b_hi) + TileGeom::kstep(j), TileGeom::lbo(), TileGeom::sbo(KS));
            const uint64_t bl = smem_desc(s32(b_lo) + TileGeom::kstep(j), TileGeom::lbo(), TileGeom::sbo(KS));
            if (STAGEWISE) {   // the stage's small products first, the first of them overwriting the accumulator
                Mma<N>::run(acc, ah, bl, j != 0);
                Mma<N>::run(acc, al, bh, 1);
            } else {
                Mma<N>::run(acc, ah, bh, 1);
                Mma<N>::run(acc, ah, bl, 1);
                Mma<N>::run(acc, al, bh, 1);
            }
        }
        if (STAGEWISE) {
#pragma unroll
            for (int j = 0; j < KS / 8; ++j) {
                const uint64_t ah = smem_desc(s32(a_hi) + a_off + TileGeom::kstep(j), TileGeom::lbo(), TileGeom::sbo(KS));
                const uint64_t bh = smem_desc(s32(b_hi) + TileGeom::kstep(j), TileGeom::lbo(), TileGeom::sbo(KS));
                Mma<N>::run(acc, ah, bh, 1);
            }
        }
        mma_commit();
        mma_wait_all();
        if (STAGEWISE) {
#pragma unroll
            for (int i = 0; i < N / 2; ++i) total[i] += acc[i];
        }
    }

    // epilogue: element i of the fragment is (row m_base + frag_row(i), column n_base + frag_col(i))
    const int lane = threadIdx.x & 31;
    const int m_base = m0 + group * 64 + (warp & 3) * 16 + (lane >> 2);
    const int n_base = n0 + 2 * (lane & 3);
    const float* ip = epi.in ? epi.in + b * epi.in_b : nullptr;
    float* op = epi.out + slice * epi.out_s + b * epi.out_b;
#pragma unroll
    for (int i = 0; i < N / 2; ++i) {
        const int m = m_base + frag_row(i), n = n_base + frag_col(i);
        if (m < A.mn_valid && n < B.mn_valid) {
            const float x = smooth_acc_opt(STAGEWISE ? total[STAGEWISE ? i : 0] : acc[i], b, m, n, sm...);
            op[m * epi.out_m + n * epi.out_n] = ip ? x * __ldg(ip + (m * epi.in_m + n * epi.in_n)) : x;
        }
    }
}


// =================================================================================================
// Both gradient contractions of the additive joint in ONE pass over Ef (the [N,T,V] factor that dominates
// the traffic).  CTA = (utterance b, 128 vocabulary entries v0..v0+127 = the accumulator rows).  Time is
// walked in chunks of TC frames; per chunk
//
//   Q[v,u] += sum_{t in chunk} Ef[t,v] Wm[t,u]        accumulates over all chunks     (K = t)
//   P[v,t]  = sum_u            Eg[u,v] Wm[t,u]        complete after this chunk       (K = u, N = t in chunk)
//   dF[t,v] = Ef[t,v] * P[v,t]                         written per chunk
//
// and after the last chunk  dG[u,v] = Eg[u,v] * Q[v,u].  Ef is read from DRAM once (the chunk's epilogue
// re-reads the tile it has just staged - an L1/L2 hit) instead of once per contraction, and the P / Q products
// of a chunk are issued back to back.  Both accumulators live in registers (16 values each per thread);
// the next chunk's global loads are in flight while the products run.
// Shared memory: EgT (staged once), EfT / WmTU / WmUT of the current chunk, each as hi and lo tf32 copies.
// =================================================================================================
struct GradFused {
    const float *ef, *eg, *wm;   // [N,T,V], [N,U,V], [N,T,kWmPad]: Wm rows zero-padded to kWmPad label positions
    float *dF, *dG;              // [N,T,V], [N,U,V]
    int T, U, V;
    Smooth sf, sg;               // SMOOTH: the dF and dG epilogue terms
};
constexpr int kWmPad = 32;       // the weights' row pitch (16-byte aligned rows: both Wm operands are fetched as float4)
template <int NU, int TC> struct GradFusedGeom {
    static constexpr int KU = NU;   // k extent of the P product (label positions, padded)
    static constexpr uint32_t A1 = TileGeom::bytes(128, KU), A2 = TileGeom::bytes(128, TC);
    static constexpr uint32_t B1 = TileGeom::bytes(TC, KU), B2 = TileGeom::bytes(NU, TC);
    static constexpr uint32_t total = 2 * (A1 + A2 + B1 + B2);
};
template <int NU, int TC, int A_MODE, bool SMOOTH = false>   // A_MODE 3: rows of Ef / Eg 16-byte aligned (V % 4 == 0), else 0
__global__ void __launch_bounds__(kThreads, 2)
grad_fused_kernel(const GradFused g) {
    static_assert(NU == 32 && TC == 32, "instantiated shape: up to 32 label positions, 32 frames per chunk");
    using G = GradFusedGeom<NU, TC>;
    constexpr int KU = G::KU;
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char* a1_hi = smem;
    unsigned char* a1_lo = a1_hi + G::A1;
    unsigned char* a2_hi = a1_lo + G::A1;
    unsigned char* a2_lo = a2_hi + G::A2;
    unsigned char* b1_hi = a2_lo + G::A2;
    unsigned char* b1_lo = b1_hi + G::B1;
    unsigned char* b2_hi = b1_lo + G::B1;
    unsigned char* b2_lo = b2_hi + G::B2;

    const int b = blockIdx.z, v0 = blockIdx.x * 128;
    const int T = g.T, U = g.U, V = g.V;
    const int warp = threadIdx.x >> 5, group = threadIdx.x >> 7, lane = threadIdx.x & 31;
    const float* ef_b = g.ef + (long long)b * T * V;
    const float* eg_b = g.eg + (long long)b * U * V;
    const float* wm_b = g.wm + (long long)b * T * kWmPad;
    const Operand EgT{g.eg, 0, 1, V, V}, EfT{g.ef, 0, 1, V, V};
    const Operand WmTU{g.wm, 0, kWmPad, 1, T};        // (n = t, k = u): k-contiguous, aligned rows
    const Operand WmUT{g.wm, 0, 1, kWmPad, kWmPad};   // (n = u, k = t): n-contiguous, transposed in registers
    const int nchunks = (T + TC - 1) / TC;

    typename std::conditional<A_MODE == 3, StageT4<128, KU>, StageRegs<0, 128, KU>>::type r_eg;
    typename std::conditional<A_MODE == 3, StageT4<128, TC>, StageRegs<0, 128, TC>>::type r_ef;
    StageRegs<2, TC, KU> r_w1;   // one float4 per thread
    StageT4<NU, TC> r_w2;        // 64 threads, a 4x4 block each
    r_eg.init(EgT, eg_b, v0);
    r_ef.init(EfT, ef_b, v0);
    r_w2.init(WmUT, wm_b, 0);
    r_eg.load(0, U);
    r_ef.load(0, T);
    r_w1.init(WmTU, wm_b, 0);
    r_w1.load(0, kWmPad);
    r_w2.load(0, T);
    r_eg.store(a1_hi, a1_lo);

    float q[NU / 2], p[TC / 2];
#pragma unroll
    for (int i = 0; i < NU / 2; ++i) q[i] = 0.0f;
#pragma unroll
    for (int i = 0; i < TC / 2; ++i) p[i] = 0.0f;
    // this warpgroup's 64 vocabulary rows start 8 row groups into the A tiles
    const uint32_t a1_off = (uint32_t)group * 8 * TileGeom::sbo(KU), a2_off = (uint32_t)group * 8 * TileGeom::sbo(TC);
    // epilogue geometry: element i of a fragment is (vocabulary row m + frag_row(i), column c0 + frag_col(i))
    const int m = v0 + group * 64 + (warp & 3) * 16 + (lane >> 2);
    const int c0 = 2 * (lane & 3);

    for (int c = 0; c < nchunks; ++c) {
        const int t0 = c * TC;
        if (c > 0) __syncthreads();   // chunk c-1's products have finished reading the stage buffers
        r_ef.store(a2_hi, a2_lo);
        r_w1.store(b1_hi, b1_lo);
        r_w2.store(b2_hi, b2_lo);
        if (c + 1 < nchunks) {
            r_ef.load(t0 + TC, T);
            r_w1.init(WmTU, wm_b, t0 + TC);
            r_w1.load(0, kWmPad);
            r_w2.load(t0 + TC, T);
        }
        fence_smem_async();
        __syncthreads();
        mma_fence();
#pragma unroll
        for (int j = 0; j < TC / 8; ++j) {
            const uint64_t ah = smem_desc(s32(a2_hi) + a2_off + TileGeom::kstep(j), TileGeom::lbo(), TileGeom::sbo(TC));
            const uint64_t al = smem_desc(s32(a2_lo) + a2_off + TileGeom::kstep(j), TileGeom::lbo(), TileGeom::sbo(TC));
            const uint64_t bh = smem_desc(s32(b2_hi) + TileGeom::kstep(j), TileGeom::lbo(), TileGeom::sbo(TC));
            const uint64_t bl = smem_desc(s32(b2_lo) + TileGeom::kstep(j), TileGeom::lbo(), TileGeom::sbo(TC));
            Mma<NU>::run(q, ah, bh, 1);
            Mma<NU>::run(q, ah, bl, 1);
            Mma<NU>::run(q, al, bh, 1);
        }
#pragma unroll
        for (int j = 0; j < KU / 8; ++j) {
            const uint64_t ah = smem_desc(s32(a1_hi) + a1_off + TileGeom::kstep(j), TileGeom::lbo(), TileGeom::sbo(KU));
            const uint64_t al = smem_desc(s32(a1_lo) + a1_off + TileGeom::kstep(j), TileGeom::lbo(), TileGeom::sbo(KU));
            const uint64_t bh = smem_desc(s32(b1_hi) + TileGeom::kstep(j), TileGeom::lbo(), TileGeom::sbo(KU));
            const uint64_t bl = smem_desc(s32(b1_lo) + TileGeom::kstep(j), TileGeom::lbo(), TileGeom::sbo(KU));
            Mma<TC>::run(p, ah, bh, j != 0);
            Mma<TC>::run(p, ah, bl, 1);
            Mma<TC>::run(p, al, bh, 1);
        }
        mma_commit();
        mma_wait_all();
        // dF of this chunk: dF[t,v] = Ef[t,v] * P[v,t]
        const float* ip = ef_b + (t0 * V);
        float* op = g.dF + (long long)b * T * V + (t0 * V);
#pragma unroll
        for (int i = 0; i < TC / 2; ++i) {
            const int v = m + frag_row(i), t = c0 + frag_col(i);
            if (v < V && t0 + t < T) op[t * V + v] = smooth_acc<SMOOTH>(p[i], g.sf, b, v, t0 + t) * __ldg(ip + (t * V + v));
        }
    }
    // dG: Q is complete.  dG[u,v] = Eg[u,v] * Q[v,u]
    const float* ip = eg_b;
    float* op = g.dG + (long long)b * U * V;
#pragma unroll
    for (int i = 0; i < NU / 2; ++i) {
        const int v = m + frag_row(i), u = c0 + frag_col(i);
        if (v < V && u < U) op[u * V + v] = smooth_acc<SMOOTH>(q[i], g.sg, b, v, u) * __ldg(ip + (u * V + v));
    }
}

template <int N, int KS>
constexpr size_t gemm_smem_bytes() {   // one stage buffer with hi and lo copies of both operand tiles
    return 2 * (size_t)TileGeom::bytes(128, KS) + 2 * (size_t)TileGeom::bytes(N, KS);
}

}  // namespace wg
}  // namespace b200rnnt
