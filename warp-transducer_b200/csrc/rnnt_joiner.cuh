// Fused joiner (DESIGN.md §14): logits[b,t,u,:] = W act(enc[b,t] + pred[b,u]) + bias on bf16 tensor cores, reduced
// to the lattice factors px / py (forward) and back from dpx / dpy to the four parameter gradients (backward),
// without the [N,T,U,V] logits.  The work runs over chunks of the padded cell grid, cells enumerated (b, u, t) with
// t fastest; a chunk of m cells is m scratch rows.  Every contraction is a 64x64 output tile per CTA, 4 warps of
// 32x32, mma.sync.m16n8k16 bf16 with fp32 accumulators, operands staged through 64x64 swizzled shared-memory tiles
// by cp.async (zero-filled past the operand's extent) and read with ldmatrix (.trans for MN-major operands).
// The pruned joiner (DESIGN.md §15) runs the same kernels with PRUNED = true over the rows (b, r, t), t fastest, of
// the windows: row (b, r, t) is cell (t, ranges[b,t] + r), and px / py are written at the cell's dense index.
// Dropout on h (DESIGN.md §16) is the DROP = true form of the two kernels that touch h element-wise, the h and ds
// kernels: the keep bit of element (b, t, u, k) is a pure function of the seed and (dense cell index, k), so the
// backward regenerates it and nothing is stored.
#pragma once
#include <cuda_bf16.h>
#include <curand_philox4x32_x.h>
#include <math.h>
#include <stdint.h>

namespace b200joiner {

typedef __nv_bfloat16 bf16;

constexpr int TILE = 64;               // rows, columns and k of every shared-memory tile
constexpr int TILE_ELEMS = TILE * TILE;
constexpr int THREADS = 128;           // 4 warps, 2 x 2 over a 64 x 64 output tile
constexpr int STAGES = 4;              // cp.async depth of the logits kernels' W stream
constexpr int PAIR_STAGES = 3;         // and of the ds and dW kernels, which stream both operands
constexpr int STAGE_TILES = 4;         // k tiles (4 x 4 = 16 MMAs per accumulator) between fp32 RN totals
enum { ACT_TANH = 0, ACT_RELU = 1 };

// The padded cell grid, the chunk, and what the epilogues need to know about a cell.
struct Geo {
    int N, T, U, S, H, V, Hp, Vp;    // S = U - 1; Hp, Vp: row strides of the h and dlogits scratch
    int c0, m;                        // first cell of the chunk and its cell count
    int blank;
    const int* xlen;                  // T_b, clamped to [1, T] as the lattice clamps it
    const int* ylen;                  // S_b, clamped to [0, S]
    const int* labels;                // [N, S]
};

// The pruned window: rows (b, r, t) with r < R stand for cells (t, ranges[b,t] + r).  Dense calls pass {nullptr, 0}
// and never read it.
struct Window {
    const int* ranges;   // [N, T]
    int R;
};

// Dropout on h: element k of the cell with dense index c is dropped iff word k & 3 of
// Philox4x32-10(ctr = (k >> 2, c, 0, 0), key = (lo32(seed), hi32(seed))) is below thr; kept elements are scaled.
// Calls without dropout pass {nullptr, 0, 1} and never read it.
struct Drop {
    const unsigned long long* seed;   // device pointer, read once per thread by the DROP kernels
    uint32_t thr;                     // floor(p 2^32)
    float scale;                      // 1 / (1 - p)
};

__device__ __forceinline__ uint2 drop_key(const Drop& d) {
    const unsigned long long s = __ldg(d.seed);
    return make_uint2((uint32_t)s, (uint32_t)(s >> 32));
}

// The four Philox words of columns 4 q .. 4 q + 3 of dense cell c.
__device__ __forceinline__ uint4 drop_words(uint2 key, int q, int c) {
    return curand_Philox4x32_10(make_uint4((uint32_t)q, (uint32_t)c, 0u, 0u), key);
}

struct Cell {
    int b, u, t;
    bool valid;       // t < T_b and 0 <= u <= S_b: the cell has a blank factor
    bool has_label;   // t < T_b and 0 <= u < S_b: it also has a label factor
    int dense;        // (b * U + u) * T + t, the cell's py index (px: (b * S + u) * T + t); meaningful when valid.
                      // The row's lse index is its grid index c0 + r (dense: the same).
};

__device__ __forceinline__ int clampi(int x, int lo, int hi) { return x < lo ? lo : (x > hi ? hi : x); }

// Row r of the chunk.  Dense: grid index (b, u, t).  PRUNED: grid index (b, r', t), u = ranges[b,t] + r' formed in
// 64 bits, so any int32 window start is well defined; rows whose u falls outside [0, S_b] are padding.
template <bool PRUNED = false>
__device__ __forceinline__ Cell decode(const Geo& g, int r, const Window& w = Window{nullptr, 0}) {
    Cell k{0, 0, 0, false, false, 0};
    if (r >= g.m) return k;
    const int c = g.c0 + r;
    k.t = c % g.T;
    const int bu = c / g.T;
    if constexpr (!PRUNED) {
        k.u = bu % g.U;
        k.b = bu / g.U;
        const int Tb = clampi(g.xlen[k.b], 1, g.T), Sb = clampi(g.ylen[k.b], 0, g.S);
        k.valid = k.t < Tb && k.u <= Sb;
        k.has_label = k.t < Tb && k.u < Sb;
        k.dense = c;
    } else {
        k.b = bu / w.R;
        const long long u = (long long)w.ranges[(size_t)k.b * g.T + k.t] + bu % w.R;
        const int Tb = clampi(g.xlen[k.b], 1, g.T), Sb = clampi(g.ylen[k.b], 0, g.S);
        k.valid = k.t < Tb && u >= 0 && u <= Sb;
        k.has_label = k.valid && u < Sb;
        k.u = k.valid ? (int)u : 0;
        k.dense = (k.b * g.U + k.u) * g.T + k.t;
    }
    return k;
}

__device__ __forceinline__ float bf2f(bf16 x) { return __bfloat162float(x); }

// Element offset of (row, col) in a 64 x 64 bf16 tile: 16-byte groups XOR-swizzled by row, so the eight rows an
// ldmatrix phase reads fall in eight different bank groups.
__device__ __forceinline__ int swz(int row, int col) {
    return row * TILE + ((((col >> 3) ^ row) & 7) << 3) + (col & 7);
}

__device__ __forceinline__ uint32_t smem_addr(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void cp16(void* dst, const void* src, bool pred) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_addr(dst)), "l"(src),
                 "r"(pred ? 16 : 0));
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// Rows r0.. and columns k0.. of a row-major bf16 matrix (leading dimension ld) into a tile, by NT threads.  A row is
// read where row < rows and a 16-byte group where its first column < cols (cols is a multiple of 8); the rest is 0.
template <int NT = THREADS>
__device__ __forceinline__ void load_tile(bf16* tile, const bf16* src, int ld, int r0, int rows, int k0, int cols) {
#pragma unroll
    for (int i = threadIdx.x; i < TILE_ELEMS / 8; i += NT) {
        const int row = i >> 3, grp = i & 7;
        const int gr = r0 + row, gk = k0 + grp * 8;
        const bool ok = gr < rows && gk < cols;
        cp16(tile + swz(row, grp * 8), ok ? src + (size_t)gr * ld + gk : src, ok);
    }
}

__device__ __forceinline__ void ldm4(uint32_t (&r)[4], const bf16* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_addr(p)));
}
__device__ __forceinline__ void ldm4t(uint32_t (&r)[4], const bf16* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_addr(p)));
}

__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
        "{%0,%1,%2,%3};\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

typedef float Acc[2][4][4];   // a warp's 32 x 32: [m16 tile][n8 tile][mma C fragment]

__device__ __forceinline__ void zero(Acc& a) {
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) a[i][j][e] = 0.f;
}

// tot += acc (fp32 round-to-nearest), acc = 0: the tensor core's accumulation error is bounded per stage.
__device__ __forceinline__ void fold(Acc& tot, Acc& acc) {
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                tot[i][j][e] += acc[i][j][e];
                acc[i][j][e] = 0.f;
            }
}

// acc += A B over the 64 k of one tile pair, for this warp's rows wm*32.. and columns wn*32...
// A_KMAJOR: the A tile's stored rows are k (columns m), else m (columns k).
// B_KMAJOR: the B tile's stored rows are k (columns n), else n (columns k).
template <bool A_KMAJOR, bool B_KMAJOR>
__device__ __forceinline__ void mma_tile(Acc& acc, const bf16* As, const bf16* Bs, int wm, int wn, int lane) {
    const int j = lane >> 3, r = lane & 7;
#pragma unroll
    for (int ks = 0; ks < TILE / 16; ++ks) {
        uint32_t a[2][4], b[2][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            const int m0 = wm * 32 + mt * 16;
            if (A_KMAJOR)
                ldm4t(a[mt], As + swz(ks * 16 + r + (j >> 1) * 8, m0 + (j & 1) * 8));
            else
                ldm4(a[mt], As + swz(m0 + (lane & 15), ks * 16 + (lane >> 4) * 8));
        }
#pragma unroll
        for (int np = 0; np < 2; ++np) {
            const int n0 = wn * 32 + np * 16;
            if (B_KMAJOR)
                ldm4t(b[np], Bs + swz(ks * 16 + r + (j & 1) * 8, n0 + (j >> 1) * 8));
            else
                ldm4(b[np], Bs + swz(n0 + r + (j >> 1) * 8, ks * 16 + (j & 1) * 8));
        }
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
                mma_bf16(acc[mt][nt], a[mt], b[nt >> 1][(nt & 1) * 2], b[nt >> 1][(nt & 1) * 2 + 1]);
    }
}

// Per-row metadata of an R-row tile of the chunk, in shared memory.
template <int R, bool PRUNED>
struct RowPy {
    int pyi[R];     // py index (b, u, t) of a valid pruned row
};
template <int R>
struct RowPy<R, false> {};   // a dense row's py index is its cell index

template <int R = TILE, bool PRUNED = false>
struct RowInfo : RowPy<R, PRUNED> {
    int flag[R];    // bit 0 valid, bit 1 has_label
    int label[R];   // labels[b, u] where has_label (compared with columns, never used as an address)
    int cell[R];    // the row's grid index: its lse index, and (dense) its py index (b, u, t)
    int pxi[R];     // px index (b, u, t) where u < S (PRUNED: where has_label), else -1

    __device__ __forceinline__ int py(int i) const {
        if constexpr (PRUNED) return this->pyi[i];
        else return cell[i];
    }
};

// Fills ri for rows r0 .. r0 + R - 1; returns whether any of them is a valid cell.
template <int R, bool PRUNED>
__device__ __forceinline__ int load_rows(const Geo& g, const Window& w, int r0, RowInfo<R, PRUNED>& ri, int* any) {
    if (threadIdx.x == 0) *any = 0;
    __syncthreads();
    if (threadIdx.x < R) {
        const int i = threadIdx.x;
        const Cell k = decode<PRUNED>(g, r0 + i, w);
        ri.flag[i] = (k.valid ? 1 : 0) | (k.has_label ? 2 : 0);
        ri.label[i] = k.has_label ? g.labels[(size_t)k.b * g.S + k.u] : 0;
        ri.cell[i] = g.c0 + r0 + i;
        if constexpr (PRUNED) {
            ri.pxi[i] = k.has_label ? (k.b * g.S + k.u) * g.T + k.t : -1;
            ri.pyi[i] = k.dense;
        } else {
            ri.pxi[i] = (r0 + i < g.m && k.u < g.S) ? (k.b * g.S + k.u) * g.T + k.t : -1;
        }
        if (k.valid) *any = 1;
    }
    __syncthreads();
    return *any;
}

// h[r, :] = round_bf16(act(enc[b,t] + pred[b,u])) for a valid cell, 0 for padding and rows past the chunk; column H
// is 1 (the dW contraction then yields dbias as its column H), columns H+1 .. Hp-1 are 0.  Padded rows of enc and
// pred are never read.  DROP: columns k < H of a valid cell hold h~ = keep ? round_bf16(h scale) : 0 (two Philox
// calls per 8 columns); column H is never dropped.
template <bool PRUNED, bool DROP = false>
__global__ void __launch_bounds__(256) joiner_h_kernel(Geo g, int act, const bf16* __restrict__ enc,
                                                       const bf16* __restrict__ pred, bf16* __restrict__ h,
                                                       int rows, Window w, Drop d = Drop{nullptr, 0u, 1.f}) {
    const int groups = g.Hp / 8;
    uint2 key = make_uint2(0u, 0u);
    if constexpr (DROP) key = drop_key(d);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (long long)rows * groups;
         i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / groups), k0 = (int)(i % groups) * 8;
    __align__(16) bf16 out[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) out[e] = __float2bfloat16_rn(0.f);
    if (k0 < g.H) {
        const Cell k = decode<PRUNED>(g, r, w);
        if (k.valid) {
            const uint4 ev = *reinterpret_cast<const uint4*>(enc + ((size_t)k.b * g.T + k.t) * g.H + k0);
            const uint4 pv = *reinterpret_cast<const uint4*>(pred + ((size_t)k.b * g.U + k.u) * g.H + k0);
            const bf16* ep = reinterpret_cast<const bf16*>(&ev);
            const bf16* pp = reinterpret_cast<const bf16*>(&pv);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float s = bf2f(ep[e]) + bf2f(pp[e]);
                const float a = act == ACT_TANH ? tanhf(s) : ((s > 0.f || s != s) ? s : 0.f);
                out[e] = __float2bfloat16_rn(a);
            }
            if constexpr (DROP) {
                const uint4 x0 = drop_words(key, k0 >> 2, k.dense), x1 = drop_words(key, (k0 >> 2) + 1, k.dense);
                const uint32_t x[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
#pragma unroll
                for (int e = 0; e < 8; ++e)
                    out[e] = x[e] < d.thr ? __float2bfloat16_rn(0.f) : __float2bfloat16_rn(bf2f(out[e]) * d.scale);
            }
        }
    } else if (k0 == g.H) {
        out[0] = __float2bfloat16_rn(1.f);
    }
    *reinterpret_cast<uint4*>(h + (size_t)r * g.Hp + k0) = *reinterpret_cast<const uint4*>(out);
    }
}

// The logits GEMM of one BM-row tile of h (BM = 64 or 128, BM / 32 x 2 warps) against every column of W,
// row-stationary: the tile's h rows stay in shared memory, W streams through in 64 x 64 tiles, each shared by all the
// rows.  BWD = false: online max / sum over the columns, the blank and label logits captured, then lse, px and py.
// BWD = true: dlogits from the forward's lse and the incoming dpx, dpy.  PRUNED: px / py are written (and dpx / dpy
// read) at valid rows only; the caller filled px / py with -inf beforehand.
template <bool BWD, int BM, bool PRUNED>
__device__ __forceinline__ void logits_tile(const Geo& g, const bf16* __restrict__ h, const bf16* __restrict__ W,
                                            const bf16* __restrict__ bias, float* __restrict__ lse,
                                            float* __restrict__ px, float* __restrict__ py,
                                            const float* __restrict__ dpx, const float* __restrict__ dpy,
                                            bf16* __restrict__ dlog, const Window& w) {
    constexpr int NT = BM * 2, RT = BM / TILE;   // threads; 64-row h tiles per k block
    extern __shared__ __align__(128) unsigned char smem_raw[];   // BM h rows, then STAGES W tiles
    __shared__ RowInfo<BM, PRUNED> ri;
    __shared__ int any;
    __shared__ float rv0[BM], rv1[BM], rv2[BM];   // fwd: blank, label logit; bwd: lse, dpx, dpy
    __shared__ float red_m[2][BM], red_s[2][BM];
    const int r0 = blockIdx.x * BM;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 1, wn = warp & 1;
    const int gq = lane >> 2, cq = lane & 3;
    const float NINF = -INFINITY;

    const bool live = load_rows<BM, PRUNED>(g, w, r0, ri, &any);
    if (tid < BM) {
        const int f = ri.flag[tid];
        if (!BWD) {
            rv0[tid] = NAN;
            rv1[tid] = NAN;
        } else {
            rv0[tid] = (f & 1) ? lse[ri.cell[tid]] : 0.f;
            rv1[tid] = (f & 2) ? dpx[ri.pxi[tid]] : 0.f;
            rv2[tid] = (f & 1) ? dpy[ri.py(tid)] : 0.f;
        }
    }
    if (!live) {   // every row padding: -inf factors, or zero dlogits
        if (!BWD) {
            if (tid < BM && r0 + tid < g.m) {
                if (!PRUNED) {
                    py[ri.cell[tid]] = NINF;
                    if (ri.pxi[tid] >= 0) px[ri.pxi[tid]] = NINF;
                }
                lse[ri.cell[tid]] = 0.f;
            }
        } else {
            const __nv_bfloat162 z = __floats2bfloat162_rn(0.f, 0.f);
            for (int i = tid; i < BM * g.Vp / 2; i += NT)
                reinterpret_cast<__nv_bfloat162*>(dlog + (size_t)r0 * g.Vp)[i] = z;
        }
        return;
    }

    const int KB = (g.H + TILE - 1) / TILE;
    bf16* As = reinterpret_cast<bf16*>(smem_raw);
    bf16* Bs = As + KB * RT * TILE_ELEMS;
    for (int kb = 0; kb < KB; ++kb)
        for (int rt = 0; rt < RT; ++rt)
            load_tile<NT>(As + (kb * RT + rt) * TILE_ELEMS, h, g.Hp, r0 + rt * TILE, 1 << 30, kb * TILE, g.H);
    cp_commit();
    const int total = (g.Vp / TILE) * KB;
#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < total) load_tile<NT>(Bs + s * TILE_ELEMS, W, g.H, (s / KB) * TILE, g.V, (s % KB) * TILE, g.H);
        cp_commit();
    }

    Acc acc;
    zero(acc);
    float run_m[4], run_s[4];   // rows (mt, half): wm*32 + mt*16 + half*8 + gq
#pragma unroll
    for (int i = 0; i < 4; ++i) run_m[i] = NINF, run_s[i] = 0.f;

    for (int it = 0; it < total; ++it) {
        cp_wait<STAGES - 2>();
        __syncthreads();
        const int nx = it + STAGES - 1;
        if (nx < total)
            load_tile<NT>(Bs + (nx % STAGES) * TILE_ELEMS, W, g.H, (nx / KB) * TILE, g.V, (nx % KB) * TILE, g.H);
        cp_commit();
        const int kb = it % KB;
        mma_tile<false, false>(acc, As + (kb * RT + (wm >> 1)) * TILE_ELEMS, Bs + (it % STAGES) * TILE_ELEMS, wm & 1,
                               wn, lane);
        if (kb != KB - 1) continue;

        const int v0 = (it / KB) * TILE;
        float bcol[4][2];   // bias of this thread's 8 columns
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int col = v0 + wn * 32 + nt * 8 + 2 * cq + e;
                bcol[nt][e] = (bias && col < g.V) ? bf2f(bias[col]) : 0.f;
            }
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int row = wm * 32 + mt * 16 + half * 8 + gq;
                const int f = ri.flag[row], lab = ri.label[row];
                if (!BWD) {
                    float tmax = NINF;
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = v0 + wn * 32 + nt * 8 + 2 * cq + e;
                            float x = acc[mt][nt][half * 2 + e];
                            if (col < g.V) {
                                x += bcol[nt][e];
                                tmax = fmaxf(tmax, x);
                                if (col == g.blank) rv0[row] = x;
                                if ((f & 2) && col == lab) rv1[row] = x;
                            }
                            acc[mt][nt][half * 2 + e] = x;
                        }
                    const int i = mt * 2 + half;
                    const float mnew = fmaxf(run_m[i], tmax);
                    if (mnew != NINF) {
                        float s = run_s[i] * expf(run_m[i] - mnew);
#pragma unroll
                        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                            for (int e = 0; e < 2; ++e)
                                if (v0 + wn * 32 + nt * 8 + 2 * cq + e < g.V)
                                    s += expf(acc[mt][nt][half * 2 + e] - mnew);
                        run_m[i] = mnew;
                        run_s[i] = s;
                    }
                } else {
                    const float L = rv0[row], dx = rv1[row], dy = rv2[row], gs = dx + dy;
                    bf16* out = dlog + (size_t)(r0 + row) * g.Vp;
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt) {
                        const int col = v0 + wn * 32 + nt * 8 + 2 * cq;
                        float d[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int c = col + e;
                            d[e] = 0.f;
                            if ((f & 1) && c < g.V) {
                                const float x = acc[mt][nt][half * 2 + e] + bcol[nt][e];
                                d[e] = -gs * expf(x - L) + (c == g.blank ? dy : 0.f) +
                                       ((f & 2) && c == lab ? dx : 0.f);
                            }
                        }
                        *reinterpret_cast<__nv_bfloat162*>(out + col) = __floats2bfloat162_rn(d[0], d[1]);
                    }
                }
            }
        zero(acc);
    }

    if constexpr (!BWD) {
        // (max, sum) across the quad's lanes, then across the two column warps
#pragma unroll
        for (int i = 0; i < 4; ++i) {
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1) {
                const float m2 = __shfl_xor_sync(0xffffffffu, run_m[i], o);
                const float s2 = __shfl_xor_sync(0xffffffffu, run_s[i], o);
                const float m = fmaxf(run_m[i], m2);
                run_s[i] = m == NINF ? 0.f : run_s[i] * expf(run_m[i] - m) + s2 * expf(m2 - m);
                run_m[i] = m;
            }
            if (cq == 0) {
                const int row = wm * 32 + (i >> 1) * 16 + (i & 1) * 8 + gq;
                red_m[wn][row] = run_m[i];
                red_s[wn][row] = run_s[i];
            }
        }
        __syncthreads();
        if (tid < BM && r0 + tid < g.m) {
            const int f = ri.flag[tid];
            const int c = ri.cell[tid], p = ri.pxi[tid];
            if (f & 1) {
                const float m0 = red_m[0][tid], m1 = red_m[1][tid], m = fmaxf(m0, m1);
                const float s = red_s[0][tid] * expf(m0 - m) + red_s[1][tid] * expf(m1 - m);
                const float L = m + logf(s);
                lse[c] = L;
                py[ri.py(tid)] = rv0[tid] - L;
                if (p >= 0) px[p] = (f & 2) ? rv1[tid] - L : NINF;
            } else {
                lse[c] = 0.f;
                if (!PRUNED) {
                    py[c] = NINF;
                    if (p >= 0) px[p] = NINF;
                }
            }
        }
    }
}

template <int BM, bool PRUNED>
__global__ void __launch_bounds__(BM * 2) joiner_lse_kernel(Geo g, const bf16* __restrict__ h,
                                                            const bf16* __restrict__ W,
                                                            const bf16* __restrict__ bias, float* __restrict__ lse,
                                                            float* __restrict__ px, float* __restrict__ py,
                                                            Window w) {
    logits_tile<false, BM, PRUNED>(g, h, W, bias, lse, px, py, nullptr, nullptr, nullptr, w);
}

template <int BM, bool PRUNED>
__global__ void __launch_bounds__(BM * 2) joiner_dlogits_kernel(Geo g, const bf16* __restrict__ h,
                                                                 const bf16* __restrict__ W,
                                                                 const bf16* __restrict__ bias,
                                                                 const float* __restrict__ lse,
                                                                 const float* __restrict__ dpx,
                                                                 const float* __restrict__ dpy,
                                                                 bf16* __restrict__ dlog, Window w) {
    logits_tile<true, BM, PRUNED>(g, h, W, bias, const_cast<float*>(lse), nullptr, nullptr, dpx, dpy, dlog, w);
}

// ds[r, n] = (dlogits[r, :] W[:, n]) act'(h[r, n]) for a 64 x 64 tile (rows r, hidden units n); W is MN-major here.
// Tiles whose rows are all padding write nothing: the reduction reads valid rows only.
// DROP: ds[r, n] = (dlogits W)[r, n] m scale act'(s), with the keep bit m regenerated from the row's dense cell index
// and n.  The scratch holds h~, not h: tanh recomputes h from the row's enc and pred elements exactly as the h kernel
// forms it; relu takes m [s > 0] as [h~ > 0] (scale > 0, and a positive s rounds to a positive bf16 h).
template <bool PRUNED, bool DROP = false>
__global__ void __launch_bounds__(THREADS) joiner_ds_kernel(Geo g, int act, const bf16* __restrict__ dlog,
                                                            const bf16* __restrict__ W,
                                                            const bf16* __restrict__ h, float* __restrict__ ds,
                                                            Window w, Drop d = Drop{nullptr, 0u, 1.f},
                                                            const bf16* __restrict__ enc = nullptr,
                                                            const bf16* __restrict__ pred = nullptr) {
    extern __shared__ __align__(128) unsigned char smem_raw[];   // PAIR_STAGES A tiles, then as many B tiles
    bf16* sm = reinterpret_cast<bf16*>(smem_raw);
    __shared__ RowInfo<TILE, PRUNED> ri;
    __shared__ int any;
    const int r0 = blockIdx.x * TILE, n0 = blockIdx.y * TILE;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 1, wn = warp & 1;
    if (!load_rows<TILE, PRUNED>(g, w, r0, ri, &any)) return;
    bf16* As = sm;
    bf16* Bs = sm + PAIR_STAGES * TILE_ELEMS;
    const int total = g.Vp / TILE;
#pragma unroll
    for (int s = 0; s < PAIR_STAGES - 1; ++s) {
        if (s < total) {
            load_tile(As + s * TILE_ELEMS, dlog, g.Vp, r0, 1 << 30, s * TILE, g.Vp);
            load_tile(Bs + s * TILE_ELEMS, W + n0, g.H, s * TILE, g.V, 0, g.H - n0);
        }
        cp_commit();
    }
    Acc acc, tot;
    zero(acc);
    zero(tot);
    for (int it = 0; it < total; ++it) {
        cp_wait<PAIR_STAGES - 2>();
        __syncthreads();
        const int nx = it + PAIR_STAGES - 1;
        if (nx < total) {
            load_tile(As + (nx % PAIR_STAGES) * TILE_ELEMS, dlog, g.Vp, r0, 1 << 30, nx * TILE, g.Vp);
            load_tile(Bs + (nx % PAIR_STAGES) * TILE_ELEMS, W + n0, g.H, nx * TILE, g.V, 0, g.H - n0);
        }
        cp_commit();
        const int st = (it % PAIR_STAGES) * TILE_ELEMS;
        mma_tile<false, true>(acc, As + st, Bs + st, wm, wn, lane);
        if ((it + 1) % STAGE_TILES == 0 || it + 1 == total) fold(tot, acc);
    }
    const int gq = lane >> 2, cq = lane & 3;
    if constexpr (DROP) {
        const uint2 key = drop_key(d);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int row = wm * 32 + mt * 16 + half * 8 + gq;
                if (!(ri.flag[row] & 1)) continue;
                const size_t r = (size_t)(r0 + row);
                const int c = ri.py(row), t = c % g.T, bu = c / g.T;   // the dense cell (b, u, t)
                const bf16* er = enc + ((size_t)(bu / g.U) * g.T + t) * g.H;
                const bf16* pr = pred + (size_t)bu * g.H;
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    const int n = n0 + wn * 32 + nt * 8 + 2 * cq;
                    if (n >= g.H) continue;
                    const uint4 x = drop_words(key, n >> 2, c);   // n is even: words n & 3 and n & 3 + 1
                    const float m0 = ((n & 2) ? x.z : x.x) < d.thr ? 0.f : d.scale;
                    const float m1 = ((n & 2) ? x.w : x.y) < d.thr ? 0.f : d.scale;
                    float d0, d1;
                    if (act == ACT_TANH) {
                        const __nv_bfloat162 ev = *reinterpret_cast<const __nv_bfloat162*>(er + n);
                        const __nv_bfloat162 pv = *reinterpret_cast<const __nv_bfloat162*>(pr + n);
                        const float h0 = bf2f(__float2bfloat16_rn(tanhf(__low2float(ev) + __low2float(pv))));
                        const float h1 = bf2f(__float2bfloat16_rn(tanhf(__high2float(ev) + __high2float(pv))));
                        d0 = (1.f - h0 * h0) * m0;
                        d1 = (1.f - h1 * h1) * m1;
                    } else {
                        const __nv_bfloat162 hv = *reinterpret_cast<const __nv_bfloat162*>(h + r * g.Hp + n);
                        d0 = __low2float(hv) > 0.f ? d.scale : 0.f;
                        d1 = __high2float(hv) > 0.f ? d.scale : 0.f;
                    }
                    *reinterpret_cast<float2*>(ds + r * g.H + n) =
                        make_float2(tot[mt][nt][half * 2] * d0, tot[mt][nt][half * 2 + 1] * d1);
                }
            }
    } else {
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int row = wm * 32 + mt * 16 + half * 8 + gq;
                if (!(ri.flag[row] & 1)) continue;
                const size_t r = (size_t)(r0 + row);
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    const int n = n0 + wn * 32 + nt * 8 + 2 * cq;
                    if (n >= g.H) continue;
                    const __nv_bfloat162 hv = *reinterpret_cast<const __nv_bfloat162*>(h + r * g.Hp + n);
                    const float h0 = __low2float(hv), h1 = __high2float(hv);
                    const float d0 = act == ACT_TANH ? 1.f - h0 * h0 : (h0 > 0.f ? 1.f : 0.f);
                    const float d1 = act == ACT_TANH ? 1.f - h1 * h1 : (h1 > 0.f ? 1.f : 0.f);
                    *reinterpret_cast<float2*>(ds + r * g.H + n) =
                        make_float2(tot[mt][nt][half * 2] * d0, tot[mt][nt][half * 2 + 1] * d1);
                }
            }
    }
}

// denc[b, t] += sum over the chunk's valid cells (b, u, t) of ds, in u order; dpred[b, u] += the same over t, in t
// order.  One thread per output element: deterministic, no atomics.  PRUNED: denc[b, t] sums the chunk's valid rows
// (b, r, t) in r order; dpred[b, u] sums, in t order over the chunk's frames of b, the valid row r = u - ranges[b,t]
// where 0 <= r < R.
template <bool PRUNED>
__global__ void __launch_bounds__(256) joiner_reduce_kernel(Geo g, const float* __restrict__ ds,
                                                            float* __restrict__ denc, float* __restrict__ dpred,
                                                            Window w) {
    if constexpr (PRUNED) {
        const int RT = w.R * g.T;                                              // rows per utterance
        const int b_lo = g.c0 / RT, b_hi = (g.c0 + g.m - 1) / RT;
        const long long n_pred = (long long)(b_hi - b_lo + 1) * g.U * g.H;
        const long long n_enc = (long long)(b_hi - b_lo + 1) * g.T * g.H;
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_pred + n_enc;
             i += (long long)gridDim.x * blockDim.x) {
            const bool is_pred = i < n_pred;
            const long long j = is_pred ? i : i - n_pred;
            const int k = (int)(j % g.H), q = (int)(j / g.H);
            const int b = b_lo + (is_pred ? q / g.U : q / g.T);
            const int Tb = clampi(g.xlen[b], 1, g.T), Sb = clampi(g.ylen[b], 0, g.S);
            const int* rb = w.ranges + (size_t)b * g.T;
            const int lo = max(g.c0 - b * RT, 0), hi = min(g.c0 + g.m - b * RT, RT);   // b's rows in the chunk
            float s = 0.f;
            bool hit = false;
            if (is_pred) {
                const int u = q % g.U;
                if (u > Sb) continue;
                int t_lo = 0, t_hi = Tb;   // the chunk's frames of b, when its rows of b do not wrap a frame
                if (hi - lo < g.T && lo % g.T <= (hi - 1) % g.T) t_lo = lo % g.T, t_hi = min((hi - 1) % g.T + 1, Tb);
                for (int t = t_lo; t < t_hi; ++t) {
                    const long long r = (long long)u - rb[t];
                    if (r < 0 || r >= w.R) continue;
                    const int row = (int)r * g.T + t;
                    if (row < lo || row >= hi) continue;
                    s += ds[(size_t)(b * RT + row - g.c0) * g.H + k];
                    hit = true;
                }
                if (hit) dpred[((size_t)b * g.U + u) * g.H + k] += s;
            } else {
                const int t = q % g.T;
                if (t >= Tb) continue;
                for (int r = 0; r < w.R; ++r) {
                    const long long u = (long long)rb[t] + r;
                    const int row = r * g.T + t;
                    if (u < 0 || u > Sb || row < lo || row >= hi) continue;
                    s += ds[(size_t)(b * RT + row - g.c0) * g.H + k];
                    hit = true;
                }
                if (hit) denc[((size_t)b * g.T + t) * g.H + k] += s;
            }
        }
        return;
    }
    const int bu_lo = g.c0 / g.T, bu_hi = (g.c0 + g.m - 1) / g.T;        // (b, u) rows the chunk touches
    const int b_lo = bu_lo / g.U, b_hi = bu_hi / g.U;
    const long long n_pred = (long long)(bu_hi - bu_lo + 1) * g.H;
    const long long n_enc = (long long)(b_hi - b_lo + 1) * g.T * g.H;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_pred + n_enc;
         i += (long long)gridDim.x * blockDim.x) {
        if (i < n_pred) {
            const int bu = bu_lo + (int)(i / g.H), k = (int)(i % g.H);
            const int b = bu / g.U, u = bu % g.U;
            const int Tb = clampi(g.xlen[b], 1, g.T), Sb = clampi(g.ylen[b], 0, g.S);
            if (u > Sb) continue;
            const int t_lo = max(g.c0 - bu * g.T, 0), t_hi = min(g.c0 + g.m - bu * g.T, Tb);
            if (t_lo >= t_hi) continue;
            float s = 0.f;
            for (int t = t_lo; t < t_hi; ++t) s += ds[(size_t)(bu * g.T + t - g.c0) * g.H + k];
            dpred[(size_t)bu * g.H + k] += s;
        } else {
            const long long j = i - n_pred;
            const int k = (int)(j % g.H);
            const int bt = (int)(j / g.H), b = b_lo + bt / g.T, t = bt % g.T;
            const int Tb = clampi(g.xlen[b], 1, g.T), Sb = clampi(g.ylen[b], 0, g.S);
            if (t >= Tb) continue;
            const int base = b * g.U * g.T + t;   // cell (b, u, t) = base + u T
            const int u_lo = g.c0 > base ? (g.c0 - base + g.T - 1) / g.T : 0;
            const int last = g.c0 + g.m - 1 - base;
            if (last < 0) continue;
            const int u_hi = min(last / g.T, Sb);
            if (u_lo > u_hi) continue;
            float s = 0.f;
            for (int u = u_lo; u <= u_hi; ++u) s += ds[(size_t)(base + u * g.T - g.c0) * g.H + k];
            denc[((size_t)b * g.T + t) * g.H + k] += s;
        }
    }
}

// acc[z][v][n] += sum over the rows of slab z of dlogits[r, v] h[r, n] for a 64 x 64 tile (v, n): dW, and dbias as
// column H.  Both operands are MN-major.  Each CTA owns its output tile: deterministic, no atomics.
__global__ void __launch_bounds__(THREADS) joiner_dw_kernel(Geo g, const bf16* __restrict__ dlog,
                                                            const bf16* __restrict__ h, float* __restrict__ acc_dw,
                                                            int row_tiles, int tiles_per_slab) {
    extern __shared__ __align__(128) unsigned char smem_raw[];   // PAIR_STAGES A tiles, then as many B tiles
    bf16* sm = reinterpret_cast<bf16*>(smem_raw);
    const int v0 = blockIdx.x * TILE, n0 = blockIdx.y * TILE, z = blockIdx.z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 1, wn = warp & 1;
    const int kt0 = z * tiles_per_slab, total = min(row_tiles - kt0, tiles_per_slab);
    if (total <= 0) return;
    bf16* As = sm;
    bf16* Bs = sm + PAIR_STAGES * TILE_ELEMS;
#pragma unroll
    for (int s = 0; s < PAIR_STAGES - 1; ++s) {
        if (s < total) {
            load_tile(As + s * TILE_ELEMS, dlog, g.Vp, (kt0 + s) * TILE, 1 << 30, v0, g.Vp);
            load_tile(Bs + s * TILE_ELEMS, h, g.Hp, (kt0 + s) * TILE, 1 << 30, n0, g.Hp);
        }
        cp_commit();
    }
    Acc acc, tot;
    zero(acc);
    zero(tot);
    for (int it = 0; it < total; ++it) {
        cp_wait<PAIR_STAGES - 2>();
        __syncthreads();
        const int nx = it + PAIR_STAGES - 1;
        if (nx < total) {
            load_tile(As + (nx % PAIR_STAGES) * TILE_ELEMS, dlog, g.Vp, (kt0 + nx) * TILE, 1 << 30, v0, g.Vp);
            load_tile(Bs + (nx % PAIR_STAGES) * TILE_ELEMS, h, g.Hp, (kt0 + nx) * TILE, 1 << 30, n0, g.Hp);
        }
        cp_commit();
        const int st = (it % PAIR_STAGES) * TILE_ELEMS;
        mma_tile<true, true>(acc, As + st, Bs + st, wm, wn, lane);
        if ((it + 1) % STAGE_TILES == 0 || it + 1 == total) fold(tot, acc);
    }
    const int gq = lane >> 2, cq = lane & 3;
    float* out = acc_dw + (size_t)z * g.Vp * g.Hp;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const size_t v = v0 + wm * 32 + mt * 16 + half * 8 + gq;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                float2* p = reinterpret_cast<float2*>(out + v * g.Hp + n0 + wn * 32 + nt * 8 + 2 * cq);
                float2 o = *p;
                o.x += tot[mt][nt][half * 2];
                o.y += tot[mt][nt][half * 2 + 1];
                *p = o;
            }
        }
}

// The fp32 accumulators rounded once to bf16: dW and dbias summed over the slabs in slab order, denc and dpred.
__global__ void __launch_bounds__(256) joiner_round_kernel(Geo g, int slabs, const float* __restrict__ acc_dw,
                                                           const float* __restrict__ denc,
                                                           const float* __restrict__ dpred, bf16* __restrict__ gw,
                                                           bf16* __restrict__ gb, bf16* __restrict__ ge,
                                                           bf16* __restrict__ gp) {
    const long long nw = (long long)g.V * g.H, nb = g.V, ne = (long long)g.N * g.T * g.H,
                    np = (long long)g.N * g.U * g.H;
    const size_t slab = (size_t)g.Vp * g.Hp;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nw + nb + ne + np;
         i += (long long)gridDim.x * blockDim.x) {
        if (i < nw + nb) {
            const bool w = i < nw;
            const size_t v = w ? i / g.H : i - nw, n = w ? i % g.H : g.H;
            float s = 0.f;
            for (int z = 0; z < slabs; ++z) s += acc_dw[z * slab + v * g.Hp + n];
            if (w)
                gw[i] = __float2bfloat16_rn(s);
            else if (gb)
                gb[v] = __float2bfloat16_rn(s);
        } else if (i < nw + nb + ne) {
            ge[i - nw - nb] = __float2bfloat16_rn(denc[i - nw - nb]);
        } else {
            gp[i - nw - nb - ne] = __float2bfloat16_rn(dpred[i - nw - nb - ne]);
        }
    }
}

// px and py of a pruned forward set to -inf before the chunk loop writes the valid rows' cells.
__global__ void __launch_bounds__(256) joiner_fill_kernel(float* __restrict__ px, long long npx,
                                                          float* __restrict__ py, long long npy) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npx + npy;
         i += (long long)gridDim.x * blockDim.x) {
        if (i < npx)
            px[i] = -INFINITY;
        else
            py[i - npx] = -INFINITY;
    }
}

}  // namespace b200joiner
