// rnnt_lattice_io.cuh — the RNN-T loss, gradient and forced alignment on factors the caller computed
// (DESIGN.md §13; k2's mutual_information_recursion).
//
//   lattice_import_kernel  px [N,S,T] / py [N,S+1,T] (k2's orientation: label-major, t contiguous) -> the
//                          workspace's factor array at skew(d, b, t, u), exactly what pass 1 writes for a dense call.
//                          The wavefronts (rnnt_lattice.cuh, lattice_kernel) and the Viterbi kernels then run unchanged.
//   lattice_grad_kernel    the transition occupancies from the factors and the lattices the wavefront left:
//                          d cost / d py[b,u,t] = -e_blank(t,u),  d cost / d px[b,u,t] = -e_label(t,u),
//                          times the per-utterance scale, in the storage type.
//
// Three layouts meet here: the caller's arrays run along t, the factors along anti-diagonals (diagonal-major), the
// fp32 lattices along u (cell-major).  Both kernels work on 32 x 32 tiles of one utterance's cells (256 threads) and
// turn the tile in shared memory, so that every global access of a warp is one contiguous run: the caller's rows of
// 32 frames, the factors of one anti-diagonal of the tile (adjacent in the diagonal-major array), the lattice values
// of one frame.  (At C4's lattice, 64 x 1500 x 301 cells, one thread per cell with strided factor and lattice
// accesses took 0.94 ms to import and 1.00 ms for the gradient, each more than the wavefront: DESIGN.md §13.)
#pragma once
#include "rnnt_kernels.cuh"

namespace b200rnnt {

constexpr int kIoTile = 32;

// Tile blockIdx.x of the grid N x ceil(maxU / 32) x ceil(maxT / 32), t fastest: utterance b, first frame t0, first
// label column u0.
struct IoTile {
    uint32_t b, t0, u0;
};
__device__ __forceinline__ IoTile io_tile(const Dims& d) {
    const uint32_t tiles_t = (d.maxT + kIoTile - 1) / kIoTile, tiles_u = (d.maxU + kIoTile - 1) / kIoTile;
    const uint32_t bu = blockIdx.x / tiles_t;
    return IoTile{bu / tiles_u, (blockIdx.x - bu * tiles_t) * kIoTile, (bu % tiles_u) * kIoTile};
}
// Index of tile cell (t0 + i, u0 + j) in the factor array: base + (i + j) * maxU + j, so the cells of the tile's
// anti-diagonal k = i + j are adjacent.
__device__ __forceinline__ size_t io_tile_skew(const Dims& d, const IoTile& c) {
    return skew(d, c.b, c.t0, c.u0);
}

// A +inf factor becomes NaN: the fp32 split of +inf is already NaN, and fp64 must report the same NaN cost rather than
// a cost of -inf.
template <typename T> __device__ __forceinline__ T finite_or_nan(T x) {
    return x == (T)INFINITY ? (T)NAN : x;
}

// Every cell of the tensor is written (padding included) with has_label = u < U_b - 1, as pass 1 does: cells outside
// an utterance are never read by the wavefronts, and a label factor only exists where a label transition does.
// Shared memory: tile[j][i] = cell (t0 + i, u0 + j); read back along anti-diagonals, 16-byte words j*31 + k apart,
// so a quarter-warp's eight loads hit eight different bank groups.
template <typename IO>
__global__ void __launch_bounds__(256)
lattice_import_kernel(const IO* __restrict__ px, const IO* __restrict__ py, const int* __restrict__ xlen,
                      const int* __restrict__ ylen, typename Lat<typename ComputeOf<IO>::type>::fac* __restrict__ lp2,
                      const Dims d) {
    using T = typename ComputeOf<IO>::type;
    __shared__ typename Lat<T>::fac tile[kIoTile][kIoTile];
    const IoTile c = io_tile(d);
    int Tb, Ub;
    utt_extent(d, xlen, ylen, c.b, Tb, Ub);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t t = c.t0 + lane;
    for (int j = warp; j < kIoTile; j += 8) {   // one label row of 32 frames per warp
        const uint32_t u = c.u0 + j;
        if (u < (uint32_t)d.maxU && t < (uint32_t)d.maxT) {
            const bool has_label = (int)u < Ub - 1;
            const T lpb = finite_or_nan(ld_scalar<T>(py + ((size_t)c.b * d.maxU + u) * d.maxT + t));
            T lpl = T(0);
            if (has_label) lpl = finite_or_nan(ld_scalar<T>(px + ((size_t)c.b * (d.maxU - 1) + u) * d.maxT + t));
            tile[j][lane] = Lat<T>::make(lpb, lpl, has_label);
        }
    }
    __syncthreads();
    const size_t base = io_tile_skew(d, c);
    for (int k = warp; k < 2 * kIoTile - 1; k += 8) {   // one anti-diagonal per warp, lane j = column u0 + j
        const int i = k - lane;
        if (i >= 0 && i < kIoTile && c.u0 + lane < (uint32_t)d.maxU && c.t0 + i < (uint32_t)d.maxT)
            lp2[base + (size_t)k * d.maxU + lane] = tile[lane][i];
    }
}

// Blank and label occupancies of cell (t, u) of a live utterance (t < T_b, u < U_b) with factors fc; zero where the
// transition does not exist.  Regular: the label leads to (t, u+1); the blank of the last frame only exists at
// u = U_b - 1.  MOD (DESIGN.md §11): the label leads to (t+1, u+1); on the last frame only u = U_b - 2 has one, into
// the virtual beta(T_b, U_b - 1) = log 1.
// fp32: lattices LogVal {e, log2 v} cell-major; every exponent in the exp2 domain, exact integer part + small float
// part (the form joint_weights uses).
template <bool MOD>
__device__ __forceinline__ void lattice_occ(const float4 fc, const LogVal* __restrict__ alphas,
                                            const LogVal* __restrict__ betas, const LogVal ll, const Dims& d,
                                            uint32_t b, uint32_t t, uint32_t u, int Tb, int Ub, float& eb, float& ey) {
    const size_t q = cell(d, b, t, u);
    const LogVal a = alphas[q];
    const int oe = a.e - ll.e;
    const float ol = a.l - ll.l;
    eb = 0.0f;
    ey = 0.0f;
    const float lpb2 = (float)__float_as_int(fc.y) + log2f(fc.x);
    if ((int)t < Tb - 1) {
        const LogVal bn = betas[q + d.maxU];
        eb = exp2f((float)(oe + bn.e) + (ol + bn.l) + lpb2);
    } else if ((int)u == Ub - 1) {
        eb = exp2f((float)oe + ol + lpb2);
    }
    if ((int)u < Ub - 1 && (!MOD || (int)t < Tb - 1 || (int)u == Ub - 2)) {
        const bool term = MOD && (int)t == Tb - 1;
        const LogVal bn = term ? LogVal{0, 0.0f} : betas[q + (MOD ? d.maxU + 1 : 1)];
        const float lpl2 = (float)__float_as_int(fc.w) + log2f(fc.z);
        ey = exp2f((float)(oe + bn.e) + (ol + bn.l) + lpl2);
    }
}
// fp64: natural-log lattices, diagonal-major: (t+1,u) at q + maxU, (t,u+1) at q + maxU + 1, (t+1,u+1) at q + 2 maxU + 1
template <bool MOD>
__device__ __forceinline__ void lattice_occ(const double2 fc, const double* __restrict__ alphas,
                                            const double* __restrict__ betas, const double ll, const Dims& d,
                                            uint32_t b, uint32_t t, uint32_t u, int Tb, int Ub, double& eb,
                                            double& ey) {
    const size_t q = skew(d, b, t, u);
    const double occ = alphas[q] - ll;
    eb = 0.0;
    ey = 0.0;
    if ((int)t < Tb - 1)
        eb = ::exp(occ + betas[q + d.maxU] + fc.x);
    else if ((int)u == Ub - 1)
        eb = ::exp(occ + fc.x);
    if ((int)u < Ub - 1 && (!MOD || (int)t < Tb - 1 || (int)u == Ub - 2)) {
        const bool term = MOD && (int)t == Tb - 1;
        const double bn = term ? 0.0 : betas[q + (MOD ? 2 * d.maxU + 1 : d.maxU + 1)];
        ey = ::exp(occ + bn + fc.y);
    }
}

// py_grad[b,u,t] = -scale_b e_blank(t,u) and, for u < maxU - 1, px_grad[b,u,t] = -scale_b e_label(t,u), with
// scale_b = scale_in * scale_vec[b] (scale_vec may be NULL).  Zero on padding and for an utterance without a path.
// Per tile: the factors in along anti-diagonals, the occupancies one frame per warp (lanes along u: the fp32
// lattices' rows), the gradients out one label row per warp (lanes along t).  fac rows are padded to 34 words: the
// anti-diagonal stores are conflict-free and the per-frame loads two-way.
template <typename IO, typename T, bool MOD>
__global__ void __launch_bounds__(256)
lattice_grad_kernel(const typename Lat<T>::fac* __restrict__ lp2, const typename Lat<T>::val* __restrict__ alphas,
                    const typename Lat<T>::val* __restrict__ betas, const typename Lat<T>::val* __restrict__ llf,
                    const int* __restrict__ xlen, const int* __restrict__ ylen, IO* __restrict__ px_grad,
                    IO* __restrict__ py_grad, const T scale_in, const T* __restrict__ scale_vec, const Dims d) {
    __shared__ typename Lat<T>::fac fac[kIoTile][kIoTile + 2];   // [u - u0][t - t0]
    __shared__ T gb[kIoTile][kIoTile + 1], gy[kIoTile][kIoTile + 1];
    const IoTile c = io_tile(d);
    int Tb, Ub;
    utt_extent(d, xlen, ylen, c.b, Tb, Ub);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool live = !ll_dead(llf, c.b);
    const size_t base = io_tile_skew(d, c);
    for (int k = warp; k < 2 * kIoTile - 1; k += 8) {
        const int i = k - lane;
        if (i >= 0 && i < kIoTile && (int)(c.u0 + lane) < Ub && (int)(c.t0 + i) < Tb)
            fac[lane][i] = lp2[base + (size_t)k * d.maxU + lane];
    }
    __syncthreads();
    const T scale = scale_vec ? scale_in * __ldg(scale_vec + c.b) : scale_in;
    const typename Lat<T>::val ll = llf[c.b];
    const uint32_t u = c.u0 + lane;
    for (int i = warp; i < kIoTile; i += 8) {
        const uint32_t t = c.t0 + i;
        T vb = T(0), vy = T(0);
        if ((int)t < Tb && (int)u < Ub && live) {
            T eb, ey;
            lattice_occ<MOD>(fac[lane][i], alphas, betas, ll, d, c.b, t, u, Tb, Ub, eb, ey);
            vb = -(scale * eb);
            vy = -(scale * ey);
        }
        gb[lane][i] = vb;
        gy[lane][i] = vy;
    }
    __syncthreads();
    const uint32_t t = c.t0 + lane;
    for (int j = warp; j < kIoTile; j += 8) {
        const uint32_t uj = c.u0 + j;
        if (uj < (uint32_t)d.maxU && t < (uint32_t)d.maxT) {
            py_grad[((size_t)c.b * d.maxU + uj) * d.maxT + t] = from_compute<IO, T>(gb[j][lane]);
            if ((int)uj < d.maxU - 1)
                px_grad[((size_t)c.b * (d.maxU - 1) + uj) * d.maxT + t] = from_compute<IO, T>(gy[j][lane]);
        }
    }
}

// blocks of the tiled kernels above
inline unsigned lattice_io_blocks(const Dims& d) {
    return (unsigned)((size_t)d.N * ((d.maxT + kIoTile - 1) / kIoTile) * ((d.maxU + kIoTile - 1) / kIoTile));
}

}  // namespace b200rnnt
