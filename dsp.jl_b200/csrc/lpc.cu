// dspb200 -- linear prediction (src/lpc.jl): Burg's method (arburg, lpc(x, p, LPCBurg())) and the Levinson recursion
// (levinson, lpc(x, p, LPCLevinson())) for every column of an n x ncols matrix in the same launches.
//
// Everything except the reductions follows src/lpc.jl operation by operation in the input's eltype: muladd is one fma for
// reals and Base.muladd's form for complex (cmuladd below), every other expression rounds at each operation (the *_rn
// intrinsics keep nvcc from contracting them).  The reductions -- dot(x, x), dot(eb, ef) and the autocorrelation lags --
// use one fixed order that depends only on the reduction length L (DESIGN.md section 4):
//   - index i belongs to tile i / 1024 and lane i % 256;
//   - each lane of a tile accumulates its (up to four) indices in increasing order, acc = muladd(term, acc) from +0;
//   - a tile's 256 lane sums are added within each warp (lanes l and l + h, h = 16, 8, 4, 2, 1), then over the eight
//     warp sums (w and w + h, h = 4, 2, 1);
//   - the ceil(L / 1024) tile sums are added pairwise, adjacent tiles first (2i and 2i + 1), an odd last sum carried up
//     unchanged, until one is left; L == 0 gives +0.
// The pairwise tile tree is what lets a cluster split a column: a CTA that owns an aligned run of 2^q tiles computes that
// subtree alone, and the cluster combines the subtrees' roots with the same rule.
#include "common.cuh"
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace dspb200 {
namespace {

constexpr int LPC_THREADS = 256;                       // the lanes of a tile
constexpr int LPC_TILE = 1024;
constexpr int LPC_WARPS = LPC_THREADS / 32;
constexpr int LPC_BATCH = 8;                           // tiles whose warp sums are staged per barrier
constexpr int LPC_MAX_CLUSTER = 8;
constexpr int64_t LPC_P_MAX = 1024;
constexpr int64_t LPC_RESIDENT_BYTES = 192 << 10;      // 4 n sizeof(E) of the resident path's error buffers
constexpr int64_t LPC_SAMPLES_PER_CTA = 1 << 16;       // streamed path: one CTA of the cluster per 64 Ki samples
constexpr int LPC_ACF_LAGS = 64;                       // lags whose warp sums acf_tiles_kernel stages per barrier
constexpr int64_t LPC_GRID_ROWS = 65535;

// ------------------------------------------------------------------------------------------------ scalar arithmetic
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ float fma_rn(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ double fma_rn(double a, double b, double c) { return __fma_rn(a, b, c); }

__host__ __device__ __forceinline__ int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
template <typename T> __device__ __forceinline__ T zero_of(T) { return T(0); }
template <typename T> __device__ __forceinline__ cx<T> zero_of(cx<T>) { return mkc<T>(T(0), T(0)); }
template <typename T> __device__ __forceinline__ T one_of(T) { return T(1); }
template <typename T> __device__ __forceinline__ cx<T> one_of(cx<T>) { return mkc<T>(T(1), T(0)); }
template <typename T> __device__ __forceinline__ T conj_(T a) { return a; }
template <typename T> __device__ __forceinline__ cx<T> conj_(cx<T> a) { return mkc<T>(a.x, -a.y); }
template <typename T> __device__ __forceinline__ T neg_(T a) { return -a; }
template <typename T> __device__ __forceinline__ cx<T> neg_(cx<T> a) { return mkc<T>(-a.x, -a.y); }
template <typename T> __device__ __forceinline__ T add_(T a, T b) { return add_rn(a, b); }
template <typename T> __device__ __forceinline__ cx<T> add_(cx<T> a, cx<T> b) { return mkc<T>(add_rn(a.x, b.x), add_rn(a.y, b.y)); }
// abs2: re*re + im*im, each operation rounded (Julia does not contract)
template <typename T> __device__ __forceinline__ T abs2_(T a) { return mul_rn(a, a); }
template <typename T> __device__ __forceinline__ T abs2_(cx<T> a) { return add_rn(mul_rn(a.x, a.x), mul_rn(a.y, a.y)); }
// muladd: one fma for reals; Base.muladd(z, w, x) for complex,
// Complex(muladd(zr, wr, -muladd(zi, wi, -xr)), muladd(zr, wi, muladd(zi, wr, xi)))
template <typename T> __device__ __forceinline__ T muladd_(T a, T b, T c) { return fma_rn(a, b, c); }
template <typename T> __device__ __forceinline__ cx<T> muladd_(cx<T> z, cx<T> w, cx<T> x) {
    return mkc<T>(fma_rn(z.x, w.x, -fma_rn(z.y, w.y, -x.x)), fma_rn(z.x, w.y, fma_rn(z.y, w.x, x.y)));
}
// z / r for a real r: Complex(re / r, im / r)
template <typename T> __device__ __forceinline__ T div_real(T a, T r) { return div_rn(a, r); }
template <typename T> __device__ __forceinline__ cx<T> div_real(cx<T> a, T r) { return mkc<T>(div_rn(a.x, r), div_rn(a.y, r)); }
// (Int) -2 * z
template <typename T> __device__ __forceinline__ T times_m2(T a) { return mul_rn(T(-2), a); }
template <typename T> __device__ __forceinline__ cx<T> times_m2(cx<T> a) { return mkc<T>(mul_rn(T(-2), a.x), mul_rn(T(-2), a.y)); }
// a / b: real division; for complex, Smith's algorithm as Julia's generic /(::Complex{T}, ::Complex{T}) writes it
template <typename T> __device__ __forceinline__ T div_(T a, T b) { return div_rn(a, b); }
template <typename T> __device__ __forceinline__ cx<T> div_(cx<T> a, cx<T> b) {
    const T are = a.x, aim = a.y, bre = b.x, bim = b.y;
    if (isinf(bre) || isinf(bim)) {
        if (isfinite(are) && isfinite(aim)) {
            const T sre = are > 0 ? T(1) : are < 0 ? T(-1) : are, sbre = bre > 0 ? T(1) : bre < 0 ? T(-1) : bre;
            const T saim = aim > 0 ? T(1) : aim < 0 ? T(-1) : aim, sbim = bim > 0 ? T(1) : bim < 0 ? T(-1) : bim;
            return mkc<T>(mul_rn(mul_rn(T(0), sre), sbre), mul_rn(mul_rn(T(-0.0), saim), sbim));
        }
        return mkc<T>(T(NAN), T(NAN));
    }
    if (fabs(bre) <= fabs(bim)) {
        const T r = div_rn(bre, bim), den = add_rn(bim, mul_rn(r, bre));
        return mkc<T>(div_rn(add_rn(mul_rn(are, r), aim), den), div_rn(sub_rn(mul_rn(aim, r), are), den));
    }
    const T r = div_rn(bim, bre), den = add_rn(bre, mul_rn(r, bim));
    return mkc<T>(div_rn(add_rn(are, mul_rn(aim, r)), den), div_rn(sub_rn(aim, mul_rn(are, r)), den));
}
// xcorr's :biased division by n, the rule of dspb200_scale_div_async (a complex sample times the rounded reciprocal of
// n + 0im, as Smith's division with a zero imaginary part does)
template <typename T> __device__ __forceinline__ T biased(T a, T n) { return div_rn(a, n); }
template <typename T> __device__ __forceinline__ cx<T> biased(cx<T> a, T n) {
    const T rat = T(0), scl = div_rn(T(1), n);
    return mkc<T>(mul_rn(add_rn(a.x, mul_rn(a.y, rat)), scl), mul_rn(sub_rn(a.y, mul_rn(a.x, rat)), scl));
}

template <typename T> __device__ __forceinline__ T shfl_down(T v, int h) { return __shfl_down_sync(0xffffffffu, v, h); }
template <typename T> __device__ __forceinline__ cx<T> shfl_down(cx<T> v, int h) {
    return mkc<T>(__shfl_down_sync(0xffffffffu, v.x, h), __shfl_down_sync(0xffffffffu, v.y, h));
}
// lane sums of one warp: lanes l and l + h for h = 16 .. 1; lane 0 holds the warp sum
template <typename S> __device__ __forceinline__ S warp_tree(S v) {
    for (int h = 16; h > 0; h >>= 1) v = add_(v, shfl_down(v, h));
    return v;
}
// the eight warp sums of a tile: w and w + h for h = 4, 2, 1
template <typename S> __device__ __forceinline__ S tile_tree(const S* w) {
    const S a0 = add_(w[0], w[4]), a1 = add_(w[1], w[5]), a2 = add_(w[2], w[6]), a3 = add_(w[3], w[7]);
    return add_(add_(a0, a2), add_(a1, a3));
}
// v[0 .. cnt) added pairwise, adjacent first, the odd last value carried; in place, the result in v[0] (cnt >= 1)
template <typename S> __device__ __forceinline__ void pair_tree(S* v, int64_t cnt, int64_t stride) {
    while (cnt > 1) {
        const int64_t h = cnt >> 1;
        for (int64_t i = 0; i < h; ++i) v[i * stride] = add_(v[2 * i * stride], v[(2 * i + 1) * stride]);
        if (cnt & 1) v[h * stride] = v[(cnt - 1) * stride];
        cnt -= h;
    }
}

// The pairwise tile tree of one CTA's aligned run of tiles, fed tile by tile (in shared memory, one thread): a binary
// counter of subtree roots; fold() adds the remaining roots right to left, which is the carry rule on a partial run.
template <typename S> struct TileStack {
    S v[40];
    int lvl[40];
    int top;
    __device__ void reset() { top = 0; }
    __device__ void push(S s) {
        v[top] = s; lvl[top] = 0; ++top;
        while (top >= 2 && lvl[top - 1] == lvl[top - 2]) { v[top - 2] = add_(v[top - 2], v[top - 1]); ++lvl[top - 2]; --top; }
    }
    __device__ S fold() const {
        if (top == 0) return zero_of(S());
        S acc = v[top - 1];
        for (int k = top - 2; k >= 0; --k) acc = add_(v[k], acc);
        return acc;
    }
};

template <typename E> using real_of = typename elt_traits<E>::real;

// dot(x, x) of arburg: |x_i|^2 summed in the real eltype (its imaginary part is zero): fma(re, re, acc), then
// fma(im, im, .) for complex
template <typename T> __device__ __forceinline__ T sq_acc(T x, T acc) { return fma_rn(x, x, acc); }
template <typename T> __device__ __forceinline__ T sq_acc(cx<T> x, T acc) { return fma_rn(x.y, x.y, fma_rn(x.x, x.x, acc)); }

template <typename E, bool RES> __device__ __forceinline__ E ld(const E* p) {
    if constexpr (RES) return *p;
    else if constexpr (std::is_same<E, float>::value || std::is_same<E, double>::value) return __ldcg(p);
    else {
        using T = real_of<E>;
        if constexpr (sizeof(T) == 4) { const float2 v = __ldcg((const float2*)p); return mkc<float>(v.x, v.y); }
        else { const double2 v = __ldcg((const double2*)p); return mkc<double>(v.x, v.y); }
    }
}

// Shared state of one CTA of the Burg kernel.
template <typename E> struct BurgShared {
    using R = real_of<E>;
    E wsum[2][LPC_BATCH][LPC_WARPS];        // warp sums of a batch of tiles (double-buffered by batch parity)
    R wsum_r[2][LPC_BATCH][LPC_WARPS];      // dot(x, x) of the first pass
    TileStack<E> stk;
    TileStack<R> stk_r;
    E bval[2];                              // the CTA's subtree root of dot(eb, ef), by order parity (read by the cluster)
    R bval_r;
    E roots[LPC_MAX_CLUSTER];
    R roots_r[LPC_MAX_CLUSTER];
    E k;
};

// One pass over a column, run by every thread of every CTA of the column's cluster (C CTAs, this one `rank`).
//   first:  reads x (ef = eb = x), accumulates dot(x, x) over n and dot(eb, ef) of order 1 over n - 1 (when want_dot).
//   else:   the error update of order m (ef_n[i] = muladd(k, eb[m+i], ef[i]), eb_n[m+i] = muladd(conj k, ef[i], eb[m+i]) for
//           i < n - m) fused with dot(eb, ef) of order m + 1 over n - m - 1 (when want_dot): the term of index i takes
//           eb_n[m+1+i] recomputed from ef[i+1] and eb[m+1+i], so no thread waits for its neighbour's write.
// The CTA's subtree root lands in sh.bval[par] (and sh.bval_r), written by thread 0 after the last barrier of the pass.
template <typename E, bool RES, bool FIRST>
__device__ void burg_pass(BurgShared<E>& sh, const E* ef_o, const E* eb_o, E* ef_n, E* eb_n, int64_t n, int64_t m, E k,
                          bool want_dot, int C, int rank, int par) {
    using R = real_of<E>;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t nupd = FIRST ? n : n - m, ldot = want_dot ? nupd - 1 : 0;
    const int64_t tupd = ceil_div(nupd, LPC_TILE), tdot = ceil_div(ldot, LPC_TILE), tsq = FIRST ? tupd : 0;
    int64_t B = 1;
    while (B * C < tupd) B <<= 1;
    const int64_t t0 = (int64_t)rank * B, t1 = t0 + B < tupd ? t0 + B : tupd;
    const E kc = conj_(k);
    if (tid == 0) { sh.stk.reset(); sh.stk_r.reset(); }
    int64_t bt = t0;                                     // first tile of the batch thread 0 has not consumed yet
    int b = 0, bp = 0;
    for (int64_t t = t0; t < t1; ++t) {
        E acc = zero_of(E());
        R accr = R(0);
#pragma unroll
        for (int j = 0; j < LPC_TILE / LPC_THREADS; ++j) {
            const int64_t i = t * LPC_TILE + j * LPC_THREADS + tid;
            if (i < nupd) {
                if constexpr (FIRST) {
                    const E xi = ef_o[i];
                    accr = sq_acc(xi, accr);
                    if (i < ldot) acc = muladd_(conj_(ef_o[i + 1]), xi, acc);
                } else {
                    const E f = ld<E, RES>(ef_o + i), e = ld<E, RES>(eb_o + m + i);
                    const E fn = muladd_(k, e, f);
                    ef_n[i] = fn;
                    eb_n[m + i] = muladd_(kc, f, e);
                    if (i < ldot) {
                        const E e1 = muladd_(kc, ld<E, RES>(ef_o + i + 1), ld<E, RES>(eb_o + m + 1 + i));
                        acc = muladd_(conj_(e1), fn, acc);
                    }
                }
            }
        }
        acc = warp_tree(acc);
        if (FIRST) accr = warp_tree(accr);
        if (lane == 0) { sh.wsum[bp][b][warp] = acc; if (FIRST) sh.wsum_r[bp][b][warp] = accr; }
        if (++b == LPC_BATCH || t + 1 == t1) {
            __syncthreads();
            if (tid == 0) {
                for (int q = 0; q < b; ++q) {
                    if (bt + q < tdot) sh.stk.push(tile_tree(sh.wsum[bp][q]));
                    if (FIRST && bt + q < tsq) sh.stk_r.push(tile_tree(sh.wsum_r[bp][q]));
                }
            }
            bt += b; b = 0; bp ^= 1;
        }
    }
    __syncthreads();
    if (tid == 0) {
        sh.bval[par] = sh.stk.fold();
        if (FIRST) sh.bval_r = sh.stk_r.fold();
    }
    (void)tsq;
}

// Combines the cluster's subtree roots (thread 0, after the barrier that publishes them): the pairwise tile tree above
// the CTAs' aligned runs.  L: reduction length, tupd: tiles of the pass, C: CTAs.
template <typename S, class Get>
__device__ S combine_roots(S* roots, int64_t L, int64_t tupd, int C, Get get) {
    int64_t B = 1;
    while (B * C < tupd) B <<= 1;
    const int64_t tl = ceil_div(L, LPC_TILE);
    const int cnt = (int)ceil_div(tl, B);
    if (cnt == 0) return zero_of(S());
    for (int r = 0; r < cnt; ++r) roots[r] = get(r);
    pair_tree(roots, cnt, 1);
    return roots[0];
}

// Burg's method (arburg, src/lpc.jl:53-92) for every column of x (n x ncols).  RES: one CTA per column, the forward and
// backward errors in shared memory.  !RES: one cluster of C CTAs per column, the errors in `work` (4 n elements per grid
// row: two ping-pong pairs), one HBM pass and one cluster barrier per order.  Both keep eb at its original index: after
// order m, ef holds indices 0 .. n-m-1 and eb indices m .. n-1.
template <typename E, bool RES>
__global__ void __launch_bounds__(LPC_THREADS, sizeof(E) == 16 ? (RES ? 3 : 2) : 4) burg_kernel(const E* __restrict__ x, int64_t n, int64_t ncols, int p,
                                                          E* __restrict__ a_out, real_of<E>* __restrict__ err_out,
                                                          E* __restrict__ refl_out, E* work) {
    using R = real_of<E>;
    extern __shared__ __align__(16) unsigned char lpc_dyn[];
    __shared__ BurgShared<E> sh;
    const int tid = threadIdx.x;
    int C = 1, rank = 0;
    if constexpr (!RES) {
        cg::cluster_group cluster = cg::this_cluster();
        C = (int)cluster.num_blocks();
        rank = (int)cluster.block_rank();
    }
    E* abuf = (E*)lpc_dyn;                               // a[0 .. p]
    E* ebase = RES ? abuf + (p + 1) : work + (RES ? 0 : (int64_t)blockIdx.y * 4 * n);
    const int64_t col0 = RES ? blockIdx.x : blockIdx.y, cstep = RES ? gridDim.x : gridDim.y;

    // publishes the CTAs' roots of a pass; thread 0 then reads them all (for RES: its own)
    auto publish = [&]() {
        if constexpr (RES) __syncthreads();
        else { __threadfence(); cg::this_cluster().sync(); }
    };
    auto remote_e = [&](int r, int par) -> E {
        if constexpr (RES) return sh.bval[par];
        else return *cg::this_cluster().map_shared_rank(&sh.bval[par], r);
    };
    auto remote_r = [&](int r) -> R {
        if constexpr (RES) return sh.bval_r;
        else return *cg::this_cluster().map_shared_rank(&sh.bval_r, r);
    };

    for (int64_t c = col0; c < ncols; c += cstep) {
        const E* xc = x + c * n;
        for (int j = tid; j <= p; j += LPC_THREADS) abuf[j] = j == 0 ? one_of(E()) : zero_of(E());
        // first pass: dot(x, x) and dot(eb, ef) of order 1
        burg_pass<E, RES, true>(sh, xc, xc, nullptr, nullptr, n, 0, zero_of(E()), p >= 1, C, rank, 0);
        publish();
        R err = R(0), den = R(0), ratio = R(1);
        E dot = zero_of(E());
        if (tid == 0) {
            const int64_t tupd = ceil_div(n, LPC_TILE);
            const R un = fabs(combine_roots<R>(sh.roots_r, n, tupd, C, [&](int r) { return remote_r(r); }));
            dot = combine_roots<E>(sh.roots, p >= 1 ? n - 1 : 0, tupd, C, [&](int r) { return remote_e(r, 0); });
            err = div_rn(un, (R)n);                       // unnormed_err / length(x)
            den = mul_rn(R(2), un);                       // convert(R, 2unnormed_err)
        }
        const E* ef_c = xc;                               // the errors after the last update: x before order 1
        const E* eb_c = xc;
        E* ef_n = ebase;                                  // where the next update goes (ping-pong with ebase + 2n)
        E* eb_n = ebase + n;
        for (int m = 1; m <= p; ++m) {
            if (tid == 0) {
                const E cf = m == 1 ? xc[n - m] : ld<E, RES>(ef_c + (n - m));   // pop!(ef)
                const E cb = m == 1 ? xc[m - 1] : ld<E, RES>(eb_c + (m - 1));   // popfirst!(eb)
                den = fma_rn(ratio, den, -add_rn(abs2_(cf), abs2_(cb)));
                const E k = div_real(times_m2(dot), den);
                sh.k = k;
                if (rank == 0 && refl_out) refl_out[c * p + (m - 1)] = k;
                ratio = sub_rn(R(1), abs2_(k));
                err = mul_rn(err, ratio);
            }
            __syncthreads();
            const E k = sh.k;
            // a[2:m+1] = muladd(k, conj(a[m:-1:1]), a[2:m+1]) (1-based); a[m+1] is still zero
            E na[LPC_P_MAX / LPC_THREADS];
#pragma unroll
            for (int r = 0; r < (int)(LPC_P_MAX / LPC_THREADS); ++r) {
                const int j = tid + 1 + r * LPC_THREADS;
                if (j <= m) na[r] = muladd_(k, conj_(abuf[m - j]), abuf[j]);
            }
            if (m < p) {
                burg_pass<E, RES, false>(sh, ef_c, eb_c, ef_n, eb_n, n, m, k, true, C, rank, m & 1);
                ef_c = ef_n; eb_c = eb_n;
                ef_n = ef_n == ebase ? ebase + 2 * n : ebase;
                eb_n = ef_n + n;
            } else {
                __syncthreads();
            }
#pragma unroll
            for (int r = 0; r < (int)(LPC_P_MAX / LPC_THREADS); ++r) {
                const int j = tid + 1 + r * LPC_THREADS;
                if (j <= m) abuf[j] = na[r];
            }
            if (m < p) {
                publish();
                if (tid == 0) {
                    const int par = m & 1;
                    dot = combine_roots<E>(sh.roots, n - m - 1, ceil_div(n - m, LPC_TILE), C,
                                           [&](int r) { return remote_e(r, par); });
                }
            }
        }
        __syncthreads();
        if (rank == 0) {
            for (int j = tid; j <= p; j += LPC_THREADS) a_out[c * (p + 1) + j] = conj_(abuf[j]);   // conj!(a)
            if (tid == 0) err_out[c] = err;
        }
        if constexpr (!RES) cg::this_cluster().sync();   // every root stays readable until the cluster has read it
        else __syncthreads();
    }
}

// The autocorrelation partials of lpc(x, p, LPCLevinson()): tile t of column c, for every lag k <= p, the tile sum of
// r[k] = sum_i x[i + k] conj(x[i]) over the indices i < n - k of the tile (acc = muladd(x[i + k], conj(x[i]), acc)), into
// part[(c (p + 1) + k) T + t], T = ceil(n / 1024).  Tiles past ceil((n - k) / 1024) hold no index of lag k and are not
// written.  The tile's samples and a halo of p are staged in shared memory.
template <typename E>
__global__ void __launch_bounds__(LPC_THREADS, 4) acf_tiles_kernel(const E* __restrict__ x, int64_t n, int64_t ncols, int p,
                                                               E* __restrict__ part) {
    extern __shared__ __align__(16) unsigned char lpc_dyn[];
    E* xs = (E*)lpc_dyn;                                     // LPC_TILE + p samples
    E* ws = xs + LPC_TILE + p;                               // [LPC_ACF_LAGS][LPC_WARPS]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t T = ceil_div(n, LPC_TILE), t = blockIdx.x;
    for (int64_t c = blockIdx.y; c < ncols; c += gridDim.y) {
        const E* xc = x + c * n;
        const int64_t base = t * LPC_TILE;
        for (int64_t q = tid; q < LPC_TILE + p; q += LPC_THREADS) xs[q] = base + q < n ? xc[base + q] : zero_of(E());
        __syncthreads();
        for (int k0 = 0; k0 <= p; k0 += LPC_ACF_LAGS) {
            const int kn = p + 1 - k0 < LPC_ACF_LAGS ? p + 1 - k0 : LPC_ACF_LAGS;
            for (int kk = 0; kk < kn; ++kk) {
                const int k = k0 + kk;
                E acc = zero_of(E());
#pragma unroll
                for (int j = 0; j < LPC_TILE / LPC_THREADS; ++j) {
                    const int q = j * LPC_THREADS + tid;
                    if (base + q < n - k) acc = muladd_(xs[q + k], conj_(xs[q]), acc);
                }
                acc = warp_tree(acc);
                if (lane == 0) ws[kk * LPC_WARPS + warp] = acc;
            }
            __syncthreads();
            if (tid < kn) {
                const int k = k0 + tid;
                if (t < ceil_div(n - k, LPC_TILE)) part[(c * (p + 1) + k) * T + t] = tile_tree(ws + tid * LPC_WARPS);
            }
            __syncthreads();
        }
    }
}

// levinson (src/lpc.jl:122-146), one thread per column.  PART: the column's autocorrelation first, from acf_tiles_kernel's
// partials (lag k: the pairwise tree over its ceil((n - k) / 1024) tiles, in place, then the :biased division by n); r[k]
// is then part[(c (p + 1) + k) T].  Otherwise r[k] = r_in[c nr + k].  a and refl are p x ncols, err ncols.
template <typename E, bool PART>
__global__ void __launch_bounds__(LPC_THREADS, 1) levinson_kernel(const E* __restrict__ r_in, int64_t nr, int64_t ncols, int p,
                                                              E* part, int64_t n, E* __restrict__ a_out,
                                                              real_of<E>* __restrict__ err_out, E* __restrict__ refl_out) {
    using R = real_of<E>;
    const int64_t T = ceil_div(n, LPC_TILE);
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < ncols; c += (int64_t)gridDim.x * blockDim.x) {
        const E* rr;
        int64_t rs;
        if constexpr (PART) {
            E* pc = part + c * (p + 1) * T;
            for (int k = 0; k <= p; ++k) {
                E* s = pc + (int64_t)k * T;
                pair_tree(s, ceil_div(n - k, LPC_TILE), 1);
                s[0] = biased(s[0], (R)n);
            }
            rr = pc;
            rs = T;
        } else {
            rr = r_in + c * nr;
            rs = 1;
        }
        E* a = a_out + c * p;
        E* refl = refl_out ? refl_out + c * p : nullptr;
        const E r0 = rr[0];
        E k = div_(neg_(rr[rs]), r0);                                       // k = -R_xx[2] / R_xx[1]
        // prediction_err = real(R_xx[1] * (one(F) - abs2(k)))
        R err;
        if constexpr (std::is_same<E, R>::value) err = mul_rn(r0, sub_rn(R(1), abs2_(k)));
        else err = sub_rn(mul_rn(r0.x, sub_rn(R(1), abs2_(k))), mul_rn(r0.y, R(0)));
        a[0] = k;
        if (refl) refl[0] = k;
        for (int m = 2; m <= p; ++m) {
            E d = zero_of(E());                                             // dotu(R_xx[2:m], a[m-1:-1:1]), in order
            for (int i = 0; i <= m - 2; ++i) d = muladd_(rr[(int64_t)(1 + i) * rs], a[m - 2 - i], d);
            k = div_real(neg_(add_(rr[(int64_t)m * rs], d)), err);
            for (int j = 0; j <= (m - 2) / 2; ++j) {                        // a[1:m-1] = muladd(k, conj(rev_a), a[1:m-1])
                const int h = m - 2 - j;
                const E lo = a[j], hi = a[h];
                a[j] = muladd_(k, conj_(hi), lo);
                if (h != j) a[h] = muladd_(k, conj_(lo), hi);
            }
            a[m - 1] = k;
            if (refl) refl[m - 1] = k;
            err = mul_rn(err, sub_rn(R(1), abs2_(k)));
        }
        err_out[c] = err;
    }
}

// ------------------------------------------------------------------------------------------------ host side
bool lpc_shape_ok(int64_t n, int64_t ncols, size_t esz) {
    if (n < 0 || ncols < 0 || n > DSPB200_INDEX_LIMIT || ncols > DSPB200_INDEX_LIMIT) return false;
    return ncols == 0 || n <= DSPB200_INDEX_LIMIT / ncols / (int64_t)esz / 4;
}
bool burg_resident_fits(int64_t n, size_t esz) { return 4 * n * (int64_t)esz <= LPC_RESIDENT_BYTES; }
// the path rule: resident when the column's four error buffers fit LPC_RESIDENT_BYTES, else a cluster of
// ceil(n / 64 Ki) CTAs, at most 8; pin overrides it (-1 resident, 1..8 that many CTAs)
int burg_ctas(int64_t n, size_t esz, int pin) {
    if (pin == -1) return 0;
    if (pin > 0) return pin;
    if (burg_resident_fits(n, esz)) return 0;
    const int64_t c = cdiv(n, LPC_SAMPLES_PER_CTA);
    return (int)(c < 1 ? 1 : c > LPC_MAX_CLUSTER ? LPC_MAX_CLUSTER : c);
}
int64_t grid_rows(int64_t ncols) { return ncols < LPC_GRID_ROWS ? ncols : LPC_GRID_ROWS; }

int64_t burg_work_bytes(int64_t n, int64_t ncols, size_t esz, int pin) {
    if (burg_ctas(n, esz, pin) == 0) return 0;
    return grid_rows(ncols) * 4 * n * (int64_t)esz;
}
int64_t levinson_work_bytes(int64_t n, int64_t ncols, int64_t p, size_t esz) {
    return ncols * (p + 1) * cdiv(n, LPC_TILE) * (int64_t)esz;
}

template <typename E>
int burg_launch(const void* x, int64_t n, int64_t ncols, int p, void* a, void* err, void* refl, void* work, int ctas,
                cudaStream_t st) {
    using R = real_of<E>;
    const size_t esz = sizeof(E);
    if (ctas == 0) {
        const size_t smem = (size_t)(p + 1) * esz + (size_t)(4 * n) * esz;
        auto kern = burg_kernel<E, true>;
        if (smem > 48 * 1024) DSP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const unsigned grid = (unsigned)(ncols < 0x7fffffff ? ncols : 0x7fffffff);
        kern<<<grid, LPC_THREADS, smem, st>>>((const E*)x, n, ncols, p, (E*)a, (R*)err, (E*)refl, nullptr);
        DSP_LAUNCH_OK();
        return DSPB200_OK;
    }
    const size_t smem = (size_t)(p + 1) * esz;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)ctas, (unsigned)grid_rows(ncols));
    cfg.blockDim = dim3(LPC_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = (unsigned)ctas;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    DSP_CUDA(cudaLaunchKernelEx(&cfg, burg_kernel<E, false>, (const E*)x, n, ncols, p, (E*)a, (R*)err, (E*)refl, (E*)work));
    DSP_LAUNCH_OK();
    return DSPB200_OK;
}

template <typename E>
int levinson_launch(const void* r, int64_t nr, int64_t ncols, int p, void* part, int64_t n, void* a, void* err, void* refl,
                    cudaStream_t st) {
    using R = real_of<E>;
    int64_t blocks = cdiv(ncols, LPC_THREADS);
    if (blocks > (int64_t)device_sm_count() * 64) blocks = (int64_t)device_sm_count() * 64;
    if (part)
        levinson_kernel<E, true><<<(unsigned)blocks, LPC_THREADS, 0, st>>>(nullptr, 0, ncols, p, (E*)part, n, (E*)a, (R*)err,
                                                                            (E*)refl);
    else
        levinson_kernel<E, false><<<(unsigned)blocks, LPC_THREADS, 0, st>>>((const E*)r, nr, ncols, p, nullptr, 0, (E*)a, (R*)err,
                                                                             (E*)refl);
    DSP_LAUNCH_OK();
    return DSPB200_OK;
}

template <typename E>
int lpc_levinson_launch(const void* x, int64_t n, int64_t ncols, int p, void* a, void* err, void* refl, void* work,
                        cudaStream_t st) {
    const int64_t T = cdiv(n, LPC_TILE);
    const size_t smem = (size_t)(LPC_TILE + p + LPC_ACF_LAGS * LPC_WARPS) * sizeof(E);
    auto kern = acf_tiles_kernel<E>;
    if (smem > 48 * 1024) DSP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<dim3((unsigned)T, (unsigned)grid_rows(ncols)), LPC_THREADS, smem, st>>>((const E*)x, n, ncols, p, (E*)work);
    DSP_LAUNCH_OK();
    return levinson_launch<E>(nullptr, 0, ncols, p, work, n, a, err, refl, st);
}

size_t real_size(int dtype) { return dtype_is_f64(dtype) ? 8 : 4; }

// the refusals shared by the three calls: outputs a (na x ncols), err (ncols), refl (p x ncols, optional) overlapping each
// other, an input or the workspace
bool outputs_disjoint(const void* in, size_t in_bytes, const void* work, size_t work_bytes, const void* a, size_t a_bytes,
                      const void* err, size_t err_bytes, const void* refl, size_t refl_bytes) {
    const void* o[3] = {a, err, refl};
    const size_t ob[3] = {a_bytes, err_bytes, refl_bytes};
    for (int i = 0; i < 3; ++i) {
        if (ranges_overlap(o[i], ob[i], in, in_bytes) || ranges_overlap(o[i], ob[i], work, work_bytes)) return false;
        for (int j = i + 1; j < 3; ++j)
            if (ranges_overlap(o[i], ob[i], o[j], ob[j])) return false;
    }
    return !ranges_overlap(in, in_bytes, work, work_bytes);
}

}  // namespace
}  // namespace dspb200

using namespace dspb200;

extern "C" {

int dspb200_lpc_work_bytes(int dtype, int64_t n, int64_t ncols, int64_t p, int method, int pin, int64_t* bytes) {
    DSP_REQUIRE(dtype_valid(dtype), "invalid dtype %d", dtype);
    DSP_REQUIRE(bytes != nullptr, "NULL argument");
    DSP_REQUIRE(method == 0 || method == 1, "method must be 0 (Burg) or 1 (Levinson)");
    const size_t esz = dtype_size(dtype);
    DSP_REQUIRE(lpc_shape_ok(n, ncols, esz) && p >= 0 && p <= DSPB200_INDEX_LIMIT, "negative or oversized size");
    DSP_REQUIRE(pin >= -1 && pin <= LPC_MAX_CLUSTER, "pin must be -1, 0 or 1 .. %d", LPC_MAX_CLUSTER);
    if (p > LPC_P_MAX) { set_error("p = %lld exceeds LPC_P_MAX = %lld", (long long)p, (long long)LPC_P_MAX); return DSPB200_EUNSUPPORTED; }
    *bytes = method == 0 ? burg_work_bytes(n, ncols, esz, pin) : levinson_work_bytes(n, ncols, p, esz);
    return DSPB200_OK;
}

int dspb200_lpc_burg_async(int dtype, const void* x, int64_t n, int64_t ncols, int64_t p, void* a, void* err, void* refl,
                           void* work, int pin, void* stream) {
    DSP_RANGE("dspb200_lpc_burg_async");
    DSP_REQUIRE(dtype_valid(dtype), "invalid dtype %d", dtype);
    const size_t esz = dtype_size(dtype), rsz = real_size(dtype);
    DSP_REQUIRE(lpc_shape_ok(n, ncols, esz) && p >= 0, "negative or oversized size");
    DSP_REQUIRE(p <= n, "Burg needs 0 <= p <= n (p %lld, n %lld)", (long long)p, (long long)n);
    DSP_REQUIRE(pin >= -1 && pin <= LPC_MAX_CLUSTER, "pin must be -1, 0 or 1 .. %d", LPC_MAX_CLUSTER);
    if (p > LPC_P_MAX) { set_error("p = %lld exceeds LPC_P_MAX = %lld", (long long)p, (long long)LPC_P_MAX); return DSPB200_EUNSUPPORTED; }
    if (pin == -1 && !burg_resident_fits(n, esz)) {
        set_error("a column of %lld samples does not fit the resident path", (long long)n);
        return DSPB200_EUNSUPPORTED;
    }
    if (ncols == 0) return DSPB200_OK;
    const int64_t wbytes = burg_work_bytes(n, ncols, esz, pin);
    DSP_REQUIRE(a && err && (x || n == 0) && (work || wbytes == 0), "NULL argument");
    const size_t xb = (size_t)(n * ncols) * esz;
    DSP_REQUIRE(outputs_disjoint(x, xb, work, (size_t)wbytes, a, (size_t)((p + 1) * ncols) * esz, err, (size_t)ncols * rsz, refl,
                                 (size_t)(p * ncols) * esz),
                "an output overlaps an input, the workspace or another output");
    const int ctas = burg_ctas(n, esz, pin);
    const cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case DSPB200_F32: return burg_launch<float>(x, n, ncols, (int)p, a, err, refl, work, ctas, st);
        case DSPB200_F64: return burg_launch<double>(x, n, ncols, (int)p, a, err, refl, work, ctas, st);
        case DSPB200_C32: return burg_launch<cx<float>>(x, n, ncols, (int)p, a, err, refl, work, ctas, st);
        default: return burg_launch<cx<double>>(x, n, ncols, (int)p, a, err, refl, work, ctas, st);
    }
}

int dspb200_lpc_levinson_async(int dtype, const void* x, int64_t n, int64_t ncols, int64_t p, void* a, void* err, void* refl,
                               void* work, void* stream) {
    DSP_RANGE("dspb200_lpc_levinson_async");
    DSP_REQUIRE(dtype_valid(dtype), "invalid dtype %d", dtype);
    const size_t esz = dtype_size(dtype), rsz = real_size(dtype);
    DSP_REQUIRE(lpc_shape_ok(n, ncols, esz) && p >= 0, "negative or oversized size");
    DSP_REQUIRE(p >= 1 && p <= n - 1, "Levinson needs 1 <= p <= n - 1 (p %lld, n %lld)", (long long)p, (long long)n);
    if (p > LPC_P_MAX) { set_error("p = %lld exceeds LPC_P_MAX = %lld", (long long)p, (long long)LPC_P_MAX); return DSPB200_EUNSUPPORTED; }
    if (ncols == 0) return DSPB200_OK;
    const int64_t wbytes = levinson_work_bytes(n, ncols, p, esz);
    DSP_REQUIRE(x && a && err && work, "NULL argument");
    DSP_REQUIRE(outputs_disjoint(x, (size_t)(n * ncols) * esz, work, (size_t)wbytes, a, (size_t)(p * ncols) * esz, err,
                                 (size_t)ncols * rsz, refl, (size_t)(p * ncols) * esz),
                "an output overlaps an input, the workspace or another output");
    const cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case DSPB200_F32: return lpc_levinson_launch<float>(x, n, ncols, (int)p, a, err, refl, work, st);
        case DSPB200_F64: return lpc_levinson_launch<double>(x, n, ncols, (int)p, a, err, refl, work, st);
        case DSPB200_C32: return lpc_levinson_launch<cx<float>>(x, n, ncols, (int)p, a, err, refl, work, st);
        default: return lpc_levinson_launch<cx<double>>(x, n, ncols, (int)p, a, err, refl, work, st);
    }
}

int dspb200_levinson_async(int dtype, const void* r, int64_t nr, int64_t ncols, int64_t p, void* a, void* err, void* refl,
                           void* stream) {
    DSP_RANGE("dspb200_levinson_async");
    DSP_REQUIRE(dtype_valid(dtype), "invalid dtype %d", dtype);
    const size_t esz = dtype_size(dtype), rsz = real_size(dtype);
    DSP_REQUIRE(lpc_shape_ok(nr, ncols, esz) && p >= 0, "negative or oversized size");
    DSP_REQUIRE(p >= 1 && p <= nr - 1, "levinson needs 1 <= p <= length(r) - 1 (p %lld, nr %lld)", (long long)p, (long long)nr);
    if (p > LPC_P_MAX) { set_error("p = %lld exceeds LPC_P_MAX = %lld", (long long)p, (long long)LPC_P_MAX); return DSPB200_EUNSUPPORTED; }
    if (ncols == 0) return DSPB200_OK;
    DSP_REQUIRE(r && a && err, "NULL argument");
    DSP_REQUIRE(outputs_disjoint(r, (size_t)(nr * ncols) * esz, nullptr, 0, a, (size_t)(p * ncols) * esz, err, (size_t)ncols * rsz,
                                 refl, (size_t)(p * ncols) * esz),
                "an output overlaps r or another output");
    const cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case DSPB200_F32: return levinson_launch<float>(r, nr, ncols, (int)p, nullptr, 0, a, err, refl, st);
        case DSPB200_F64: return levinson_launch<double>(r, nr, ncols, (int)p, nullptr, 0, a, err, refl, st);
        case DSPB200_C32: return levinson_launch<cx<float>>(r, nr, ncols, (int)p, nullptr, 0, a, err, refl, st);
        default: return levinson_launch<cx<double>>(r, nr, ncols, (int)p, nullptr, 0, a, err, refl, st);
    }
}

}  // extern "C"
