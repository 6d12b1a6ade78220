// dspb200 -- the device work of the thin clients of the convolution path (src/dspbase.jl:867-898, src/util.jl:336-427,
// src/Filters/filt.jl:245-259, 301-337): the odd-symmetric extension of filtfilt, the peak search of finddelay, the zero-filled
// shift of shiftsignal / alignsignals, the :biased scaling of xcorr and the column-batched FFT convolution of xcorr's
// :fft_simple route.  The filtering and correlation themselves run on the FIR, overlap-save and direct kernels unchanged.
#include "common.cuh"
#include "cufft_exec.cuh"
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace dspb200 {
namespace {

template <typename T, bool CPLX> struct cl_elt { using type = T; };
template <typename T> struct cl_elt<T, true> { using type = cx<T>; };

// Correctly rounded scalar operations: the compiler may not contract them into a fused multiply-add, so every step rounds
// as numpy's does on the host.
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }

// 2x0 - x[k] of extrapolate_signal!: the factor 2 is a complex number for complex data (numpy multiplies 2 + 0im by the
// sample, so the signs of zeros follow the full complex product)
template <typename T> __device__ __forceinline__ T reflect(T x0, T xk) { return sub_rn(mul_rn(T(2), x0), xk); }
template <typename T> __device__ __forceinline__ cx<T> reflect(cx<T> x0, cx<T> xk) {
    const T re = sub_rn(mul_rn(T(2), x0.x), mul_rn(T(0), x0.y)), im = add_rn(mul_rn(T(2), x0.y), mul_rn(T(0), x0.x));
    return mkc<T>(sub_rn(re, xk.x), sub_rn(im, xk.y));
}

// extrapolate_signal!, src/Filters/filt.jl:245-259: column c of ext (n + 2 pad samples) is
// [2x0 - x[pad:-1:1]; x; 2x[n-1] - x[n-2:-1:n-1-pad]] (0-based) of column c of x.  Consecutive threads write consecutive
// samples of a column and read consecutive (ascending or descending) samples of it.
template <typename E>
__global__ void filtfilt_extend_kernel(const E* __restrict__ x, int64_t n, int64_t ncols, int64_t pad, E* __restrict__ ext) {
    const int64_t next = n + 2 * pad;
    for (int64_t c = blockIdx.y; c < ncols; c += gridDim.y) {
        const E* xc = x + c * n;
        E* ec = ext + c * next;
        for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < next; r += (int64_t)gridDim.x * blockDim.x) {
            E v;
            if (r < pad) v = reflect(xc[0], xc[pad - r]);
            else if (r < pad + n) v = xc[r - pad];
            else v = reflect(xc[n - 1], xc[n - 2 - (r - pad - n)]);
            ec[r] = v;
        }
    }
}

// finddelay's choice among the samples of largest magnitude (src/util.jl:360-368): the one closest to `center`
// (1-based), the lower index on a tie.  i < 0 marks "no candidate yet".  Every key is distinct (i is), so this is a strict
// total order and the maximum is the same whatever order the reduction visits the samples in.
template <typename T>
__device__ __forceinline__ bool peak_better(T ma, int64_t ia, T mb, int64_t ib, int64_t center) {
    if (ia < 0) return false;
    if (ib < 0) return true;
    if (ma != mb) return ma > mb;
    const int64_t da = center - 1 - ia, db = center - 1 - ib;
    const int64_t aa = da < 0 ? -da : da, ab = db < 0 ? -db : db;
    if (aa != ab) return aa < ab;
    return ia < ib;
}

constexpr int PEAK_THREADS = 512;
constexpr int PEAK_MAX_CLUSTER = 8;

// One cluster of `cs` CTAs per column of s (nres x ncols, column-major): each CTA reduces a contiguous slice, the cluster's
// first CTA combines the slices through distributed shared memory and writes delay[c] = center - (i + 1) and nanflag[c]
// (1 when the column holds a NaN: the reference's argmin over an empty set throws).  reversed != 0: sample p of the column
// is the correlation at logical index nres - 1 - p (xcorr(y, x) read off xcorr(x, y) for real data).
template <typename T>
__global__ void __launch_bounds__(PEAK_THREADS) xcorr_peak_kernel(const T* __restrict__ s, int64_t nres, int64_t ncols,
                                                                  int64_t center, int reversed, int64_t* __restrict__ delay,
                                                                  int* __restrict__ nanflag) {
    cg::cluster_group cluster = cg::this_cluster();
    const int cs = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
    __shared__ T w_mag[PEAK_THREADS / 32];
    __shared__ int64_t w_idx[PEAK_THREADS / 32];
    __shared__ int w_nan[PEAK_THREADS / 32];
    __shared__ T b_mag;
    __shared__ int64_t b_idx;
    __shared__ int b_nan;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t c = blockIdx.y; c < ncols; c += gridDim.y) {
        const T* col = s + c * nres;
        const int64_t lo = nres * rank / cs, hi = nres * (rank + 1) / cs;
        T m = T(-1);
        int64_t idx = -1;
        int nan = 0;
        for (int64_t p = lo + threadIdx.x; p < hi; p += PEAK_THREADS) {
            const T a = fabs(col[p]);
            const int64_t i = reversed ? nres - 1 - p : p;
            if (a != a) nan = 1;
            else if (peak_better(a, i, m, idx, center)) { m = a; idx = i; }
        }
        for (int off = 16; off > 0; off >>= 1) {
            const T om = __shfl_down_sync(0xffffffffu, m, off);
            const int64_t oi = __shfl_down_sync(0xffffffffu, idx, off);
            nan |= __shfl_down_sync(0xffffffffu, nan, off);
            if (peak_better(om, oi, m, idx, center)) { m = om; idx = oi; }
        }
        if (lane == 0) { w_mag[warp] = m; w_idx[warp] = idx; w_nan[warp] = nan; }
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int k = 1; k < PEAK_THREADS / 32; ++k) {
                nan |= w_nan[k];
                if (peak_better(w_mag[k], w_idx[k], m, idx, center)) { m = w_mag[k]; idx = w_idx[k]; }
            }
            b_mag = m; b_idx = idx; b_nan = nan;
        }
        cluster.sync();
        if (rank == 0 && threadIdx.x == 0) {
            for (int r = 1; r < cs; ++r) {
                const T om = *cluster.map_shared_rank(&b_mag, r);
                const int64_t oi = *cluster.map_shared_rank(&b_idx, r);
                nan |= *cluster.map_shared_rank(&b_nan, r);
                if (peak_better(om, oi, m, idx, center)) { m = om; idx = oi; }
            }
            delay[c] = center - (idx + 1);
            nanflag[c] = nan;
        }
        cluster.sync();                      // the slices' results stay readable until rank 0 has combined them
    }
}

// shiftsignal (src/util.jl:379-412), out of place: out[i, c] = x[i - s_c, c] where 0 <= i - s_c < nx, else zero, for
// i < nout.  s_c = shifts[c] (negated when `negate`) when shifts is given, else `shift`.
template <typename E>
__global__ void shift_kernel(const E* __restrict__ x, int64_t nx, int64_t ncols, int64_t shift, const int64_t* __restrict__ shifts,
                             int negate, E* __restrict__ out, int64_t nout) {
    for (int64_t c = blockIdx.y; c < ncols; c += gridDim.y) {
        int64_t s = shift;
        if (shifts) s = negate ? -shifts[c] : shifts[c];
        const E* xc = x + c * nx;
        E* oc = out + c * nout;
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nout; i += (int64_t)gridDim.x * blockDim.x) {
            const int64_t j = i - s;
            E v;
            if (j >= 0 && j < nx) v = xc[j];
            else memset(&v, 0, sizeof(E));
            oc[i] = v;
        }
    }
}

// xcorr's :biased scaling res / su (src/dspbase.jl:894), as numpy divides: a real sample by su, a complex sample by the
// complex number su + 0im (Smith's algorithm with ratio 0: both parts times the rounded reciprocal 1 / su)
template <typename T> __device__ __forceinline__ T div_scalar(T a, T su) { return div_rn(a, su); }
template <typename T> __device__ __forceinline__ cx<T> div_scalar(cx<T> a, T su) {
    const T rat = T(0), scl = div_rn(T(1), su);
    return mkc<T>(mul_rn(add_rn(a.x, mul_rn(a.y, rat)), scl), mul_rn(sub_rn(a.y, mul_rn(a.x, rat)), scl));
}
template <typename E, typename T>
__global__ void scale_div_kernel(E* __restrict__ x, int64_t total, T su) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
        x[i] = div_scalar(x[i], su);
}

// spectra of the :fft_simple route: H scaled by 1 / nfft, then every column's spectrum times H (the rank-1 transform pair
// of dspb200_conv_nd_exec scales and multiplies in the same order)
template <typename T>
__global__ void cl_scale_kernel(cx<T>* __restrict__ H, int64_t n, T scale) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        H[i] = cscale(H[i], scale);
}
template <typename T>
__global__ void cl_cmul_kernel(cx<T>* __restrict__ X, const cx<T>* __restrict__ H, int64_t nbins, int64_t ncols) {
    const int64_t total = nbins * ncols;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
        X[i] = cmul(X[i], H[i % nbins]);
}

int grid_rows(int64_t rows, int threads) {
    int64_t g = cdiv(rows, threads);
    const int64_t cap = (int64_t)device_sm_count() * 32;
    return (int)(g < 1 ? 1 : g > cap ? cap : g);
}
unsigned grid_cols(int64_t ncols) { return (unsigned)(ncols < 65535 ? ncols : 65535); }

// n x ncols column-major elements of esz bytes, every index and byte count inside DSPB200_INDEX_LIMIT
bool shape_ok(int64_t n, int64_t ncols, size_t esz) {
    if (n < 0 || ncols < 0 || n > DSPB200_INDEX_LIMIT || ncols > DSPB200_INDEX_LIMIT) return false;
    return ncols == 0 || n <= DSPB200_INDEX_LIMIT / ncols / (int64_t)esz;
}

template <typename E>
int extend_launch(const void* x, int64_t n, int64_t ncols, int64_t pad, void* ext, cudaStream_t st) {
    const int threads = 256;
    filtfilt_extend_kernel<E><<<dim3(grid_rows(n + 2 * pad, threads), grid_cols(ncols)), threads, 0, st>>>(
        (const E*)x, n, ncols, pad, (E*)ext);
    DSP_LAUNCH_OK();
    return DSPB200_OK;
}

template <typename T>
int peak_launch(const void* s, int64_t nres, int64_t ncols, int64_t center, int reversed, int64_t* delay, int* nanflag,
                cudaStream_t st) {
    int64_t cs = cdiv(nres, 32 * PEAK_THREADS);
    if (cs > PEAK_MAX_CLUSTER) cs = PEAK_MAX_CLUSTER;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)cs, grid_cols(ncols));
    cfg.blockDim = dim3(PEAK_THREADS);
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = (unsigned)cs;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    DSP_CUDA(cudaLaunchKernelEx(&cfg, xcorr_peak_kernel<T>, (const T*)s, nres, ncols, center, reversed, delay, nanflag));
    DSP_LAUNCH_OK();
    return DSPB200_OK;
}

template <typename E>
int shift_launch(const void* x, int64_t nx, int64_t ncols, int64_t shift, const int64_t* shifts, int negate, void* out,
                 int64_t nout, cudaStream_t st) {
    const int threads = 256;
    shift_kernel<E><<<dim3(grid_rows(nout, threads), grid_cols(ncols)), threads, 0, st>>>((const E*)x, nx, ncols, shift, shifts,
                                                                                        negate, (E*)out, nout);
    DSP_LAUNCH_OK();
    return DSPB200_OK;
}

template <typename E, typename T>
int scale_launch(void* x, int64_t total, double su, cudaStream_t st) {
    const int threads = 256;
    scale_div_kernel<E, T><<<grid_rows(total, threads), threads, 0, st>>>((E*)x, total, (T)su);
    DSP_LAUNCH_OK();
    return DSPB200_OK;
}

// conv of every column of u (nu x ncols) with v: one batched 1-D transform pair of nfft points over the columns (the rank-1
// _conv_kern_fft! of src/dspbase.jl:611-644 per column; no transform along the channels).  The caller holds the
// ConvenienceLock (cached plans, arena slots 3-5).
template <typename T, bool CPLX>
int fft_columns_queue(const void* d_u, int64_t nu, int64_t ncols, const void* d_v, int64_t nv, int64_t nfft, void* d_out,
                      cudaStream_t st) {
    using E = typename cl_elt<T, CPLX>::type;
    const bool f64 = sizeof(T) == 8;
    const int64_t nres = nu + nv - 1, nbins = CPLX ? nfft : nfft / 2 + 1;
    DevBuf &tu = scratch_buf(3), &fu = scratch_buf(4), &fv = scratch_buf(5);
    DSP_TRY(tu.reserve((size_t)(nfft * ncols) * sizeof(E)));
    DSP_TRY(fu.reserve((size_t)(nbins * ncols) * sizeof(cx<T>)));
    DSP_TRY(fv.reserve((size_t)nbins * sizeof(cx<T>)));
    const long long nn[1] = {(long long)nfft};
    const int tf = fft_type(CPLX, f64, CUFFT_FORWARD), ti = fft_type(CPLX, f64, CUFFT_INVERSE);
    int h1 = 0, hf = 0, hi = 0;
    DSP_TRY(plan_cache_get(&h1, 1, nn, false, 0, 0, tf, 1));
    DSP_TRY(plan_cache_get(&hf, 1, nn, false, 0, 0, tf, ncols));
    DSP_TRY(plan_cache_get(&hi, 1, nn, false, 0, 0, ti, ncols));
    const size_t esz = sizeof(E);
    // v zero-padded to nfft in column 0 of tu, transformed into fv; then the columns of u, zero-padded, into fu
    DSP_CUDA(cudaMemsetAsync(tu.p, 0, (size_t)nfft * esz, st));
    DSP_CUDA(cudaMemcpyAsync(tu.p, d_v, (size_t)nv * esz, cudaMemcpyDeviceToDevice, st));
    DSP_TRY(fft_exec((cufftHandle)h1, CPLX, f64, CUFFT_FORWARD, tu.p, fv.p, st));
    DSP_CUDA(cudaMemsetAsync(tu.p, 0, (size_t)(nfft * ncols) * esz, st));
    DSP_TRY(memcpy2d_dd(tu.p, (size_t)nfft * esz, d_u, (size_t)nu * esz, (size_t)nu * esz, (size_t)ncols, st));
    DSP_TRY(fft_exec((cufftHandle)hf, CPLX, f64, CUFFT_FORWARD, tu.p, fu.p, st));
    const int threads = 256;
    cl_scale_kernel<T><<<grid_rows(nbins, threads), threads, 0, st>>>((cx<T>*)fv.p, nbins, T(1) / (T)nfft);
    DSP_LAUNCH_OK();
    cl_cmul_kernel<T><<<grid_rows(nbins * ncols, threads), threads, 0, st>>>((cx<T>*)fu.p, (const cx<T>*)fv.p, nbins, ncols);
    DSP_LAUNCH_OK();
    DSP_TRY(fft_exec((cufftHandle)hi, CPLX, f64, CUFFT_INVERSE, fu.p, tu.p, st));
    DSP_TRY(memcpy2d_dd(d_out, (size_t)nres * esz, tu.p, (size_t)nfft * esz, (size_t)nres * esz, (size_t)ncols, st));
    return DSPB200_OK;
}

}  // namespace
}  // namespace dspb200

using namespace dspb200;

extern "C" {

int dspb200_filtfilt_extend_async(int dtype, const void* x, int64_t n, int64_t ncols, int64_t pad, void* ext, void* stream) {
    DSP_RANGE("dspb200_filtfilt_extend_async");
    DSP_REQUIRE(dtype_valid(dtype), "invalid dtype %d", dtype);
    const size_t esz = dtype_size(dtype);
    DSP_REQUIRE(pad >= 0 && pad <= DSPB200_INDEX_LIMIT / 4 && shape_ok(n, ncols, esz), "negative or oversized size");
    if (ncols == 0) return DSPB200_OK;
    DSP_REQUIRE(pad < n, "the extension needs pad < n (pad %lld, n %lld)", (long long)pad, (long long)n);
    DSP_REQUIRE(shape_ok(n + 2 * pad, ncols, esz), "oversized extension");
    DSP_REQUIRE(x && ext, "NULL argument");
    DSP_REQUIRE(!ranges_overlap(x, (size_t)(n * ncols) * esz, ext, (size_t)((n + 2 * pad) * ncols) * esz), "x and ext overlap");
    const cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case DSPB200_F32: return extend_launch<float>(x, n, ncols, pad, ext, st);
        case DSPB200_F64: return extend_launch<double>(x, n, ncols, pad, ext, st);
        case DSPB200_C32: return extend_launch<cx<float>>(x, n, ncols, pad, ext, st);
        default: return extend_launch<cx<double>>(x, n, ncols, pad, ext, st);
    }
}

int dspb200_xcorr_peak_async(int dtype, const void* s, int64_t nres, int64_t ncols, int64_t center, int reversed, int64_t* delay,
                             int* nanflag, void* stream) {
    DSP_RANGE("dspb200_xcorr_peak_async");
    DSP_REQUIRE(dtype_valid(dtype), "invalid dtype %d", dtype);
    DSP_REQUIRE(!dtype_is_cplx(dtype), "the peak search takes a real correlation (dtype %d)", dtype);
    const size_t esz = dtype_size(dtype);
    DSP_REQUIRE(shape_ok(nres, ncols, esz) && index_in_domain(center), "negative or oversized size");
    if (ncols == 0) return DSPB200_OK;
    DSP_REQUIRE(nres >= 1, "empty correlation");
    DSP_REQUIRE(s && delay && nanflag, "NULL argument");
    const size_t sbytes = (size_t)(nres * ncols) * esz;
    DSP_REQUIRE(!ranges_overlap(s, sbytes, delay, (size_t)ncols * 8) && !ranges_overlap(s, sbytes, nanflag, (size_t)ncols * 4) &&
                    !ranges_overlap(delay, (size_t)ncols * 8, nanflag, (size_t)ncols * 4),
                "output buffers overlap");
    const cudaStream_t st = (cudaStream_t)stream;
    if (dtype == DSPB200_F32) return peak_launch<float>(s, nres, ncols, center, reversed ? 1 : 0, delay, nanflag, st);
    return peak_launch<double>(s, nres, ncols, center, reversed ? 1 : 0, delay, nanflag, st);
}

int dspb200_shift_async(int dtype, const void* x, int64_t nx, int64_t ncols, int64_t shift, const int64_t* shifts, int negate,
                        void* out, int64_t nout, void* stream) {
    DSP_RANGE("dspb200_shift_async");
    DSP_REQUIRE(dtype_valid(dtype), "invalid dtype %d", dtype);
    const size_t esz = dtype_size(dtype);
    DSP_REQUIRE(shape_ok(nx, ncols, esz) && shape_ok(nout, ncols, esz), "negative or oversized size");
    DSP_REQUIRE(shifts || (shift >= -nx && shift <= nx), "|shift| %lld exceeds the column length %lld", (long long)shift,
                (long long)nx);
    if (ncols == 0 || nout == 0) return DSPB200_OK;
    DSP_REQUIRE(out && (x || nx == 0), "NULL argument");
    DSP_REQUIRE(!ranges_overlap(x, (size_t)(nx * ncols) * esz, out, (size_t)(nout * ncols) * esz), "x and out overlap");
    DSP_REQUIRE(!ranges_overlap(shifts, (size_t)ncols * 8, out, (size_t)(nout * ncols) * esz), "shifts and out overlap");
    const cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case DSPB200_F32: return shift_launch<float>(x, nx, ncols, shift, shifts, negate, out, nout, st);
        case DSPB200_F64: return shift_launch<double>(x, nx, ncols, shift, shifts, negate, out, nout, st);
        case DSPB200_C32: return shift_launch<cx<float>>(x, nx, ncols, shift, shifts, negate, out, nout, st);
        default: return shift_launch<cx<double>>(x, nx, ncols, shift, shifts, negate, out, nout, st);
    }
}

int dspb200_scale_div_async(int dtype, void* x, int64_t n, double divisor, void* stream) {
    DSP_RANGE("dspb200_scale_div_async");
    DSP_REQUIRE(dtype_valid(dtype), "invalid dtype %d", dtype);
    DSP_REQUIRE(shape_ok(n, 1, dtype_size(dtype)), "negative or oversized size");
    if (n == 0) return DSPB200_OK;
    DSP_REQUIRE(x != nullptr, "NULL argument");
    const cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case DSPB200_F32: return scale_launch<float, float>(x, n, divisor, st);
        case DSPB200_F64: return scale_launch<double, double>(x, n, divisor, st);
        case DSPB200_C32: return scale_launch<cx<float>, float>(x, n, divisor, st);
        default: return scale_launch<cx<double>, double>(x, n, divisor, st);
    }
}

int dspb200_conv_fft_columns(int dtype, const void* d_u, int64_t nu, int64_t ncols, const void* d_v, int64_t nv, int64_t nfft,
                             void* d_out, void* stream) {
    DSP_RANGE("dspb200_conv_fft_columns");
    DSP_REQUIRE(dtype_valid(dtype), "invalid dtype %d", dtype);
    const size_t esz = dtype_size(dtype);
    DSP_REQUIRE(shape_ok(nu, ncols, esz) && nv >= 0 && nfft >= 0 && shape_ok(nfft, ncols, 16), "negative or oversized size");
    if (ncols == 0) return DSPB200_OK;
    DSP_REQUIRE(nu >= 1 && nv >= 1, "empty input");
    DSP_REQUIRE(nfft >= nu + nv - 1 && nfft < (int64_t(1) << 31), "nfft must cover the full output");
    DSP_REQUIRE(d_u && d_v && d_out, "NULL argument");
    const size_t obytes = (size_t)((nu + nv - 1) * ncols) * esz;
    DSP_REQUIRE(!ranges_overlap(d_u, (size_t)(nu * ncols) * esz, d_out, obytes) && !ranges_overlap(d_v, (size_t)nv * esz, d_out, obytes),
                "an input overlaps out");
    return convenience_call((cudaStream_t)stream, [&](cudaStream_t st) {
        switch (dtype) {
            case DSPB200_F32: return fft_columns_queue<float, false>(d_u, nu, ncols, d_v, nv, nfft, d_out, st);
            case DSPB200_F64: return fft_columns_queue<double, false>(d_u, nu, ncols, d_v, nv, nfft, d_out, st);
            case DSPB200_C32: return fft_columns_queue<float, true>(d_u, nu, ncols, d_v, nv, nfft, d_out, st);
            default: return fft_columns_queue<double, true>(d_u, nu, ncols, d_v, nv, nfft, d_out, st);
        }
    });
}

}  // extern "C"
