/* dspb200.h -- C ABI of libdspb200.so: the H100-native (sm_90a) implementation of DSP.jl's
 * data-parallel hot path.  Plain pointers and sizes only; callable from Julia `ccall`, Python `ctypes`, C.
 *
 * Each entry point names the reference interface it replaces (paths relative to the DSP.jl tree,
 * v0.8.5 @ 2d57c27).  The reference has no FFI of its own: its only native boundary is FFTW.jl's plan
 * API called from src/dspbase.jl, src/Filters/filt.jl, src/Filters/stream_filt.jl, src/periodograms.jl.
 * This library replaces those FFTW calls *and* the Julia inner loops around them.
 *
 * Conventions
 *  - every function returns a status (DSPB200_OK == 0, negative on error) and never throws/aborts;
 *    dspb200_last_error() returns a thread-local message for the last failure.
 *  - dtype: element type of the signal (DSPB200_F32/F64/C32/C64); complex = interleaved (re, im),
 *    the memory layout of Julia's Complex{T}.  Arrays are column-major: dim 1 is time, every column
 *    is an independent channel (src/dspbase.jl:55, src/Filters/filt.jl:504).
 *  - `*_exec`     : HOST pointers (caller-owned, never retained); copies in, computes on the GPU, copies
 *                   out; synchronous on return.  Pinned host memory (dspb200_host_alloc) is streamed in
 *                   chunks so copies overlap compute.
 *  - `*_exec_dev` : DEVICE pointers; enqueued on `stream` (a cudaStream_t, NULL = default stream);
 *                   asynchronous: every launch and copy goes to `stream`, and the call returns without waiting for it.
 *                   The plan-less _dev calls (conv_nd, conv_nd_os, hilbert, periodogram2) and the multitaper ones
 *                   (mt_*) are the exception: they return after the work on that stream has completed.
 *  - the asynchronous _dev calls may be captured in a CUDA graph (stream capture on `stream`) once a call with the same
 *    plan, shapes and pointers has run outside the capture, which sizes the plan's scratch; the graph replays the call
 *    with the arguments it was captured with.  dspb200_welch_begin_dev / _accumulate_dev / _finalize_dev keep host
 *    state between calls, so the three are captured together, in one graph.
 *  - plans own device scratch, twiddle tables and cuFFT plans; one caller at a time per plan (the
 *    reference's WelchConfig / FIRFilter / ArraySplit scratch is equally non-reentrant:
 *    src/periodograms.jl:88-90,525-526; src/Filters/stream_filt.jl:137-142).
 *  - there is no CPU fallback: without a CUDA device every exec call fails with DSPB200_ECUDA.
 */
#ifndef DSPB200_H
#define DSPB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DSPB200_VERSION 100

#if defined(__GNUC__)
#define DSPB200_API __attribute__((visibility("default")))
#else
#define DSPB200_API
#endif

enum { DSPB200_F32 = 0, DSPB200_F64 = 1, DSPB200_C32 = 2, DSPB200_C64 = 3 };

enum {
    DSPB200_OK = 0,
    DSPB200_EINVALID = -1,      /* argument check failed (the Julia glue raises the reference's exception types first) */
    DSPB200_ECUDA = -2,         /* CUDA runtime error / no device */
    DSPB200_ECUFFT = -3,        /* cuFFT error (generic-size path) */
    DSPB200_ENOMEM = -4,        /* device or pinned-host allocation failed */
    DSPB200_EUNSUPPORTED = -5   /* combination outside the hot-path scope */
};

/* ------------------------------------------------------------------------------------------ runtime */
DSPB200_API int dspb200_version(void);
DSPB200_API const char* dspb200_last_error(void);
DSPB200_API int dspb200_device_count(int* count);
DSPB200_API int dspb200_set_device(int device);                 /* device used by plans created afterwards on this thread */
DSPB200_API int dspb200_device_info(int* sm_count, int* cc_major, int* cc_minor, size_t* total_mem, size_t* l2_bytes);
DSPB200_API int dspb200_malloc(void** dptr, size_t bytes);      /* device memory, for hosts without a CUDA binding */
DSPB200_API int dspb200_free(void* dptr);
DSPB200_API int dspb200_host_alloc(void** hptr, size_t bytes);  /* pinned host memory */
DSPB200_API int dspb200_host_free(void* hptr);
DSPB200_API int dspb200_memcpy_h2d(void* dst, const void* src, size_t bytes, void* stream);
DSPB200_API int dspb200_memcpy_d2h(void* dst, const void* src, size_t bytes, void* stream);
/* height rows of width bytes, row r at src + r*spitch -> dst + r*dpitch, device to device, enqueued on `stream` (cropping
 * the columns of a column-major matrix: one row per column).  Pitches past the device's limit for 2-D copies (about 2 GiB)
 * are copied row by row, so any column length within DSPB200_INDEX_LIMIT works. */
DSPB200_API int dspb200_memcpy2d_d2d(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t height,
                                     void* stream);
DSPB200_API int dspb200_stream_sync(void* stream);

/* Number of kernels this library has launched in this process (bench.py's `gpu_launches`). */
DSPB200_API int64_t dspb200_launch_count(void);

/* Index domain of the range forms (dspb200_os_exec_range_dev, dspb200_resample_exec_range_dev,
 * dspb200_welch_exec_range_dev, dspb200_welch_accumulate_dev).  Their offsets are global sample indices of one long
 * stream, so they may be far larger than the buffers passed with them.  The kernels form differences of two such
 * indices (the local position of a global sample) in int64_t, so every global index a call names must lie within
 * +-DSPB200_INDEX_LIMIT, and the polyphase phase phi0 + j*decim within DSPB200_PHASE_LIMIT; then every sample, output and
 * phase index the kernels compute stays representable in int64_t.  (Pointers formed from such an index to a sample that is
 * not stored are never dereferenced.)  Calls outside return DSPB200_EINVALID before any launch. */
#define DSPB200_INDEX_LIMIT ((int64_t)1 << 61)
#define DSPB200_PHASE_LIMIT ((int64_t)1 << 62)

/* ------------------------------------------------------------------------------------------ FIR, time domain
 * filt(b, 1, x) / filt!(out, b, 1, x) / tdfilt(h, x): src/dspbase.jl:14-15, 26-66, 95-154;
 * src/Filters/filt.jl:431-443.  y[i] = sum_k b[k] x[i-k+1] per column, evaluated with the reference's
 * accumulation order (oldest tap first, one fused multiply-add per tap).  b, x and y share `dtype`
 * (the host promotes, src/dspbase.jl:15); b is normalised by a[1] on the host (src/dspbase.jl:43-47). */
typedef struct dspb200_fir_plan dspb200_fir_plan;
DSPB200_API int dspb200_fir_plan_create(dspb200_fir_plan** plan, int dtype, const void* b_host, int64_t nb);
DSPB200_API int dspb200_fir_exec(dspb200_fir_plan* plan, const void* x, int64_t nx, int64_t ncols, void* out);
DSPB200_API int dspb200_fir_exec_dev(dspb200_fir_plan* plan, const void* x, int64_t nx, int64_t ncols, void* out, void* stream);
/* Stateful FIR: filt!(out, DF2TFilter(PolynomialRatio(b, 1), si), x) and the deprecated filt(b, 1, x, si)
 * (src/Filters/filt.jl:157-181, src/deprecated.jl:80-101).  si_in / si_out hold the transposed direct-form state,
 * (nb-1) x ncols column-major in the plan's dtype: si_in is the state before x, si_out receives the state after it,
 * so feeding si_out to the next call filters a chunked stream bit-identically to one call over the whole stream.
 * si_in == NULL means a zero state, si_out == NULL discards the final state.  nx == 0 passes the state through;
 * nb == 1 has no state and computes out = x * b[1].  The _dev form takes device pointers, enqueues one kernel on
 * `stream` and returns; there no two of x, out, si_in and si_out may overlap where one of them is written (x with out,
 * si_in with si_out, a state buffer with x or out): DSPB200_EINVALID, because CTAs read the samples and state of their
 * neighbours' outputs.  The host form stages x and the state through plan scratch, so there out may be x (in-place
 * filtering, as filt!(out, f, x) allows) and si_out may be si_in.  (dspb200_fir_exec_dev has the same restriction on
 * x and out; it is not checked there.) */
DSPB200_API int dspb200_fir_exec_state(dspb200_fir_plan* plan, const void* x, int64_t nx, int64_t ncols, const void* si_in,
                                       void* si_out, void* out);
DSPB200_API int dspb200_fir_exec_state_dev(dspb200_fir_plan* plan, const void* x, int64_t nx, int64_t ncols, const void* si_in,
                                           void* si_out, void* out, void* stream);
DSPB200_API int dspb200_fir_plan_destroy(dspb200_fir_plan* plan);

/* ------------------------------------------------------------------------------------------ overlap-save
 * conv(u, v; algorithm=:fft_overlapsave) / unsafe_conv_kern_os! (src/dspbase.jl:490-609, 299-356) and
 * fftfilt / _fftfilt! / filt(b, x) (src/Filters/filt.jl:458-555).
 * out[m] = sum_j u[j] v[m-j], m = 0 .. nout-1, per column; nout = nu for fftfilt/filt (src/Filters/filt.jl:517),
 * nout = nu+nv-1 for conv; samples of `out` beyond nu+nv-1 are zero-filled (src/dspbase.jl:733-735).
 * u, v and out share `dtype` (real: two blocks ride one complex FFT; complex: one block per FFT).
 * nfft: 0 = library choice (largest shared-memory transform that amortises the nv-1 halo; the reference's
 *       optimalfftfiltlength, src/dspbase.jl:268-291, is a CPU cost model -- any nfft >= nv gives the same
 *       convolution); otherwise a power of two in [32, 16384] (F64/C64: 8192) runs the fused kernel and
 *       any other value >= nv runs gather -> cuFFT -> multiply -> cuFFT -> scatter. */
typedef struct dspb200_os_plan dspb200_os_plan;
DSPB200_API int dspb200_os_plan_create(dspb200_os_plan** plan, int dtype, const void* v_host, int64_t nv, int64_t nfft);
DSPB200_API int dspb200_os_plan_nfft(const dspb200_os_plan* plan, int64_t* nfft, int* fused);
DSPB200_API int dspb200_os_plan_geometry(const dspb200_os_plan* plan, int* dtype, int64_t* nv, int64_t* nfft);
DSPB200_API int dspb200_os_exec(dspb200_os_plan* plan, const void* u, int64_t nu, int64_t ncols, void* out, int64_t nout);
DSPB200_API int dspb200_os_exec_dev(dspb200_os_plan* plan, const void* u, int64_t nu, int64_t ncols, void* out, int64_t nout,
                        void* stream);
/* Range form for sharding one long column across GPUs (SURVEY.md 8e): compute outputs
 * [out_begin, out_begin+out_count) of the convolution of the virtual signal whose samples
 * [u_begin, u_begin+nu_local) are stored at `u_local` (everything outside is zero).  No collective.
 * Domain (DSPB200_INDEX_LIMIT = 2^61): 0 <= out_begin, 0 <= out_count, 0 <= nu_local, |u_begin| <= 2^61,
 * out_begin + out_count <= 2^61 and u_begin + nu_local <= 2^61; otherwise DSPB200_EINVALID before any launch.
 * Outputs that no stored sample reaches are transformed like the others: they are zero, of either sign. */
DSPB200_API int dspb200_os_exec_range_dev(dspb200_os_plan* plan, const void* u_local, int64_t u_begin, int64_t nu_local,
                              void* out_local, int64_t out_begin, int64_t out_count, void* stream);
/* Stateful overlap-save: fftfilt(f::DF2TFilter, x) / fftfilt!(out, f::DF2TFilter, x), the overlap-save counterpart of
 * dspb200_fir_exec_state with the same state: si_in / si_out hold the transposed direct-form FIR state, (nv-1) x ncols
 * column-major in the plan's dtype.  Per column, with full = conv(v, x) (nx + nv - 1 outputs), full[i] += si_in[i] for
 * i < nv-1, out = full[0 .. nx-1] and si_out = full[nx .. nx+nv-2]; so a chunked stream fed back its si_out equals the
 * stateful FIR filter within FFT rounding, and the two entry points may alternate on one state.  si_in == NULL means a zero
 * state, si_out == NULL discards the final state.  nx == 0 passes the state through; nv == 1 has no state.  Takes plans made
 * with nfft = 0 (a fused plan with nfft < 1024 gives DSPB200_EUNSUPPORTED).  The _dev form takes device pointers, enqueues
 * one kernel on `stream` (fused sizes; the generic path launches per column) and returns; there no two of x, out, si_in and
 * si_out may overlap where one of them is written (x with out, si_in with si_out, a state buffer with x or out):
 * DSPB200_EINVALID before any launch, because a column's first unit reads si_in while its last units write si_out, and
 * units read the samples behind their neighbours' outputs.  The host form stages x and the state through plan scratch, so
 * there out may be x and si_out may be si_in. */
DSPB200_API int dspb200_os_exec_state(dspb200_os_plan* plan, const void* x, int64_t nx, int64_t ncols, const void* si_in,
                                      void* si_out, void* out);
DSPB200_API int dspb200_os_exec_state_dev(dspb200_os_plan* plan, const void* x, int64_t nx, int64_t ncols, const void* si_in,
                                          void* si_out, void* out, void* stream);
DSPB200_API int dspb200_os_plan_destroy(dspb200_os_plan* plan);

/* conv(u, v; algorithm=:fft_simple) / _conv_kern_fft!: src/dspbase.jl:611-644 -- one FFT pair of size
 * nfft >= nu+nv-1 (the host passes nextfastfft(nu+nv-1), src/util.jl:134); out has nu+nv-1 samples. */
DSPB200_API int dspb200_conv_fft_exec(int dtype, const void* u, int64_t nu, const void* v, int64_t nv, int64_t nfft, void* out);
/* conv(u, v; algorithm=:direct) / _conv_td!: src/dspbase.jl:646-660 -- direct muladd convolution in the reference's order:
 * each output sums its products in ascending index of the shorter of u and v (u when nu == nv), each one
 * muladd(u[m], v[n], acc), so the result is bit-identical to the reference's loop on FMA hardware. */
DSPB200_API int dspb200_conv_direct_exec(int dtype, const void* u, int64_t nu, const void* v, int64_t nv, void* out);

/* conv(u, v; algorithm) for matrices and rank-3 arrays: src/dspbase.jl:611-660 (_conv_kern_fft!, _conv_td!), 709-757.
 * Column-major arrays of `rank` <= 3 dimensions, sizes usize / vsize; out has usize + vsize - 1 per dimension.
 * nffts != NULL: one N-D FFT pair of size nffts (the host passes nextfastfft.(usize .+ vsize .- 1), :618, :632);
 * nffts == NULL: direct muladd convolution (:646-660).  The _dev forms take device pointers and a cudaStream_t and return
 * after the work on that stream has completed (plans and scratch come from the library's cache). */
DSPB200_API int dspb200_conv_nd_exec(int dtype, int rank, const int64_t* usize, const void* u, const int64_t* vsize, const void* v,
                                     const int64_t* nffts, void* out);
DSPB200_API int dspb200_conv_nd_exec_dev(int dtype, int rank, const int64_t* usize, const void* d_u, const int64_t* vsize,
                                         const void* d_v, const int64_t* nffts, void* d_out, void* stream);
/* conv(u, v; algorithm=:fft_overlapsave) for arrays of rank <= 3: unsafe_conv_kern_os! with its perimeter blocks
 * unsafe_conv_kern_os_edge!, src/dspbase.jl:371-609.  u is the array with more elements (:746-751); nffts[d] >= vsize[d] is
 * the block transform per dimension (the host passes optimalfftfiltlength.(vsize, usize), :736); every block contributes
 * save_blocksize = nffts - vsize + 1 outputs per dimension (:500-506).  Blocks are gathered (zero outside u), transformed
 * by ONE batched N-D cuFFT plan, multiplied by the filter spectrum and scattered, as many per batch as fit the block-buffer
 * budget (default 1 GiB; dspb200_conv_nd_os_set_budget) -- so arrays whose single transform would not fit are convolved
 * in bounded memory, which is what the reference's blocking is for.  The _dev form takes device pointers and a cudaStream_t
 * and returns after the work on that stream has completed. */
DSPB200_API int dspb200_conv_nd_os_exec(int dtype, int rank, const int64_t* usize, const void* u, const int64_t* vsize, const void* v,
                                        const int64_t* nffts, void* out);
DSPB200_API int dspb200_conv_nd_os_exec_dev(int dtype, int rank, const int64_t* usize, const void* d_u, const int64_t* vsize,
                                            const void* d_v, const int64_t* nffts, void* d_out, void* stream);
DSPB200_API int dspb200_conv_nd_os_set_budget(size_t bytes);
/* hilbert(x): src/util.jl:31-75 -- analytic signal of a real [n x ncols] column-major array along dim 1 (rfft, bins
 * 2 .. n/2+isodd(n) doubled, the rest of the negative half zero, normalised inverse FFT).  dtype F32 -> ComplexF32 out,
 * F64 -> ComplexF64 (integers are converted by the host, src/util.jl:43).  Any n (cuFFT).  The _dev form takes device
 * pointers and a cudaStream_t and returns after the work on that stream has completed. */
DSPB200_API int dspb200_hilbert_exec(int dtype, const void* x, int64_t n, int64_t ncols, void* out);
DSPB200_API int dspb200_hilbert_exec_dev(int dtype, const void* d_x, int64_t n, int64_t ncols, void* d_out, void* stream);

/* ------------------------------------------------------------------------------------------ xcorr / filtfilt / finddelay
 * The device work of xcorr, FIR filtfilt, finddelay, shiftsignal and alignsignals (src/dspbase.jl:867-898,
 * src/util.jl:336-427, src/Filters/filt.jl:245-259, 301-337) that surrounds the filter and correlation calls above.  The
 * *_async calls follow the conventions of the asynchronous _dev calls: device pointers, every launch on `stream`, no
 * synchronisation, capturable in a CUDA graph.  Matrices are column-major, one channel per column.  DSPB200_EINVALID,
 * before any launch: a NULL buffer, a negative size, an output overlapping an input, a size past DSPB200_INDEX_LIMIT.
 * ncols == 0 (and nout == 0, n == 0 where they are sizes of the output) launches nothing.  Each call is one launch. */
/* extrapolate_signal! (src/Filters/filt.jl:245-259): column c of ext ((n + 2 pad) x ncols) is the odd-symmetric extension
 * [2x[0] - x[pad..1]; x; 2x[n-1] - x[n-2..n-1-pad]] of column c of x (n x ncols), each sample rounded in dtype as the
 * host computes it.  pad >= n gives DSPB200_EINVALID. */
DSPB200_API int dspb200_filtfilt_extend_async(int dtype, const void* x, int64_t n, int64_t ncols, int64_t pad, void* ext,
                                              void* stream);
/* finddelay's peak (src/util.jl:360-368) of every column of the real correlation s (nres x ncols, F32 or F64): among the
 * samples of largest |s| the one closest to `center` (1-based index), the lower one on a tie; delay[c] = center - index.
 * Exact comparisons, no floating-point atomics: the result does not depend on the launch.  nanflag[c] = 1 when the column
 * holds a NaN (the reference throws; delay[c] is then meaningless), else 0.  reversed != 0: sample p of a column stands at
 * index nres - 1 - p (xcorr(y, x) stored as xcorr(x, y)).  One cluster of up to 8 CTAs per column.  Complex dtypes give
 * DSPB200_EINVALID; nres == 0 with ncols > 0 too. */
DSPB200_API int dspb200_xcorr_peak_async(int dtype, const void* s, int64_t nres, int64_t ncols, int64_t center, int reversed,
                                         int64_t* delay, int* nanflag, void* stream);
/* shiftsignal (src/util.jl:379-412), out of place: out[i, c] = x[i - s_c, c] where 0 <= i - s_c < nx, else zero, for
 * i < nout (nout == nx: shiftsignal; nout > nx with s = 0: zero padding).  s_c = shifts[c] (device int64, negated when
 * negate != 0: alignsignals' -delay) when shifts != NULL, else `shift`, which must satisfy |shift| <= nx. */
DSPB200_API int dspb200_shift_async(int dtype, const void* x, int64_t nx, int64_t ncols, int64_t shift, const int64_t* shifts,
                                    int negate, void* out, int64_t nout, void* stream);
/* xcorr's :biased scaling, in place: x[i] / divisor in dtype for i < n, as numpy divides by a Python integer (a complex
 * sample times the rounded reciprocal of divisor + 0im, as Smith's division does with a zero imaginary part). */
DSPB200_API int dspb200_scale_div_async(int dtype, void* x, int64_t n, double divisor, void* stream);
/* conv(u[:, c], v; algorithm=:fft_simple) for every column of u (nu x ncols) with one vector v (nv): one batched 1-D transform
 * pair of nfft >= nu + nv - 1 points over the columns (no transform along the channels); out is (nu + nv - 1) x ncols.  Device
 * pointers; like the plan-less _dev calls it uses the cached plans and returns after the work on `stream` has completed.
 * Five launches whatever ncols. */
DSPB200_API int dspb200_conv_fft_columns(int dtype, const void* d_u, int64_t nu, int64_t ncols, const void* d_v, int64_t nv,
                                         int64_t nfft, void* d_out, void* stream);

/* ------------------------------------------------------------------------------------------ linear prediction
 * arburg / lpc / levinson (src/lpc.jl) of every column of an n x ncols column-major matrix.  The *_async conventions above:
 * device pointers, every launch on `stream`, no synchronisation, capturable in a CUDA graph.  Outputs: a, err (ncols, in the
 * real eltype: F32 for F32 and C32) and refl (NULL: not wanted), in dtype, one column per input column.
 * Everything but the reductions follows src/lpc.jl operation by operation in dtype (muladd = one fma for reals, Base.muladd
 * for complex; every other operation rounded).  The reductions dot(x, x), dot(eb, ef) and the autocorrelation lags run in
 * one fixed order that depends only on their length: tiles of 1024 indices, in a tile 256 lanes (index i in lane i % 256)
 * each a muladd chain in increasing index from +0, then lanes l + h into l for h = 16 .. 1 inside each warp and warps
 * w + h into w for h = 4, 2, 1; tile sums added pairwise, adjacent first, an odd last one carried.  dot(x, x) is the real
 * sum of |x_i|^2 (fma(re, re, .), then fma(im, im, .)).  The result does not depend on ncols, the column's position, the
 * path or the stream.
 * DSPB200_EINVALID, before any launch: a NULL required buffer, a negative size, p outside the call's range, an output
 * overlapping an input, the workspace or another output, a size past DSPB200_INDEX_LIMIT.  p > 1024 (LPC_P_MAX):
 * DSPB200_EUNSUPPORTED.  ncols == 0 launches nothing. */
/* Bytes of `work` for dspb200_lpc_burg_async (method 0, with its pin) or dspb200_lpc_levinson_async (method 1). */
DSPB200_API int dspb200_lpc_work_bytes(int dtype, int64_t n, int64_t ncols, int64_t p, int method, int pin, int64_t* bytes);
/* arburg(x, p), 0 <= p <= n: a is (p + 1) x ncols with a[0] = 1, conjugated as arburg returns it; lpc(x, p, LPCBurg()) is
 * rows 1 .. p.  One launch.  Path, from n alone: one CTA per column with the errors in shared memory when
 * 4 n sizeof(dtype) <= 192 KiB, else a cluster of min(8, ceil(n / 65536)) CTAs per column with the errors in `work` (one
 * HBM pass and one cluster barrier per order).  pin is a testing aid: 0 the rule above, -1 the shared-memory path
 * (DSPB200_EUNSUPPORTED where it does not fit), 1 .. 8 the streamed path with that many CTAs per column. */
DSPB200_API int dspb200_lpc_burg_async(int dtype, const void* x, int64_t n, int64_t ncols, int64_t p, void* a, void* err,
                                       void* refl, void* work, int pin, void* stream);
/* lpc(x, p, LPCLevinson()), 1 <= p <= n - 1: the biased autocorrelation at lags 0 .. p as a direct sum
 * r[k] = sum_i x[i + k] conj(x[i]) (the order above) divided by n as dspb200_scale_div_async divides, then levinson.  a and
 * refl are p x ncols.  Two launches. */
DSPB200_API int dspb200_lpc_levinson_async(int dtype, const void* x, int64_t n, int64_t ncols, int64_t p, void* a, void* err,
                                           void* refl, void* work, void* stream);
/* levinson(r, p) of every column of r (nr x ncols), 1 <= p <= nr - 1; a and refl are p x ncols.  dotu is the in-order
 * muladd chain; the first k of a complex r is Smith's division.  One launch. */
DSPB200_API int dspb200_levinson_async(int dtype, const void* r, int64_t nr, int64_t ncols, int64_t p, void* a, void* err,
                                       void* refl, void* stream);

/* ------------------------------------------------------------------------------------------ Welch / STFT
 * One plan per (dtype, n, noverlap, nfft, onesided, window): the analogue of WelchConfig
 * (src/periodograms.jl:516-576) = ArraySplit segmenter (:32-73) + forward_plan (:511-514) + fft2pow! (:142-172)
 * + fft2oneortwosided! (:234-244).  `window`: n Float64 values or NULL for `nothing` (:248-257; the sample *
 * window product is formed in Float64 and rounded to the buffer eltype, :66).  Power-of-two nfft in
 * [32, 16384] (F64/C64: 8192) runs fused shared-memory kernels; other sizes use cuFFT. */
typedef struct dspb200_spec_plan dspb200_spec_plan;
DSPB200_API int dspb200_spec_plan_create(dspb200_spec_plan** plan, int dtype, int64_t n, int64_t noverlap, int64_t nfft,
                             int onesided, const double* window_host);
DSPB200_API int dspb200_spec_plan_info(const dspb200_spec_plan* plan, int64_t* nout, int* fused);
DSPB200_API int dspb200_spec_plan_geometry(const dspb200_spec_plan* plan, int* dtype, int64_t* n, int64_t* hop, int64_t* nout);
DSPB200_API int64_t dspb200_spec_nsegments(const dspb200_spec_plan* plan, int64_t len);   /* k, src/periodograms.jl:49-50 */

/* welch_pgram / welch_pgram! / welch_pgram_helper!: src/periodograms.jl:647-759.
 * out[nout] (real eltype of dtype) = sum over segments of fft2pow!(.., r, onesided) with r = k*fs*norm2 (:751).
 * periodogram (:393-417) is the k = 1 case (n = length(s)). */
DSPB200_API int dspb200_welch_exec(dspb200_spec_plan* plan, const void* s, int64_t len, double r, void* out);
DSPB200_API int dspb200_welch_exec_dev(dspb200_spec_plan* plan, const void* s, int64_t len, double r, void* out, void* stream);
/* Batched welch_pgram (an extension: the reference's welch_pgram takes a vector): `s` is a column-major len x nchan matrix
 * whose columns are independent signals, each Welch-averaged with the plan's configuration; out is nout x nchan (real
 * eltype of dtype, column c = channel c).  r = k*fs*norm2 is the same for every column.  k == 0 writes zeros; nchan == 0
 * returns at once; negative sizes give DSPB200_EINVALID.  Power-of-two fused sizes run every channel in one launch over
 * (channel, slice) work items, with partial rows in scratch of the plan's own, at most 32 MiB (more channels run in groups);
 * cuFFT sizes run channel by channel.  The batch does not touch the accumulator of dspb200_welch_begin_dev /
 * dspb200_welch_accumulate_dev, so a streaming accumulation open on the plan may continue after it (in stream order).
 * The _dev form takes device pointers and a cudaStream_t and returns without synchronising; the host form copies `s` in
 * and `out` back and returns when done. */
DSPB200_API int dspb200_welch_batch_exec(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t nchan, double r, void* out);
DSPB200_API int dspb200_welch_batch_exec_dev(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t nchan, double r,
                                             void* out, void* stream);
/* Segment-range form for multi-GPU sharding: accumulates only segments [seg_begin, seg_end) of the signal
 * whose sample `sample_offset` is s[0]; the caller sums the partial spectra (NCCL all-reduce, SURVEY.md 8e).
 * Domain (also of dspb200_welch_accumulate_dev; DSPB200_INDEX_LIMIT = 2^61): 0 <= len, |sample_offset| <= 2^61,
 * sample_offset + len <= 2^61, 0 <= seg_begin <= seg_end and, for a non-empty range, (seg_end - 1) * hop + n <= 2^61;
 * otherwise DSPB200_EINVALID before any launch. */
DSPB200_API int dspb200_welch_exec_range_dev(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t sample_offset,
                                 int64_t seg_begin, int64_t seg_end, double r, void* out, void* stream);

/* Streaming form of welch_pgram_helper! (src/periodograms.jl:746-759): begin zeroes the accumulator, accumulate adds the
 * segments [seg_begin, seg_end) found in a buffer whose first sample is `sample_offset` (any number of calls, any chunking),
 * finalize applies the fft2pow! scaling with r = k*fs*norm2 and writes out[nout]. */
DSPB200_API int dspb200_welch_begin_dev(dspb200_spec_plan* plan, void* stream);
DSPB200_API int dspb200_welch_accumulate_dev(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t sample_offset,
                                 int64_t seg_begin, int64_t seg_end, void* stream);
DSPB200_API int dspb200_welch_finalize_dev(dspb200_spec_plan* plan, double r, void* out, void* stream);
/* Testing aid: pin the fused Welch launch configuration of `plan` (batched = 0: the single-signal kernel of the calls above,
 * 1: the batched kernel of dspb200_welch_batch_exec(_dev)).  Each plan picks, per alignment class, one instance of
 * MODE (0 direct loads, 1 TMA staging, 2 TMA + window in shared memory, 3 TMA + window in registers) x G (thread groups
 * per CTA, 1..3) on its first call; pinning replaces that choice, so that a test can run every instance on the same data.
 * A pinned TMA mode (1-3) applies to calls whose segments are 16-byte aligned; the others run MODE 0, G = 1.
 * mode < 0 unpins (the next call selects as before).  vctas > 0 fixes the number of virtual CTAs (CTAs x G; the grid is
 * vctas / groups, and need not fit one resident wave), 0 keeps the occupancy-derived grid; in the batched form it replaces
 * the resident virtual-CTA count the channels are sliced for.  DSPB200_EUNSUPPORTED: not a fused plan, no such instance
 * for the plan's (dtype, nfft), or its shared memory exceeds the opt-in limit for the plan's n and hop.
 * DSPB200_EINVALID: vctas < 0 or not a multiple of groups, or more virtual CTAs than the plan has partial rows
 * (single-signal form).  On a multitaper plan, batched = 1 also pins the taper-row instance of that MODE 0 or 1 and G that
 * dspb200_mt_pgram(_batch)_exec(_dev) runs at fused sizes (MODE 2 / 3 hold one window and have none: those calls then
 * select their own).  Pinning does not change what is computed, only which instance and grid compute it. */
DSPB200_API int dspb200_spec_plan_pin_welch(dspb200_spec_plan* plan, int batched, int mode, int groups, int64_t vctas);
/* The configuration the last fused Welch call of the given form (batched = 2: the mt_pgram calls of a multitaper plan) and
 * alignment class (0 unaligned, 1 aligned) used:
 * mode, groups and virtual CTAs of its launch.  *groups = 0 (mode -1, vctas 0) when no such call has run since the plan
 * was created or last pinned / unpinned. */
DSPB200_API int dspb200_spec_plan_welch_config(const dspb200_spec_plan* plan, int batched, int aligned, int* mode, int* groups,
                                               int64_t* vctas);
/* welch_pgram(filt(b, x), config) as ONE host-pointer call (src/dspbase.jl:14-15 + src/periodograms.jl:702-759): x[n] on the
 * host (pinned memory lets the copies overlap), out[nout] on the host.  The stream goes through the GPU in chunks: the H2D copy
 * of chunk c+1 overlaps the overlap-save convolution of chunk c (os plan: taps b, dtype of x) and the Welch accumulation of
 * the segments chunk c completes; the filter output y = (b * x)[0:n] stays in HBM.  r = k*fs*norm2 with k = segments of n. */
DSPB200_API int dspb200_filt_welch_exec(dspb200_os_plan* os, dspb200_spec_plan* spec, const void* x_host, int64_t n, double r,
                            void* out_host);

/* stft / spectrogram: src/periodograms.jl:828-897.  `s` holds nchan columns of `len` samples; out holds
 * nchan matrices of nout x k (column-major, column = segment).  psd_only != 0: PSD columns (real eltype)
 * scaled with r = fs*norm2 (:883,890); psd_only == 0: raw spectra (complex eltype), two-sided real input
 * completed by conjugate symmetry (:234-244).  nchan > 1 is the batched form of the per-vector reference
 * signature (SURVEY.md hard part 4).  psd_only == 3 (device form, fused sizes): the PSD columns are ADDED to the contents
 * of `out`. */
DSPB200_API int dspb200_stft_exec(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t nchan, double r, int psd_only,
                      void* out);
DSPB200_API int dspb200_stft_exec_dev(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t nchan, double r, int psd_only,
                          void* out, void* stream);
/* Streaming stft / spectrogram (an extension; the reference's stft takes one vector).  Every channel c has the virtual column
 * v = [hist_in[:, c] (nhist samples); x[:, c] (nx samples)]; hist_in / hist_out are ldh x nchan, x is nx x nchan (all
 * column-major).  The call emits segments 0 .. nseg-1 of each v (segment s starts at s*hop) -- column s of channel c at
 * out + (c*ldo + s)*nout, ldo >= nseg -- then writes the new history v[nseg*hop, nhist + nx) to hist_out.  hist_in == NULL:
 * an empty history.  psd_only: 0 raw spectra, 1 PSD columns scaled with r = fs*norm2 (no accumulate form).  Real input:
 * segments 2u and 2u+1 are transformed together, as the one-shot call pairs them, and an odd nseg transforms the last one
 * alone; so a stream whose calls start at even global segments reproduces stft of the concatenated signal bit for bit.  The
 * plan is the one an aligned one-shot call runs, whatever the alignment of the history or chunk.  DSPB200_EINVALID, before
 * any launch, when hist_out overlaps hist_in, x or out, when out overlaps x or a history buffer, when ldo < nseg, when
 * (nseg-1)*hop + n > nhist + nx, or when the new history would exceed ldh.  nx == 0 with nseg == 0 launches nothing and
 * leaves hist_out as it was (the history is still hist_in).  Fused sizes: at most two launches; cuFFT sizes: three per
 * batch of (channel, segment) pairs plus the history.
 * A multitaper plan (dspb200_mt_plan_create) streams mt_spectrogram: psd_only must be 1 and r 1.0 (the taper rows carry
 * 1/sqrt(r_t)), otherwise DSPB200_EINVALID before any launch.  Column s of channel c is then the PSD of that segment summed
 * over the plan's taper rows in taper order, the bits of column s of dspb200_mt_spectrogram_batch_exec_dev over the
 * concatenated signal; the virtual columns, pairing, plan and refusals are those above, and the call is queued on the
 * caller's stream like every other call of this form.  Fused sizes: at most two launches (the history, then every taper row
 * of every segment in one launch); cuFFT sizes: per taper three launches per batch of (channel, segment) pairs, one add per
 * taper after the first, plus the history. */
DSPB200_API int dspb200_stft_stream_exec_dev(dspb200_spec_plan* plan, const void* hist_in, int64_t nhist, void* hist_out, int64_t ldh,
                                             const void* x, int64_t nx, int64_t nchan, int64_t nseg, double r, int psd_only,
                                             void* out, int64_t ldo, void* stream);
/* host pointers; hist_in / hist_out hold ldh x nchan elements, the rows of hist_out past the new history are unspecified */
DSPB200_API int dspb200_stft_stream_exec(dspb200_spec_plan* plan, const void* hist_in, int64_t nhist, void* hist_out, int64_t ldh,
                                         const void* x, int64_t nx, int64_t nchan, int64_t nseg, double r, int psd_only,
                                         void* out, int64_t ldo);
/* Streaming Welch (an extension; the reference's welch_pgram takes one vector): the virtual columns, histories and checks of
 * dspb200_stft_stream_exec_dev.  The call adds the power spectra |FFT(window .* segment)|^2 of segments 0 .. nseg-1 of every
 * channel's v = [hist_in; x] to acc -- an nout x nchan Float64 matrix, column-major, bin k of channel c at acc[c*nout + k]
 * (add = 1), or writes them there (add = 0: a fresh accumulation, no separate zeroing) -- then writes the new history
 * v[nseg*hop, nhist + nx) to hist_out.  A call with nseg == 0 leaves acc as it is.  Every segment of a call is summed
 * in a fixed order: the result is deterministic.  DSPB200_EINVALID, before any launch, for the rules of the STFT stream
 * (overlapping buffers, acc in place of out; segments past the virtual column; a new history larger than ldh) and add not
 * 0 or 1.  Fused sizes: at most four launches per group of channels (see dspb200_welch_batch_exec_dev); a call whose
 * segments all lie in x (nhist == 0) runs the launch of dspb200_welch_batch_exec_dev on x, so one call over the whole
 * matrix followed by dspb200_welch_stream_power_dev gives the batched welch_pgram bit for bit.  cuFFT sizes: three
 * launches per batch of (channel, segment) pairs plus the history. */
DSPB200_API int dspb200_welch_stream_exec_dev(dspb200_spec_plan* plan, const void* hist_in, int64_t nhist, void* hist_out,
                                              int64_t ldh, const void* x, int64_t nx, int64_t nchan, int64_t nseg, double* acc,
                                              int add, void* stream);
/* host pointers; acc is read (add = 1) and written on the host */
DSPB200_API int dspb200_welch_stream_exec(dspb200_spec_plan* plan, const void* hist_in, int64_t nhist, void* hist_out,
                                          int64_t ldh, const void* x, int64_t nx, int64_t nchan, int64_t nseg, double* acc,
                                          int add);
/* The Welch power of a streaming accumulation: out (nout x nchan, real eltype of the plan) = acc with the fft2pow! scaling
 * of welch_pgram (src/periodograms.jl:142-172), r = nsegments*fs*norm2.  One launch; out may not overlap acc. */
DSPB200_API int dspb200_welch_stream_power_dev(dspb200_spec_plan* plan, const double* acc, int64_t nchan, double r, void* out,
                                               void* stream);
DSPB200_API int dspb200_welch_stream_power(dspb200_spec_plan* plan, const double* acc, int64_t nchan, double r, void* out);
/* arraysplit(s, n, noverlap, nfft, window) / ArraySplit: src/periodograms.jl:32-73, 134-137.  out = k x nfft matrix, row i =
 * [window .* s[i*hop .. i*hop+n) ; zeros(nfft-n)] (the reference yields the rows one at a time into one reused buffer). */
DSPB200_API int dspb200_arraysplit_exec(dspb200_spec_plan* plan, const void* s, int64_t len, void* out);
/* periodogram(s::AbstractMatrix; nfft, fs, radialsum, radialavg): src/periodograms.jl:473-509 with fft2pow2! (:175-181) and
 * fft2pow2radial! (:183-232).  s is an n1 x n2 real matrix (column-major), zero-padded to nfft1 x nfft2; r = fs * length(s).
 * ptype 0: out = real[nfft1 x nfft2] two-dimensional PSD; 1 (radialsum) / 2 (radialavg): out = real[min(nfft)>>1 + 1]. */
DSPB200_API int dspb200_periodogram2_exec(int dtype, const void* s, int64_t n1, int64_t n2, int64_t nfft1, int64_t nfft2, double r,
                                          int ptype, void* out);
/* device pointers + cudaStream_t; returns after the work on that stream has completed */
DSPB200_API int dspb200_periodogram2_exec_dev(int dtype, const void* d_s, int64_t n1, int64_t n2, int64_t nfft1, int64_t nfft2,
                                              double r, int ptype, void* d_out, void* stream);

/* Multitaper (SURVEY.md 8f, "next" rank 1): mt_pgram / mt_spectrogram, src/multitaper.jl:117-242, 262-404.
 * `tapers` = ntapers rows of n Float64 samples, each pre-scaled by the host with 1/sqrt(r_t),
 * r_t = fs * sum|w_t|^2 / weight_t (:135-139); the library then sums fft2pow!(FFT(w_t .* segment), 1) over tapers.
 * mt_pgram: len must equal n (DimensionMismatch :226); out = nout values.  mt_spectrogram: out = nout x k.  These are the
 * nchan = 1 case of the _batch forms below. */
DSPB200_API int dspb200_mt_plan_create(dspb200_spec_plan** plan, int dtype, int64_t n, int64_t noverlap, int64_t nfft,
                           int onesided, const double* tapers_host, int64_t ntapers);
DSPB200_API int dspb200_mt_pgram_exec(dspb200_spec_plan* plan, const void* s, int64_t len, void* out);
DSPB200_API int dspb200_mt_spectrogram_exec(dspb200_spec_plan* plan, const void* s, int64_t len, void* out);
/* device pointers + cudaStream_t; return after the work on that stream has completed */
DSPB200_API int dspb200_mt_pgram_exec_dev(dspb200_spec_plan* plan, const void* d_s, int64_t len, void* d_out, void* stream);
DSPB200_API int dspb200_mt_spectrogram_exec_dev(dspb200_spec_plan* plan, const void* d_s, int64_t len, void* d_out, void* stream);
/* Multitaper of many channels (an extension; the reference's mt_pgram / mt_spectrogram take one vector): `s` holds nchan
 * columns of len samples (column-major), each estimated with the plan's tapers; column c's result is that of the vector call
 * on it (fused sizes; the one exception: a Float32 nfft = 1024 mt_spectrogram of a matrix whose channels are not 16-byte
 * aligned runs the block kernel, while an aligned vector runs the warp-per-unit kernel, which rounds differently).
 * mt_pgram: len must equal n; out = nout x nchan.  mt_spectrogram: out = nchan matrices of nout x k (column-major,
 * the layout of the batched spectrogram).  Every channel's tapers are summed in taper order.  nchan == 0, or k == 0,
 * launches nothing and leaves out as it is.  DSPB200_EINVALID, before any launch: a NULL buffer, len != n (mt_pgram), a
 * negative size, or (device form) out overlapping s.  Fused sizes: mt_pgram runs two launches per group of channels (the
 * batched Welch kernel, one work item per channel whose units are its tapers, then the finalize kernel); mt_spectrogram one
 * launch, which transforms every segment pair under every taper inside one CTA (warp, for Float32 nfft = 1024) and writes
 * each PSD column once per taper.  cuFFT sizes: mt_pgram three launches per batch of (channel, taper) pairs plus one;
 * mt_spectrogram one batched STFT over all channels per taper, plus one add per taper after the first.  The _dev forms take
 * device pointers and a cudaStream_t and return after the work on that stream has completed; the host forms copy `s` in and
 * `out` back. */
DSPB200_API int dspb200_mt_pgram_batch_exec(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t nchan, void* out);
DSPB200_API int dspb200_mt_pgram_batch_exec_dev(dspb200_spec_plan* plan, const void* d_s, int64_t len, int64_t nchan, void* d_out,
                                                void* stream);
DSPB200_API int dspb200_mt_spectrogram_batch_exec(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t nchan, void* out);
DSPB200_API int dspb200_mt_spectrogram_batch_exec_dev(dspb200_spec_plan* plan, const void* d_s, int64_t len, int64_t nchan,
                                                      void* d_out, void* stream);
/* mt_cross_power_spectra! / mt_coherence!: src/multitaper.jl:553-616, 672-693, 722-790.  `signal` is the reference's
 * n_channels x n_samples matrix (column-major: channel index fastest), n_samples = the plan's n; the plan must be real and
 * one-sided (:411-416) with noverlap = 0.  demean != 0 subtracts the channel means (:566-570).  [f_lo, f_lo+nf) is the
 * 0-based range of retained frequency bins (freq_range, :497-503).  coherence == 0: out = Complex[n_channels x n_channels
 * x nf] cross power spectra; != 0: out = real[n_channels x n_channels x nf] pairwise coherences.  The _dev form takes
 * device pointers and a cudaStream_t and returns after the work on that stream has completed. */
DSPB200_API int dspb200_mt_cross_spectra_exec(dspb200_spec_plan* plan, const void* signal, int64_t nchan, int demean,
                                              int64_t f_lo, int64_t nf, int coherence, void* out);
DSPB200_API int dspb200_mt_cross_spectra_exec_dev(dspb200_spec_plan* plan, const void* d_signal, int64_t nchan, int demean,
                                                  int64_t f_lo, int64_t nf, int coherence, void* d_out, void* stream);
/* The same estimate over many epochs (trials), an extension: `signal` is n_channels x n_samples x nepochs (column-major:
 * signal[:, :, e] is epoch e's matrix).  With M_e the cross spectra of dspb200_mt_cross_spectra_exec on epoch e (same plan,
 * demean per channel per epoch, same [f_lo, f_lo+nf)), the cross spectra are S / nepochs with S = ((M_0 + M_1) + M_2) + ...
 * summed in epoch order in the output eltype and each of its real and imaginary parts divided by nepochs (nepochs == 1: M_0,
 * bit for bit the matrix call's result); coherence != 0 gives the coherence of that epoch-mean cross spectrum.  Each M_e is
 * the taper sum of the matrix call, term for term.  Work: the epochs run in groups whose raw spectra (nout x n_channels x
 * ntapers per epoch) fit 1 GiB, at least one epoch per group; per group one mean-removal launch, one raw-spectra STFT call
 * per taper over all the group's (channel, epoch) columns (fused sizes: one launch; even 7-smooth cuFFT sizes: three launches
 * per batch of the plan's cuFFT batch size; other cuFFT sizes, whose batched transforms couple neighbouring columns: one such
 * call per taper and epoch, over that epoch's channels), and one accumulate launch that sums every taper and epoch of the
 * group into each output element and writes it once; coherence adds one launch.  The matrix call is the nepochs == 1 case of this path.
 * DSPB200_EINVALID before any launch: the matrix call's refusals, nepochs < 1, a signal or output past
 * DSPB200_INDEX_LIMIT, and (device form) an output overlapping the signal.  nf == 0 launches nothing.
 * dspb200_mt_cross_spectra_epochs takes device pointers and a cudaStream_t and returns after the work on that stream has
 * completed; the _exec form copies `signal` in and `out` back. */
DSPB200_API int dspb200_mt_cross_spectra_epochs(dspb200_spec_plan* plan, const void* d_signal, int64_t nchan, int64_t nepochs,
                                                int demean, int64_t f_lo, int64_t nf, int coherence, void* d_out, void* stream);
DSPB200_API int dspb200_mt_cross_spectra_epochs_exec(dspb200_spec_plan* plan, const void* signal, int64_t nchan, int64_t nepochs,
                                                     int demean, int64_t f_lo, int64_t nf, int coherence, void* out);
DSPB200_API int dspb200_spec_plan_destroy(dspb200_spec_plan* plan);

/* ------------------------------------------------------------------------------------------ polyphase resample
 * resample(x, rate, h) with Integer / Rational rate = interp // decim: FIRFilter{FIRRational | FIRInterpolator |
 * FIRDecimator} + filt! loops (src/Filters/stream_filt.jl:8-78, 137-178, 294-307, 431-560) and _resample!
 * (:696-725).  y[j] = sum_t hp[phi + t*interp] x[n - t], p = phi0 + j*decim, n = n0 + p / interp,
 * phi = p % interp (closed form of the (inputIdx, phiIdx) recurrence); x is zero outside [0, nx).
 * (n0, phi0) come from setphase!(timedelay) on the host (:223-229, 400-403, 706-714).
 * dtype_x in {F32,F64,C32,C64}, dtype_h in {F32,F64}; output eltype = promote_type(dtype_h, dtype_x) (:654). */
typedef struct dspb200_resample_plan dspb200_resample_plan;
DSPB200_API int dspb200_resample_plan_create(dspb200_resample_plan** plan, int dtype_x, int dtype_h, const void* h_host,
                                 int64_t hlen, int64_t interp, int64_t decim);
DSPB200_API int dspb200_resample_out_dtype(const dspb200_resample_plan* plan, int* dtype_out);
DSPB200_API int dspb200_resample_exec(dspb200_resample_plan* plan, const void* x, int64_t nx, int64_t ncols, int64_t n0,
                          int64_t phi0, void* out, int64_t nout);
DSPB200_API int dspb200_resample_exec_dev(dspb200_resample_plan* plan, const void* x, int64_t nx, int64_t ncols, int64_t n0,
                              int64_t phi0, void* out, int64_t nout, void* stream);
/* Range form: outputs [j_begin, j_begin+nout_local) of the virtual input whose samples
 * [x_begin, x_begin+nx_local) are stored at x_local (zero elsewhere).
 * Domain (DSPB200_INDEX_LIMIT = 2^61, DSPB200_PHASE_LIMIT = 2^62), with j_end = j_begin + nout_local:
 * 0 <= j_begin, 0 <= nout_local, j_end <= 2^61, phi0 + j_end * decim <= 2^62, 0 <= n0 and the newest input sample
 * n0 + (phi0 + j_end * decim) / interp <= 2^61, 0 <= nx_local, |x_begin| <= 2^61 and x_begin + nx_local <= 2^61;
 * otherwise DSPB200_EINVALID before any launch. */
DSPB200_API int dspb200_resample_exec_range_dev(dspb200_resample_plan* plan, const void* x_local, int64_t x_begin,
                                    int64_t nx_local, int64_t n0, int64_t phi0, void* out_local, int64_t j_begin,
                                    int64_t nout_local, void* stream);
/* Arbitrary (floating-point) rate: FIRArbitrary / filt!(buffer, ::FIRFilter{FIRArbitrary}, x),
 * src/Filters/stream_filt.jl:92-134, 567-625.  The plan holds pfb = taps2pfb(h, nphases) and dpfb = taps2pfb([diff(h); 0],
 * nphases).  Output j (0-based) of a call sits at total phase P_j = acc0 + j*delta (delta = nphases / rate, acc0 = the
 * kernel's phiAccumulator in [0, nphases)): newest input sample n0 + floor(P_j / nphases) (0-based index into x, which the
 * host passes as [history; x]), phase floor(P_j mod nphases), alpha = its fraction; y_j = muladd(yUpper, alpha, yLower)
 * (:606-616).  Samples outside [0, nx) are zero.  Out eltype = promote(eltype(h), eltype(x)) as for the rational plan. */
DSPB200_API int dspb200_resample_arb_plan_create(dspb200_resample_plan** plan, int dtype_x, int dtype_h, const void* h_host,
                                                 int64_t hlen, int64_t nphases);
DSPB200_API int dspb200_resample_arb_exec(dspb200_resample_plan* plan, const void* x, int64_t nx, int64_t n0, double acc0,
                                          double delta, void* out, int64_t nout);
DSPB200_API int dspb200_resample_arb_exec_dev(dspb200_resample_plan* plan, const void* x, int64_t nx, int64_t n0, double acc0,
                                              double delta, void* out, int64_t nout, void* stream);
/* Column c holds samples x[c*ldx + i], i in [0, nx), zero elsewhere (ldx >= nx); output column c is out[c*nout + j].
 * Every column uses the same (n0, acc0, delta) -- a fresh filter after undelay!, as resample(X, rate; dims) does.
 * One kernel launch for all columns; ncols == 0 launches nothing. */
DSPB200_API int dspb200_resample_arb_batch_exec(dspb200_resample_plan* plan, const void* x, int64_t nx, int64_t ldx,
                                                int64_t ncols, int64_t n0, double acc0, double delta, void* out, int64_t nout);
DSPB200_API int dspb200_resample_arb_batch_exec_dev(dspb200_resample_plan* plan, const void* x, int64_t nx, int64_t ldx,
                                                    int64_t ncols, int64_t n0, double acc0, double delta, void* out,
                                                    int64_t nout, void* stream);
/* Streaming FIRFilter (filt!(buffer, self::FIRFilter, x), src/Filters/stream_filt.jl:137-403, 409-625) on ncols channels
 * that share one phase state; device pointers, enqueued on `stream`, no synchronisation.  A call filters each channel's
 * virtual column [history; x] (history: the plan's tpp - 1 samples, x: nx samples) from the state (input_deficit >= 1 and
 * phi0 in [0, interp) -- 0-based phiIdx -- or acc0 = phiAccumulator in [0, nphases)), exactly as the reference's filt! on
 * that channel, and writes the nout outputs the host computed from the same state (outputlength) to out[c*ldo + j].
 * x is nx x ncols column-major; hist_in / hist_out are (tpp - 1) x ncols column-major in x's element type: hist_in is the
 * history before x (NULL: zeros), hist_out receives the last tpp - 1 samples of [history; x].  Chunks fed one after the
 * other with the returned state give outputs bit-identical to the reference's filt! on each channel.
 * DSPB200_EINVALID before any launch when hist_out overlaps hist_in, x or out, when out overlaps x or a history buffer,
 * when ldo < nout, or when nx == 0 with nout > 0.  nout == 0 with nx > 0 only updates the history (a chunk shorter than
 * inputDeficit, :484-488, :590-594); nx == 0 or ncols == 0 launches nothing.
 * Rational plans (dspb200_resample_plan_create): at most two launches -- the outputs whose window reaches into the
 * history together with the new history, then the rest on the chunk through the same kernels as dspb200_resample_exec_dev.
 * Arbitrary-rate plans (dspb200_resample_arb_plan_create): the batched kernel reads [history; x] itself, plus one launch
 * for the history. */
DSPB200_API int dspb200_resample_stream_exec_dev(dspb200_resample_plan* plan, const void* hist_in, void* hist_out, const void* x,
                                                 int64_t nx, int64_t ncols, int64_t input_deficit, int64_t phi0, void* out,
                                                 int64_t ldo, int64_t nout, void* stream);
DSPB200_API int dspb200_resample_arb_stream_exec_dev(dspb200_resample_plan* plan, const void* hist_in, void* hist_out,
                                                     const void* x, int64_t nx, int64_t ncols, int64_t input_deficit, double acc0,
                                                     double delta, void* out, int64_t ldo, int64_t nout, void* stream);
DSPB200_API int dspb200_resample_plan_destroy(dspb200_resample_plan* plan);

#ifdef __cplusplus
}
#endif
#endif /* DSPB200_H */
