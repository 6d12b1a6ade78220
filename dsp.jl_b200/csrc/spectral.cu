// dspb200 -- Welch / periodogram / STFT / spectrogram.
//
// Reference path: src/periodograms.jl -- ArraySplit (:32-73), fft2pow! (:142-172), fft2oneortwosided!
// (:234-244), welch_pgram_helper! (:746-759), stft (:872-897).
//
// Fused path (power-of-two nfft that fits shared memory): one kernel does segment gather, window
// multiply (Float64 product rounded to the signal eltype, :66), the FFT out of shared memory and
//   * Welch: |Z|^2 accumulated in registers across all segments a CTA owns; real signals ride two
//     segments per complex FFT (z = a + i b), and because |A_k|^2 + |B_k|^2 = (|Z_k|^2 + |Z_{N-k}|^2)/2
//     the split is deferred to the finalize kernel -- the inner loop never un-mixes the two spectra.
//     One kernel body with two work assignments: one signal (a unit range per CTA, one partial row each, added to
//     across streaming calls) or the columns of a matrix (a range of (channel, slice) items, one row per item); one
//     finalize kernel reduces the rows of each channel.
//   * STFT / spectrogram: the spectrum is parked in shared memory (natural order), un-mixed per bin and
//     stored column by column, coalesced along frequency.
// Generic path (any other nfft): seg_window_kernel -> batched cuFFT -> power / store kernels.  Every cuFFT-size Welch and
// mt_pgram is one segment list per channel through seg_window_kernel, cuFFT and a Float64 accumulate kernel, then
// welch_stream_power_kernel.
// STFT: one-shot and streaming calls (dspb200_stft_stream_exec(_dev)) run the same kernels over each channel's virtual column
// [history; chunk] (StftStream; a one-shot call has no history), a stream after stft_stream_edge_kernel has copied the seam
// samples and written the new history; cuFFT sizes run a call's (channel, segment) pairs through seg_window_kernel -> cuFFT ->
// stft_store_kernel.
#include "fft_core.cuh"
#include "async_copy.cuh"
#include "cufft_exec.cuh"
#include <math.h>
#include <stdlib.h>
#include <new>
#include <vector>

namespace dspb200 {

struct SpecPlanImpl {
    int dtype = 0;
    bool cplx = false, f64 = false;
    int64_t n = 0, noverlap = 0, hop = 0, nfft = 0;
    int onesided = 0;
    int64_t nout = 0;
    bool fused = false;
    int device = 0;
    int sm_count = 0;               // device_sm_count() at plan creation
    void* d_window = nullptr;     // n window values (double, or float2 hi/lo pairs for Float32 signals) or null
    void* d_tw = nullptr;         // last-pass twiddle table (fused; fft_fill_tl)
    void* d_t32 = nullptr;        // nfft = 1024, Float32: W_1024^t rows of the warp-per-unit STFT kernel (stft_w1k_kernel)
    void* d_t16 = nullptr;        // cx<T>[16][8], cx<T>[256][8]: radix-16 twiddle tables (fused)
    void* d_t256 = nullptr;
    size_t smem_optin = 0;        // cudaDevAttrMaxSharedMemoryPerBlockOptin
    int64_t ntapers = 0;          // multitaper plans: d_window holds ntapers rows of n values
    DevBuf tmp;                   // multitaper spectrogram, cuFFT sizes: one taper's PSD matrices
    // launch configuration of the fused Welch kernel, chosen once per (plan, alignment class): the selection walks up to nine
    // kernel instances through cudaFuncSetAttribute + the occupancy calculator (tens of microseconds per launch otherwise)
    // (mode: MODE of the instance; vctas: virtual CTAs pinned by dspb200_spec_plan_pin_welch, 0 = one resident wave;
    //  used: virtual CTAs of the last launch, 0 = none yet)
    struct WelchCfg { void* kern = nullptr; size_t smem = 0; int g = 0, per_sm = 0, threads = 0, mode = -1; int64_t vctas = 0, used = 0; };
    WelchCfg welch_cfg[2];        // [0]: unaligned segments (direct loads), [1]: TMA-capable
    int nparts = 0;               // CTAs of the Welch kernel == rows of `partial`
    int rows_used = 0;            // rows of `partial` written since welch_begin (host bookkeeping, stream order = call order)
    DevBuf partial;               // fused Welch: [nparts][nfft] real T
    // batched Welch (dspb200_welch_batch_exec_dev): its own kernel configuration cache and scratch, so that a streaming
    // accumulation open on the plan (partial / rows_used, acc) is left as it was
    WelchCfg welch_batch_cfg[2];
    WelchCfg welch_mt_cfg[2];     // the batched kernel's taper-row instances (mt_pgram), which share `bpartial`
    DevBuf bpartial;              // fused: one row of nfft real T per (channel, slice), at most WELCH_BATCH_SCRATCH bytes
    DevBuf bacc;                  // generic: double[nout], one channel at a time (mt_pgram: double[nout][nchan])
    // generic path
    cufftHandle fft = 0;
    bool fft_ok = false;
    int64_t batch = 0;            // segments per cuFFT call
    int64_t nbins_fft = 0;        // nfft/2+1 (real) or nfft (complex)
    DevBuf segbuf, specbuf, acc;  // acc: double[nout], the accumulation open since welch_begin
    // host-pointer path
    HostPipe pipe;
    DevBuf hin, hout;             // dspb200_stft_stream_exec: the staged histories
    DevBuf seam;                  // streaming STFT, fused sizes: the seam samples of the last call (stft_stream_edge_kernel)
    DevBuf y;                     // dspb200_filt_welch_exec: the filter output, n samples
};

// ---------------------------------------------------------------------------------------------- helpers
// src/periodograms.jl:66 forms sample * window in Float64 (window functions return Vector{Float64}) and rounds
// the product to the buffer eltype.  Float64 signals: one DMUL.  Float32 signals: the window is held as an
// unevaluated float pair w = wh + wl (|wl| <= ulp(wh)/2) and the product is fma(x, wh, x*wl): it equals
// round(x * w * (1 + e)), |e| < 2^-47, i.e. the reference's correctly rounded value except when x*w falls within
// 2^-47 (relative) of a Float32 rounding boundary (about one sample in 10^7, then off by one ulp) -- without
// putting two conversions and a DMUL per sample on the FP64 pipe.
template <typename T> struct win_t { using type = double; };
template <> struct win_t<float> { using type = float2; };
__device__ __forceinline__ double win_mul(double v, double w) { return v * w; }
__device__ __forceinline__ float win_mul(float v, float2 w) { return fmaf(v, w.x, v * w.y); }

// out + val rounded once per operation: the accumulate form of a PSD store (psd_only == 3) must give the eltype sum of the
// two stored values, which a contraction of val's product into the add (one FMA, one rounding) would not
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }

template <typename T, bool CPLX> struct in_type { using type = T; };
template <typename T> struct in_type<T, true> { using type = cx<T>; };

// ---------------------------------------------------------------------------------------------- fused Welch
// Persistent CTAs; a virtual CTA (below) runs a sequence of units (unit = one complex segment, or two consecutive real
// segments packed as re/im).  TMA variant: the raw samples of the NEXT unit (one contiguous hop+n range) are
// fetched by a single cp.async.bulk into a staging buffer while the current unit's FFT passes run, so the HBM
// latency of the segment loads is off the critical path; the first FFT pass reads the staged samples from
// shared memory.  The direct variant (unaligned segments, or staging does not fit) loads from global memory
// in the first pass.
// MODE 0: direct loads; 1: TMA staging; 2: TMA staging + the window table copied to shared memory once per CTA (when
// that does not cost residency): the per-unit window reads were the kernel's main long-scoreboard stall;
// 3: TMA staging + the window in REGISTERS: thread t multiplies the samples j = t + r N/16 of every segment, so its 16
// window values never change -- they are loaded once (32 registers for the Float32 hi/lo pairs), which removes the window
// reads (13 % of the kernel's shared-memory wavefronts at nfft = 4096) and the 32 KB table.
// G > 1: G independent thread groups per CTA, each a "virtual CTA" with its own data buffer, staging buffer and mbarrier
// and its own work, synchronising among themselves only (named barriers); the groups share ONE copy of the
// twiddle tables and of the window table, so three 4096-point transforms fit one SM where two single-group CTAs with
// private tables did (ncu on the two-CTA configuration: 4 warps per scheduler, issue slots 60 % busy, the stalls that
// remain -- wait, short scoreboard -- are latency a third warp set hides).
// Shared-memory layout: [tables][window (MODE 2)] then per group [data buffer][staging][mbarrier].
template <typename T, int N, bool CPLX, int MODE> struct welch_layout {
    using In = typename in_type<T, CPLX>::type;
    using W = typename win_t<T>::type;
    __host__ __device__ static size_t table_bytes() { return (size_t)fft_table_elems<T, N>() * sizeof(cx<T>); }
    __host__ __device__ static size_t window_bytes(int64_t n) { return MODE == 2 ? (size_t)n * sizeof(W) : 0; }
    __host__ __device__ static size_t stage_elems(int64_t n, int64_t hop) { return MODE >= 1 ? (size_t)(CPLX ? n : hop + n) : 0; }
    __host__ __device__ static size_t group_bytes(int64_t n, int64_t hop) {
        return (((size_t)padded_len<T>(N) * sizeof(cx<T>) + stage_elems(n, hop) * sizeof(In) + 15) & ~(size_t)15) + 16;
    }
    __host__ __device__ static size_t total(int64_t n, int64_t hop, int groups) {
        return table_bytes() + window_bytes(n) + (size_t)groups * group_bytes(n, hop);
    }
};
template <typename T, int N, int G> struct welch_bounds {
    static constexpr int NTG = fft_threads<N>::value;
    static constexpr int minblocks = G == 1 ? fft_minblocks<T, N>::value : 1;
};

// The two work assignments of welch_fused_kernel; virtual CTA v of nv takes the v-th of nv equal contiguous shares of the
// work.  One signal (BATCH = false: welch_exec*, range, streaming, filt_welch): the work is the units of segments
// seg0 .. seg0 + nseg - 1 (`sample_offset`: the signal index of the buffer's first sample), and v writes partial row v
// once, at the end.  Many channels (BATCH = true: welch_batch_exec*): the columns of a len x nchan matrix, `chan_stride`
// samples apart, nseg segments (upc units) each.  The work is nitems (channel, slice) items: slice j of a channel owns its
// units [j per, min((j+1) per, upc)), so units never cross a channel and a real unit's two segments always belong to one
// channel (the finalize pass un-mixes bins k and N-k of one row).  v writes ONE partial row per item (row = item index);
// the TMA prefetch of the next unit runs across item and channel boundaries.  No atomics: the result is deterministic.
// Each work assignment's parameters are Nil in the other's instances, and each keeps the parameter order it had as a kernel
// of its own: ptxas assigns the parameters' uniform registers by offset, and a struct of them compiles to different code.
// TAPERS (batch only: multitaper periodograms, mt_pgram): unit u of a channel is taper u -- all of a channel's units read the
// same n samples at the channel's start, unit u under window row u (rows n values apart), and nseg = 1 (no unit has a second
// real segment).  The staged samples serve every taper of the channel; the next channel's are fetched after the last taper's
// first pass.  Only MODE 0 / 1 address a window row per unit.
struct Nil {};
template <bool USED, typename X> using welch_arg = typename std::conditional<USED, X, Nil>::type;

template <typename T, int N, bool CPLX, int MODE, int G, bool BATCH, bool TAPERS = false>
__global__ void __launch_bounds__((welch_bounds<T, N, G>::NTG * G), (welch_bounds<T, N, G>::minblocks))
welch_fused_kernel(const void* __restrict__ s_, welch_arg<BATCH, int64_t> chan_stride, welch_arg<!BATCH, int64_t> seg0,
                   int64_t nseg, welch_arg<BATCH, int64_t> upc, welch_arg<BATCH, int64_t> per, welch_arg<BATCH, int> slices,
                   welch_arg<BATCH, int64_t> nitems, int64_t hop, int n, welch_arg<!BATCH, int64_t> sample_offset,
                   const typename win_t<T>::type* __restrict__ win, const cx<T>* __restrict__ tw,
                   const cx<T>* __restrict__ g16, const cx<T>* __restrict__ g256, T* __restrict__ partial,
                   welch_arg<!BATCH, int> fresh_from) {
    constexpr int NT = fft_threads<N>::value;                 // threads of one group
    constexpr int NB16 = N / 16;
    constexpr int ITL = (NB16 + NT - 1) / NT;
    using L = welch_layout<T, N, CPLX, MODE>;
    using Scope = typename std::conditional<G == 1, FftCtaScope, FftGroupScope<NT>>::type;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    using In = typename in_type<T, CPLX>::type;
    const In* s = reinterpret_cast<const In*>(s_);
    const int gid = G == 1 ? 0 : threadIdx.x / NT;
    const int tid = G == 1 ? threadIdx.x : threadIdx.x - gid * NT;
    constexpr bool TMA = MODE >= 1;
    constexpr bool WSM = MODE == 2;
    constexpr bool WREG = MODE == 3;
    static_assert(!TAPERS || (BATCH && MODE <= 1), "taper rows: the batched work assignment, window read per unit");
    using W = typename win_t<T>::type;
    cx<T>* tabs = reinterpret_cast<cx<T>*>(smem_raw);
    W* wsm = reinterpret_cast<W*>(smem_raw + L::table_bytes());
    unsigned char* gbase = smem_raw + L::table_bytes() + L::window_bytes(n) + (size_t)gid * L::group_bytes(n, hop);
    cx<T>* sm = reinterpret_cast<cx<T>*>(gbase);
    In* stage = reinterpret_cast<In*>(sm + padded_len<T>(N));                  // TMA staging: hop + n samples
    uint64_t* bar = reinterpret_cast<uint64_t*>(gbase + L::group_bytes(n, hop) - 16);
    // tables and window: staged once by all threads of the CTA
    pdl_launch_dependents();
    const FftCtx<T> ctx = fft_make_ctx_at<T, N, NT * G>(sm, tabs, g16, g256, tw, threadIdx.x);
    if constexpr (WSM) {
        for (int i = threadIdx.x; i < n; i += NT * G) wsm[i] = win[i];
    }
    Scope scope;
    if constexpr (G > 1) scope.id = 8 + gid;
    W wreg[WREG ? ITL : 1][WREG ? 16 : 1];
    if constexpr (WREG) {
#pragma unroll
        for (int it = 0; it < ITL; ++it)
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                const int j = tid + it * NT + r * NB16;
                wreg[it][r] = (j < n && tid + it * NT < NB16) ? win[j] : W{};
            }
    }

    T acc[ITL][16];                                   // thread t: |X[t + it NT + r N/16]|^2 summed over its units (natural order)
#pragma unroll
    for (int i = 0; i < ITL; ++i)
#pragma unroll
        for (int r = 0; r < 16; ++r) acc[i][r] = T(0);

    // this virtual CTA's share [w0, w1) of the units (one signal) or of the items (batch)
    int64_t work;
    if constexpr (BATCH) work = nitems;
    else work = CPLX ? nseg : (nseg + 1) / 2;
    const int64_t vcta = (int64_t)blockIdx.x * G + gid, nvcta = (int64_t)gridDim.x * G;     // (CTA, group) = virtual CTA
    const int64_t share = (work + nvcta - 1) / nvcta;
    const int64_t w0 = vcta * share < work ? vcta * share : work;
    const int64_t w1 = w0 + share < work ? w0 + share : work;

    // unit u (of channel c in a batch)
    auto unit_src = [&](int64_t c, int64_t u) -> const In* {
        if constexpr (TAPERS) return s + c * chan_stride;
        else if constexpr (BATCH) return s + c * chan_stride + (CPLX ? u : 2 * u) * hop;
        else return s + ((seg0 + (CPLX ? u : 2 * u)) * hop - sample_offset);
    };
    auto unit_bytes = [&](int64_t u) -> uint32_t {
        const bool hasB = !CPLX && (2 * u + 1 < nseg);
        return (uint32_t)((hasB ? hop + n : n) * sizeof(In));
    };
    // batch: item i -> (channel c, units [ua, ub))
    auto item_range = [&](int64_t i, int64_t& c, int64_t& ua, int64_t& ub) {
        if constexpr (BATCH) {
            c = i / slices;
            ua = (i - c * slices) * per;
            ub = ua + per < upc ? ua + per : upc;
        }
    };
    if constexpr (TMA) {
        if (tid == 0) {
            mbar_init(bar, 1);
            mbar_fence_init();
        }
    }
    pdl_wait();                                       // constants staged; the samples and `partial` come from preceding kernels
    __syncthreads();                                  // twiddle tables staged, barrier initialised
    // the current item: channel c, units [ua, ub); one signal is one item, its whole range
    int64_t c = 0, ua = BATCH ? 0 : w0, ub = BATCH ? 0 : w1;
    if constexpr (BATCH) {
        if (w0 < w1) item_range(w0, c, ua, ub);
    }
    if constexpr (TMA) {
        if (tid == 0 && w0 < w1) {
            mbar_expect_tx(bar, unit_bytes(ua));
            tma_load_1d(stage, unit_src(c, ua), unit_bytes(ua), bar);
        }
    }
    uint32_t parity = 0;

    for (int64_t item = w0; !BATCH || item < w1; ++item) {
        for (int64_t u = ua; u < ub; ++u) {
            const bool hasB = !CPLX && (2 * u + 1 < nseg);
            const In* pa = TMA ? stage : unit_src(c, u);
            const In* pb = pa + hop;
            const W* wu = TAPERS ? win + u * n : win;
            if constexpr (TMA) {
                if (!TAPERS || u == ua) {                    // taper rows: one staged copy per channel
                    mbar_wait(bar, parity);
                    parity ^= 1;
                }
            }
            auto ld0 = [&](int j, int it, int r) -> cx<T> {
                if (j >= n) return mkc<T>(T(0), T(0));
                if constexpr (CPLX) {
                    cx<T> v = pa[j];
                    if (WREG || WSM || wu) { const W w = WREG ? wreg[WREG ? it : 0][WREG ? r : 0] : (WSM ? wsm[j] : wu[j]); v = mkc<T>(win_mul(v.x, w), win_mul(v.y, w)); }
                    return v;
                } else {
                    T a = pa[j];
                    T b = hasB ? pb[j] : T(0);
                    if (WREG || WSM || wu) { const W w = WREG ? wreg[WREG ? it : 0][WREG ? r : 0] : (WSM ? wsm[j] : wu[j]); a = win_mul(a, w); b = win_mul(b, w); }
                    return mkc<T>(a, b);
                }
            };
            // first pass: the staged samples are read and transformed, then -- one barrier later, which also ends the
            // previous unit's last pass -- stored; once every thread is past its reads (the barrier after the pass: with two
            // first-pass iterations, N = 16384, the second one reads after the pass's own barrier) the staging buffer is
            // refilled with the next unit while the remaining passes run -- behind a proxy fence, which orders those
            // generic-proxy reads before the bulk copy's async-proxy writes
            fft_first_pass<T, N, NT, true>(ctx, tid, ld0, scope);
            scope.sync();
            if constexpr (TMA && !BATCH) {
                if (tid == 0 && u + 1 < ub) {
                    fence_proxy_async_shared();
                    mbar_expect_tx(bar, unit_bytes(u + 1));
                    tma_load_1d(stage, unit_src(c, u + 1), unit_bytes(u + 1), bar);
                }
            }
            if constexpr (TMA && BATCH) {
                // the next unit: the following one of this item, else the first one of the next item
                if (tid == 0) {
                    int64_t nc = c, nu = u + 1, nub = ub;
                    if (nu == ub && item + 1 < w1) item_range(item + 1, nc, nu, nub);
                    else if (TAPERS) nu = nub;                  // the next taper reads the samples already staged
                    if (nu < nub) {
                        fence_proxy_async_shared();
                        mbar_expect_tx(bar, unit_bytes(nu));
                        tma_load_1d(stage, unit_src(nc, nu), unit_bytes(nu), bar);
                    }
                }
            }
            fft_middle<T, N, NT>(ctx, tid, scope);
#pragma unroll
            for (int it = 0; it < ITL; ++it) {
                const int tp = tid + it * NT;
                if (NB16 % NT != 0 && tp >= NB16) break;
                cx<T> v[16];
                fft_last_pass<T, N>(ctx, tp, v);
#pragma unroll
                for (int r = 0; r < 16; ++r) acc[it][r] += cabs2(v[r]);
            }
        }

        // one signal: rows below `fresh_from` hold the sums of earlier launches since welch_begin and are added to; the
        // others are written for the first time (no memset of the partial rows, and the finalize pass reads only rows that
        // were written).  Batch: row `item`, and the next item starts from zero.
        T* dst = partial + (BATCH ? item : vcta) * N;
        bool add = false;
        if constexpr (!BATCH) add = vcta < fresh_from;
#pragma unroll
        for (int it = 0; it < ITL; ++it) {
            const int tp = tid + it * NT;
            if (tp < NB16) {
#pragma unroll
                for (int r = 0; r < 16; ++r) {                                   // natural order, coalesced along tp
                    if constexpr (BATCH) {
                        dst[tp + r * NB16] = acc[it][r];
                        acc[it][r] = T(0);
                    } else {
                        T* q = dst + tp + r * NB16;
                        *q = add ? *q + acc[it][r] : acc[it][r];
                    }
                }
            }
        }
        if constexpr (BATCH) {
            if (item + 1 < w1) item_range(item + 1, c, ua, ub);
        } else {
            break;                                    // one signal: one pass
        }
    }
}

// Reduce the partial spectra of channel blockIdx.y -- its `rows` rows, written since welch_begin (one signal) or one per slice
// (batch) -- in Float64, fold the two-for-one mixing for real input, apply the fft2pow! scale (m1 = 1/r, m2 = 2/r; :142-172)
// and write column blockIdx.y of the nout x nchan result.  A CTA owns 32 consecutive bins; warp sl of the nw = blockDim.x / 32
// sums rows sl, sl + nw, ... (a warp reads 128 contiguous bytes of a row -- the earlier one-warp-per-bin form read a 32-byte
// sector per element and took 14 us for 592 rows, 5 % of the whole C3 Welch), then the nw slices are added in a fixed order.
template <typename T, int N>
__global__ void __launch_bounds__(1024) welch_finalize_kernel(const T* __restrict__ partial, int rows, T* __restrict__ out,
                                                              int nout, int real_in, int onesided, double m1, double m2) {
    __shared__ double red[32][33];
    pdl_launch_dependents();
    pdl_wait();
    const int b = threadIdx.x & 31, sl = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int k = blockIdx.x * 32 + b;
    const T* chan = partial + (int64_t)blockIdx.y * rows * N;
    double sum = 0.0;
    if (k < nout) {
        const T* c0 = chan + k;                             // the partial spectra are in natural order
        const T* c1 = chan + ((N - k) & (N - 1));
        if (real_in) {
            for (int c = sl; c < rows; c += nw) sum += (double)c0[(int64_t)c * N] + (double)c1[(int64_t)c * N];
        } else {
            for (int c = sl; c < rows; c += nw) sum += (double)c0[(int64_t)c * N];
        }
    }
    red[sl][b] = sum;
    __syncthreads();
    if (sl == 0 && k < nout) {
        for (int i = 1; i < nw; ++i) sum += red[i][b];
        double m = m1;
        if (real_in) {
            sum *= 0.5;
            if (onesided && !(k == 0 || k == N / 2)) m = m2;
        }
        out[(int64_t)blockIdx.y * nout + k] = (T)(sum * m);
    }
}

// ---------------------------------------------------------------------------------------------- fused STFT
// Persistent CTAs over units (unit = one complex segment or two consecutive real segments of one channel); same
// front end as the Welch kernel (TMA bulk prefetch of the next unit's samples when segment starts are 16-byte
// aligned).  The last pass writes the spectrum back to shared memory in natural order (in place: a thread stores the
// slots it loaded); every thread then emits the bins k = tid + NT*i, un-mixing the two real segments per bin, and the
// global stores of a column are coalesced along frequency.
// MODE 1: PSD columns (fft2pow!), 0: raw spectra (fft2oneortwosided!).  HASB: the unit carries a second real segment
// (-1: decided at run time by `hasB`).  ONES (real input): one-sided output, nout = N/2 + 1 (-1: run time).
template <typename T, int N, bool CPLX, int MODE, int HASB, int ONES, bool ACC = false>
__device__ __forceinline__ void stft_emit(const cx<T>* __restrict__ sm, void* __restrict__ out_, int64_t colA, int nout,
                                          bool hasB_rt, int onesided_rt, T m1, T m2, int tid) {
    constexpr int NT = fft_threads<N>::value;
    // ACC: PSD columns are ADDED to what `out` holds (psd_only == 3, and the tapers after a unit's first in mt_spectrogram).
    // Compile time: as a run-time predicate the read-modify-write put a scoreboard wait in front of every store (ncu).
    auto put = [&](T* ptr, T val) { if constexpr (ACC) *ptr = add_rn(*ptr, val); else *ptr = val; };
    const bool hasB = HASB < 0 ? hasB_rt : (HASB != 0);
    const bool onesided = ONES < 0 ? (onesided_rt != 0) : (ONES != 0);
    // `edge`: the bin is DC or Nyquist (scaled by m1 even in a one-sided PSD, src/periodograms.jl:142-172)
    auto emit = [&](int kk, cx<T> zk, cx<T> zm, bool edge) {
        if constexpr (MODE == 1) {                       // PSD columns
            T* out = reinterpret_cast<T*>(out_);
            if constexpr (CPLX) {
                put(out + colA + kk, cabs2(zk) * m1);
            } else {
                // A = (zk + conj zm) / 2, B = (zk - conj zm) / 2i: the halving is exact, so |A|^2 m is formed as the reference does
                const cx<T> A = mkc<T>(T(0.5) * (zk.x + zm.x), T(0.5) * (zk.y - zm.y));
                const cx<T> B = mkc<T>(T(0.5) * (zk.y + zm.y), T(0.5) * (zm.x - zk.x));
                const T m = (onesided && !edge) ? m2 : m1;
                put(out + colA + kk, cabs2(A) * m);
                if (hasB) put(out + colA + nout + kk, cabs2(B) * m);
            }
        } else {                                         // raw spectra
            cx<T>* out = reinterpret_cast<cx<T>*>(out_);
            if constexpr (CPLX) {
                out[colA + kk] = zk;
            } else {
                out[colA + kk] = mkc<T>(T(0.5) * (zk.x + zm.x), T(0.5) * (zk.y - zm.y));
                if (hasB) out[colA + nout + kk] = mkc<T>(T(0.5) * (zk.y + zm.y), T(0.5) * (zm.x - zk.x));
            }
        }
    };
    // the spectrum is in natural order: consecutive lanes read consecutive slots (k) / consecutive slots backwards (N - k)
    if constexpr (NT * 16 == N) {
        // bins kk = tid + Q i: padaddr(kk) = padaddr(tid) + padaddr(Q i), and for tid > 0
        // padaddr(N - kk) = padaddr(Q - tid) + padaddr(Q (15 - i)) -- every per-bin offset is a compile-time constant
        // (ncu on the 1024-point spectrogram kernel: a generic loop spent ~50 instructions per output bin, mostly integer
        // address arithmetic and predicates)
        constexpr int Q = N / 16;
        const cx<T>* pk = sm + padaddr<T, N>(tid);
        const cx<T>* pm = tid ? sm + padaddr<T, N>(Q - tid) : sm;
        const bool half = !CPLX && onesided;             // bins 0 .. N/2: i = 0..7 for every thread, bin N/2 for thread 0
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            if (i >= 8 && half) break;
            const cx<T> zk = pk[padaddr<T, N>(Q * i)];
            cx<T> zm = zk;
            if constexpr (!CPLX) zm = pm[tid ? padaddr<T, N>(Q * (15 - i)) : padaddr<T, N>((Q * (16 - i)) & (N - 1))];
            emit(tid + Q * i, zk, zm, (i == 0 || i == 8) && tid == 0);
        }
        if (half && tid == 0) {
            const cx<T> z = sm[padaddr<T, N>(N / 2)];
            emit(N / 2, z, z, true);
        }
    } else {
        for (int kk = tid; kk < nout; kk += NT) {
            const cx<T> zk = sm[padaddr<T, N>(kk)];
            cx<T> zm = zk;
            if constexpr (!CPLX) zm = sm[padaddr<T, N>((N - kk) & (N - 1))];
            emit(kk, zk, zm, kk == 0 || kk == N / 2);
        }
    }
}

// An STFT call transforms segments 0 .. k - 1 of every channel's virtual column v = [history (h samples); x]; a one-shot call
// is one with h = 0 and ldo = k.  A unit that starts in the history (a seam unit) reads the copy of v's first samples that
// the call's edge kernel wrote to `seam` (stft_stream_edge_kernel); every other unit reads x + start - h.  Either way a
// unit's samples are one contiguous range, staged by TMA or loaded directly, so a stream puts the same values into the same
// butterflies as one call over the concatenated signal.
template <typename In> struct StftStream {
    const In* seam;             // lds x nchan: v[0, lds) of every channel (the samples of its seam units)
    int64_t lds, h;             // column stride of `seam`, samples of history
    int64_t ldo;                // output columns per channel (replaces k as the column stride)
    int tma;                    // the call meets the TMA alignment conditions (stft_w1k_kernel: stage every unit)
    int ntapers;                // WIN == 2 instances (mt_spectrogram): taper rows of the window, n values apart
    // first sample of the unit that starts at v[start] of channel c (x: the chunk, chan_stride = nx)
    __device__ __forceinline__ const In* src(const In* x, int64_t chan_stride, int64_t c, int64_t start) const {
        return start < h ? seam + c * lds + start : x + c * chan_stride + (start - h);
    }
};

// One unit of the STFT kernel.  FAST: n == N (no zero padding) and, for real input, both segments present -- no per-sample
// predicates; WIN: 1 window table present, 0 none (compile time), -1 run time, 2 one row of a multitaper plan's tapers (PSD
// columns; `add`: added to what `out` holds, in the emit step).
template <typename T, int N, bool CPLX, bool TMA, int WIN, bool FAST, class IssueNext>
__device__ __forceinline__ void stft_unit(const FftCtx<T>& ctx, cx<T>* sm, int tid, const typename in_type<T, CPLX>::type* pa,
                                          int64_t hop, int n, bool hasB_rt, const typename win_t<T>::type* __restrict__ win,
                                          void* __restrict__ out_, int64_t colA, int nout, int psd_only, int onesided, T m1,
                                          T m2, IssueNext issue_next, bool add = false) {
    constexpr int NT = fft_threads<N>::value;
    constexpr int NB16 = N / 16;
    constexpr int ITL = (NB16 + NT - 1) / NT;
    using In = typename in_type<T, CPLX>::type;
    const In* pb = pa + hop;
    const bool hasB = FAST ? !CPLX : hasB_rt;
    // (Float64 taper rows keep the run-time test of WIN = -1: a product known to be taken is contracted into the first
    //  butterfly's adds, which rounds differently from the spectrogram of one taper)
    const bool use_win = (WIN < 0 || (WIN == 2 && sizeof(T) == 8)) ? (win != nullptr) : (WIN != 0);
    auto ld0 = [&](int j, int, int) -> cx<T> {
        if constexpr (!FAST) { if (j >= n) return mkc<T>(T(0), T(0)); }
        if constexpr (CPLX) {
            cx<T> v = pa[j];
            if (use_win) { const auto w = win[j]; v = mkc<T>(win_mul(v.x, w), win_mul(v.y, w)); }
            return v;
        } else {
            T a = pa[j];
            T b = hasB ? pb[j] : T(0);
            if (use_win) { const auto w = win[j]; a = win_mul(a, w); b = win_mul(b, w); }
            return mkc<T>(a, b);
        }
    };
    // (the barrier inside the first pass also ends the previous unit's emit step)
    fft_first_pass<T, N, NT, true>(ctx, tid, ld0);
    __syncthreads();
    issue_next();                                        // every thread has read the staging buffer: refill it
    fft_middle<T, N, NT>(ctx, tid);
#pragma unroll
    for (int it = 0; it < ITL; ++it) {
        const int tp = tid + it * NT;
        if (NB16 % NT != 0 && tp >= NB16) break;
        cx<T> v[16];
        fft_last_pass<T, N>(ctx, tp, v);
        cx<T>* p = sm + padaddr<T, N>(tp);
#pragma unroll
        for (int r = 0; r < 16; ++r) p[padaddr<T, N>(r * NB16)] = v[r];       // natural order, in place
    }
    __syncthreads();
    constexpr int HB = FAST ? (CPLX ? 0 : 1) : -1;
    if constexpr (WIN == 2) {
        if (add) stft_emit<T, N, CPLX, 1, HB, -1, true>(sm, out_, colA, nout, hasB, onesided, m1, m2, tid);
        else stft_emit<T, N, CPLX, 1, HB, -1, false>(sm, out_, colA, nout, hasB, onesided, m1, m2, tid);
    } else if (psd_only & 2) {                           // bit 1: accumulate into `out`
        stft_emit<T, N, CPLX, 1, -1, -1, true>(sm, out_, colA, nout, hasB, onesided, m1, m2, tid);
    } else if (psd_only) {
        if (CPLX || !onesided) stft_emit<T, N, CPLX, 1, HB, 0>(sm, out_, colA, nout, hasB, 0, m1, m2, tid);
        else stft_emit<T, N, CPLX, 1, HB, 1>(sm, out_, colA, nout, hasB, 1, m1, m2, tid);
    } else {
        stft_emit<T, N, CPLX, 0, HB, -1>(sm, out_, colA, nout, hasB, onesided, m1, m2, tid);
    }
}

// (tried: compiling the Float32 STFT kernels for 768 resident threads per SM -- the 1024-point kernel fits 64 registers and
//  gets 11 CTAs per SM instead of 8 -- but the spectrogram got slower and the windowed variants spill; kept at 512 threads /
//  128 registers)
// s_ is the chunk x (chan_stride = its column length), k the call's segments per channel; a unit's samples come from
// StftStream::src and its columns are ldo apart.
template <typename T, int N, bool CPLX, bool TMA, int WIN>
__global__ void __launch_bounds__(fft_threads<N>::value, fft_minblocks<T, N>::value)
stft_fused_kernel(const void* __restrict__ s_, int64_t chan_stride, int64_t k, int64_t units_per_chan, int64_t total_units,
                  int64_t hop, int n, const typename win_t<T>::type* __restrict__ win, const cx<T>* __restrict__ tw,
                  const cx<T>* __restrict__ g16, const cx<T>* __restrict__ g256, void* __restrict__ out_, int nout,
                  int psd_only, int onesided, T m1, T m2, const StftStream<typename in_type<T, CPLX>::type> ss) {
    constexpr int NT = fft_threads<N>::value;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    using In = typename in_type<T, CPLX>::type;
    const In* s = reinterpret_cast<const In*>(s_);
    const int tid = threadIdx.x;
    const FftCtx<T> ctx = fft_make_ctx<T, N, NT>(sm, g16, g256, tw, tid);
    In* stage = reinterpret_cast<In*>(sm + fft_smem_elems<T, N>());
    uint64_t* bar = reinterpret_cast<uint64_t*>(stage + (CPLX ? n : (hop + n)));

    const int64_t per = (total_units + gridDim.x - 1) / gridDim.x;
    const int64_t u0 = (int64_t)blockIdx.x * per;
    const int64_t u1 = u0 + per < total_units ? u0 + per : total_units;
    // (channel, unit inside the channel) of the current unit, advanced incrementally: no 64-bit division in the loop
    int64_t chan = u0 < u1 ? u0 / units_per_chan : 0;
    int64_t uin = u0 < u1 ? u0 - chan * units_per_chan : 0;
    auto src_of = [&](int64_t c, int64_t u) -> const In* { return ss.src(s, chan_stride, c, (CPLX ? u : 2 * u) * hop); };
    auto bytes_of = [&](int64_t u) -> uint32_t {
        const bool hb = !CPLX && (2 * u + 1 < k);
        return (uint32_t)((hb ? hop + n : n) * sizeof(In));
    };
    if constexpr (TMA) {
        if (tid == 0) {
            mbar_init(bar, 1);
            mbar_fence_init();
        }
    }
    __syncthreads();
    if constexpr (TMA) {
        if (tid == 0 && u0 < u1) {
            mbar_expect_tx(bar, bytes_of(uin));
            tma_load_1d(stage, src_of(chan, uin), bytes_of(uin), bar);
        }
    }
    uint32_t parity = 0;
    const bool full = (n == N);

    for (int64_t gu = u0; gu < u1; ++gu) {
        const int64_t segA = CPLX ? uin : 2 * uin;
        const bool hasB = !CPLX && (segA + 1 < k);
        const In* pa = TMA ? stage : src_of(chan, uin);
        // the next unit
        int64_t nchan = chan, nuin = uin + 1;
        if (nuin == units_per_chan) { nuin = 0; ++nchan; }
        if constexpr (TMA) {
            mbar_wait(bar, parity);
            parity ^= 1;
        }
        auto issue_next = [&]() {
            if constexpr (TMA) {
                if (tid == 0 && gu + 1 < u1) {
                    fence_proxy_async_shared();          // after the generic-proxy reads of the staging buffer
                    mbar_expect_tx(bar, bytes_of(nuin));
                    tma_load_1d(stage, src_of(nchan, nuin), bytes_of(nuin), bar);
                }
            }
        };
        const int64_t colA = (chan * ss.ldo + segA) * (int64_t)nout;
        if constexpr (WIN == 2) {
            // every taper transforms the staged unit, in taper order; the staging buffer is refilled after the last one's
            // first pass
            for (int t = 0; t < ss.ntapers; ++t) {
                const auto* wt = win + (int64_t)t * n;
                auto issue_last = [&]() { if (t + 1 == ss.ntapers) issue_next(); };
                if (full && (CPLX || hasB))
                    stft_unit<T, N, CPLX, TMA, WIN, true>(ctx, sm, tid, pa, hop, n, hasB, wt, out_, colA, nout, 1, onesided, m1, m2, issue_last, t > 0);
                else
                    stft_unit<T, N, CPLX, TMA, WIN, false>(ctx, sm, tid, pa, hop, n, hasB, wt, out_, colA, nout, 1, onesided, m1, m2, issue_last, t > 0);
            }
        } else {
            if (full && (CPLX || hasB))
                stft_unit<T, N, CPLX, TMA, WIN, true>(ctx, sm, tid, pa, hop, n, hasB, win, out_, colA, nout, psd_only, onesided, m1, m2, issue_next);
            else
                stft_unit<T, N, CPLX, TMA, WIN, false>(ctx, sm, tid, pa, hop, n, hasB, win, out_, colA, nout, psd_only, onesided, m1, m2, issue_next);
        }
        chan = nchan;
        uin = nuin;
    }
}

// ---------------------------------------------------------------------------------------------- 1024-point STFT, one warp per unit
// nfft = 1024 = 32 x 32 (BASELINE config 4): a warp owns a whole transform -- lane c computes the plain 32-point DFT of
// x[c + 32 m], one shared-memory exchange, then lane t the twiddled radix-32 butterfly that leaves X[t + 32 s] -- so a unit
// needs ONE exchange instead of two, no CTA-wide barrier at all (__syncwarp only) and every warp of the SM is an independent
// stream of work (its own staging buffer, mbarrier and TMA prefetch of its next unit).  Float32 only.
namespace w1k {
constexpr int N = 1024;
__host__ __device__ __forceinline__ constexpr int pad(int p) { return p + 2 * (p >> 4) + 2 * (p >> 5); }   // 32-runs 38 apart: odd multiple of 16 B
constexpr int DATA_LEN = 1216;                         // pad(1023) + 1 = 1212, rounded up to a multiple of 4
constexpr int T32_LEN = 32 * 16;
// host side: the twiddles W_1024^t of the second radix-32 pass, all 16 of lane t's butterfly, pair-major (word i*32 + t
// holds values 2i, 2i+1 of row t)
inline void fill_t32(cx<float>* t32) {
    cx<float> row[16];
    for (int t = 0; t < 32; ++t) {
        fft_fill_row<float>(row, 32, t, 1024);
        for (int i = 0; i < 16; ++i) t32[((i >> 1) * 32 + t) * 2 + (i & 1)] = row[i];
    }
}
__host__ __device__ inline size_t warp_bytes(int64_t stage_elems, size_t elt) { return (((size_t)DATA_LEN * 8 + (size_t)stage_elems * elt + 15) & ~(size_t)15) + 16; }
}  // namespace w1k

// Arguments as stft_fused_kernel.  A stream keeps this plan whatever the alignment of the call: ss.tma = 0 (unaligned) reads
// every unit directly from global memory in the first pass instead of staging it.  WIN: 0 no window, 1 the window staged in
// shared memory, 2 the ss.ntapers taper rows of a multitaper plan, read through L1 (7 rows of 8 KB would cost residency),
// each unit transformed under every row in turn and its PSD columns summed over them in `out`.
template <bool CPLX, int WIN, int WARPS>
__global__ void __launch_bounds__(32 * WARPS)
stft_w1k_kernel(const void* __restrict__ s_, int64_t chan_stride, int64_t k, int64_t units_per_chan, int64_t total_units,
                int64_t hop, int n, const float2* __restrict__ win, const cx<float>* __restrict__ g32, void* __restrict__ out_,
                int nout, int psd_only, int onesided, float m1, float m2,
                const StftStream<typename in_type<float, CPLX>::type> ss) {
    using T = float;
    using In = typename in_type<T, CPLX>::type;
    constexpr int N = w1k::N;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const In* s = reinterpret_cast<const In*>(s_);
    // layout: [T32][window (n float2, when present)] then per warp [data][staging][mbarrier]
    cx<T>* t32 = reinterpret_cast<cx<T>*>(smem_raw);
    float2* wsm = reinterpret_cast<float2*>(smem_raw + w1k::T32_LEN * sizeof(cx<T>));
    const size_t stage_elems = (size_t)(CPLX ? n : hop + n);
    const size_t wbytes = w1k::warp_bytes((int64_t)stage_elems, sizeof(In));
    unsigned char* wbase = smem_raw + w1k::T32_LEN * sizeof(cx<T>) + (WIN == 1 ? (size_t)n * sizeof(float2) : 0) + (size_t)warp * wbytes;
    cx<T>* sm = reinterpret_cast<cx<T>*>(wbase);
    In* stage = reinterpret_cast<In*>(sm + w1k::DATA_LEN);
    uint64_t* bar = reinterpret_cast<uint64_t*>(wbase + wbytes - 16);
    for (int i = threadIdx.x; i < w1k::T32_LEN; i += 32 * WARPS) t32[i] = g32[i];
    if constexpr (WIN == 1) {
        for (int i = threadIdx.x; i < n; i += 32 * WARPS) wsm[i] = win[i];
    }
    if (lane == 0) {
        mbar_init(bar, 1);
        mbar_fence_init();
    }
    __syncthreads();                                    // tables staged, barriers initialised -- the only CTA-wide barrier

    const int64_t vw = (int64_t)blockIdx.x * WARPS + warp, nvw = (int64_t)gridDim.x * WARPS;     // virtual CTA = warp
    const int64_t per = (total_units + nvw - 1) / nvw;
    const int64_t u0 = vw * per < total_units ? vw * per : total_units;
    const int64_t u1 = u0 + per < total_units ? u0 + per : total_units;
    int64_t chan = u0 < u1 ? u0 / units_per_chan : 0;
    int64_t uin = u0 < u1 ? u0 - chan * units_per_chan : 0;
    auto src_of = [&](int64_t c, int64_t u) -> const In* { return ss.src(s, chan_stride, c, (CPLX ? u : 2 * u) * hop); };
    auto bytes_of = [&](int64_t u) -> uint32_t {
        const bool hb = !CPLX && (2 * u + 1 < k);
        return (uint32_t)((hb ? hop + n : n) * sizeof(In));
    };
    if (lane == 0 && u0 < u1 && ss.tma) {
        mbar_expect_tx(bar, bytes_of(uin));
        tma_load_1d(stage, src_of(chan, uin), bytes_of(uin), bar);
    }
    uint32_t parity = 0;
    const bool full = (n == N);
    // twiddle row of this lane's last-pass butterfly (w = W_1024^lane): the same for every unit -- kept in registers
    cx<T> tw[16];
#pragma unroll
    for (int i = 0; i < 16; i += 2) lds2<T>(t32 + ((i >> 1) * 32 + lane) * 2, tw[i], tw[i + 1]);

    for (int64_t gu = u0; gu < u1; ++gu) {
        const int64_t segA = CPLX ? uin : 2 * uin;
        const bool hasB = !CPLX && (segA + 1 < k);
        int64_t nchan = chan, nuin = uin + 1;
        if (nuin == units_per_chan) { nuin = 0; ++nchan; }
        if (ss.tma) {
            mbar_wait(bar, parity);
            parity ^= 1;
        }
        // WIN == 2: every taper row transforms the unit in turn, in taper order (the same staged samples)
        for (int t = 0; t < (WIN == 2 ? ss.ntapers : 1); ++t) {
            const float2* wrow = WIN == 2 ? win + (int64_t)t * n : wsm;
            // first pass: plain 32-point DFT of x[lane + 32 m] (window applied), 32 contiguous slots at block `lane`.  Written
            // out once per source, so that a staged unit is read by shared-memory loads (through a pointer that may point to
            // either space they become generic loads); an unaligned streaming call reads its units directly
            cx<T> v[32];
            const bool fast = full && (CPLX || hasB);
            auto first_pass = [&](const In* pa) {
                const In* pb = pa + hop;
#pragma unroll
                for (int m = 0; m < 32; ++m) {
                    const int j = lane + 32 * m;
                    if constexpr (CPLX) {
                        cx<T> x = (fast || j < n) ? pa[j] : mkc<T>(0.f, 0.f);
                        if constexpr (WIN != 0) { const float2 w = wrow[fast || j < n ? j : 0]; x = mkc<T>(win_mul(x.x, w), win_mul(x.y, w)); }
                        v[m] = x;
                    } else {
                        float a = (fast || j < n) ? pa[j] : 0.f;
                        float b = (fast || (hasB && j < n)) ? pb[j] : 0.f;
                        if constexpr (WIN != 0) { const float2 w = wrow[fast || j < n ? j : 0]; a = win_mul(a, w); b = win_mul(b, w); }
                        v[m] = mkc<T>(a, b);
                    }
                }
            };
            if (ss.tma) first_pass(stage);
            else first_pass(src_of(chan, uin));
            __syncwarp();                                  // every lane has read the staging buffer (and the previous unit's spectrum)
            // refill it with the next unit while this one is transformed (after the last taper's first pass)
            if (lane == 0 && gu + 1 < u1 && ss.tma && (WIN != 2 || t + 1 == ss.ntapers)) {
                fence_proxy_async_shared();
                mbar_expect_tx(bar, bytes_of(nuin));
                tma_load_1d(stage, src_of(nchan, nuin), bytes_of(nuin), bar);
            }
            fft_bfly<T, 32, true>(v, nullptr);
            {
                cx<T>* p = sm + w1k::pad(32 * lane);
#pragma unroll
                for (int r = 0; r < 32; r += 2) sts2<T>(p + w1k::pad(r), v[r], v[r + 1]);
            }
            __syncwarp();
            // last pass: radix 32 at stride 32, twiddles W_1024^lane; the spectrum goes back in natural order, in place
            {
                cx<T>* p = sm + w1k::pad(lane);
#pragma unroll
                for (int r = 0; r < 32; ++r) v[r] = p[38 * r];
                fft_bfly<T, 32, false>(v, tw);
#pragma unroll
                for (int r = 0; r < 32; ++r) p[38 * r] = v[r];
            }
            __syncwarp();
            // emit: bins kk = lane + 32 i; N - kk = (32 - lane) + 32 (31 - i) for lane > 0
            const int64_t colA = (chan * ss.ldo + segA) * (int64_t)nout;
            const cx<T>* pk = sm + w1k::pad(lane);
            const cx<T>* pm = lane ? sm + w1k::pad(32 - lane) : sm;
            const bool half = !CPLX && onesided;
            // (the accumulate flag is resolved once per unit: as a run-time predicate inside the stores it put a scoreboard wait
            //  in front of every one of them)
            auto emit_all = [&](auto acc_) {
                constexpr bool ACC = decltype(acc_)::value;
                auto put = [&](T* ptr, T val) { if constexpr (ACC) *ptr = add_rn(*ptr, val); else *ptr = val; };
                auto emit = [&](int kk, cx<T> zk, cx<T> zm, bool edge) {
                    if (psd_only) {
                        T* out = reinterpret_cast<T*>(out_);
                        if constexpr (CPLX) {
                            put(out + colA + kk, cabs2(zk) * m1);
                        } else {
                            const cx<T> A = mkc<T>(0.5f * (zk.x + zm.x), 0.5f * (zk.y - zm.y));
                            const cx<T> B = mkc<T>(0.5f * (zk.y + zm.y), 0.5f * (zm.x - zk.x));
                            const T m = (onesided && !edge) ? m2 : m1;
                            put(out + colA + kk, cabs2(A) * m);
                            if (hasB) put(out + colA + nout + kk, cabs2(B) * m);
                        }
                    } else {
                        cx<T>* out = reinterpret_cast<cx<T>*>(out_);
                        if constexpr (CPLX) {
                            out[colA + kk] = zk;
                        } else {
                            out[colA + kk] = mkc<T>(0.5f * (zk.x + zm.x), 0.5f * (zk.y - zm.y));
                            if (hasB) out[colA + nout + kk] = mkc<T>(0.5f * (zk.y + zm.y), 0.5f * (zm.x - zk.x));
                        }
                    }
                };
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                    if (i >= 16 && half) break;
                    const cx<T> zk = pk[38 * i];
                    cx<T> zm = zk;
                    if constexpr (!CPLX) zm = pm[lane ? 38 * (31 - i) : 38 * ((32 - i) & 31)];
                    emit(lane + 32 * i, zk, zm, (i == 0 || i == 16) && lane == 0);
                }
                if (half && lane == 0) {
                    const cx<T> z = sm[w1k::pad(N / 2)];
                    emit(N / 2, z, z, true);
                }
            };
            if constexpr (WIN == 2) {                  // later tapers add to the first one's columns
                if (t > 0) emit_all(std::true_type{});
                else emit_all(std::false_type{});
            } else {
                if (psd_only & 2) emit_all(std::true_type{});
                else emit_all(std::false_type{});
            }
        }
        chan = nchan;
        uin = nuin;
    }
}

// ---------------------------------------------------------------------------------------------- STFT, small kernels
// Launch 1 of a streaming call, one grid-stride pass over nchan x (ls + hn) items: (a) seam[c lds + i] = v_c[i], i < ls --
// the samples of the units that start in the history, contiguous, so that the transform reads every unit from one range;
// (b) the new history hist_out[c ldh + i] = v_c[skip + i], i < hn.  v_c = [hist_in (h samples, column stride ldh); x_c].
template <typename E>
__global__ void stft_stream_edge_kernel(const E* __restrict__ hist_in, int64_t h, int64_t ldh, const E* __restrict__ x,
                                        int64_t nx, int64_t nchan, E* __restrict__ seam, int64_t ls, int64_t lds, int64_t skip,
                                        int64_t hn, E* __restrict__ hist_out) {
    const int64_t per = ls + hn, total = nchan * per;
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += (int64_t)gridDim.x * blockDim.x) {
        const int64_t c = w / per, i = w - c * per;
        const int64_t t = (i < ls ? i : skip + i - ls) - h;                     // index in x (negative: history)
        const E v = t < 0 ? hist_in[c * ldh + h + t] : x[c * nx + t];
        if (i < ls) seam[c * lds + i] = v;
        else hist_out[c * ldh + i - ls] = v;
    }
}

// cuFFT sizes (STFT, Welch, multitaper, arraysplit): the call's nchan x k (channel c, segment j) pairs, f = c k + j, fill
// the cuFFT batch in order.  Slot b = blockIdx.y holds pair f0 + b: buf[b][i] = w_j[i] * v_c[j hop + i] (i < n), 0 for
// n <= i < nfft and for slots past the list, read from the virtual column v_c = [history (h samples); x_c].  The window
// of segment j is win + j wstride: the plan's one window (wstride = 0), or taper row j of a multitaper plan (hop = 0,
// wstride = n: every taper of a channel reads the same n samples).  One slot per grid row: the pair is resolved once per
// block, not per element.
template <typename T, bool CPLX>
__global__ void seg_window_kernel(const void* __restrict__ hist_, int64_t h, int64_t ldh, const void* __restrict__ x_,
                                  int64_t nx, int64_t f0, int64_t nf, int64_t k, int64_t hop, int64_t n, int64_t nfft,
                                  const typename win_t<T>::type* __restrict__ win, int64_t wstride, void* __restrict__ buf_) {
    using In = typename in_type<T, CPLX>::type;
    const In* hist = reinterpret_cast<const In*>(hist_);
    const In* x = reinterpret_cast<const In*>(x_);
    const int64_t b = blockIdx.y;
    In* buf = reinterpret_cast<In*>(buf_) + b * nfft;
    const int64_t f = f0 + b, c = f / k, j = f - c * k, t0 = j * hop - h;  // index in x of the segment's first sample
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nfft; i += (int64_t)gridDim.x * blockDim.x) {
        In v;
        if constexpr (CPLX) v = mkc<T>(T(0), T(0)); else v = T(0);
        if (b < nf && i < n) {
            const int64_t t = t0 + i;
            v = t < 0 ? hist[c * ldh + h + t] : x[c * nx + t];
            if (win) {
                const auto w = win[j * wstride + i];
                if constexpr (CPLX) v = mkc<T>(win_mul(v.x, w), win_mul(v.y, w)); else v = win_mul(v, w);
            }
        }
        buf[i] = v;
    }
}

// The spectra of pairs f0 .. f0 + nf - 1 (slot b = blockIdx.y) into column (c ldo + j) of out: raw (the real two-sided
// mirror conjugated), or PSD (fft2pow! scaling, :142-172)
template <typename T>
__global__ void stft_store_kernel(const cx<T>* __restrict__ X, int64_t nbins_fft, int64_t nfft, int64_t nout, int64_t f0,
                                  int64_t k, int64_t ldo, int psd_only, int onesided, T m1, T m2, void* __restrict__ out_) {
    const int64_t b = blockIdx.y, f = f0 + b, c = f / k, col = c * ldo + (f - c * k);
    const cx<T>* Xb = X + b * nbins_fft;
    for (int64_t kk = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; kk < nout; kk += (int64_t)gridDim.x * blockDim.x) {
        const bool mirrored = kk >= nbins_fft;
        const cx<T> z = Xb[mirrored ? nfft - kk : kk];
        if (psd_only) {
            T m = m1;
            if (onesided && kk != 0 && !(kk == nbins_fft - 1 && (nfft % 2 == 0))) m = m2;
            reinterpret_cast<T*>(out_)[col * nout + kk] = cabs2(z) * m;
        } else {
            reinterpret_cast<cx<T>*>(out_)[col * nout + kk] = mirrored ? cconj(z) : z;
        }
    }
}

// mt_pgram, cuFFT sizes: thread (bin kk, channel f0 / ntapers + blockIdx.y) adds (double)|X|^2 of its channel's slots to
// acc (nout x nchan) one taper at a time, in taper order -- continuing the channel's sum when its first tapers were in an
// earlier batch -- so that every channel gets one running sum over its tapers whatever the batch boundaries
// (welch_stream_acc_kernel instead adds each batch's partial sum, which rounds differently).  Two-sided real output: bin
// kk >= nbins_fft reads nfft - kk.
template <typename T>
__global__ void mt_pow_acc_kernel(const cx<T>* __restrict__ X, int64_t nbins_fft, int64_t nfft, int64_t nout, int64_t f0,
                                  int64_t nf, int64_t ntapers, double* __restrict__ acc) {
    const int64_t kk = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (kk >= nout) return;
    const int64_t c = f0 / ntapers + blockIdx.y;
    const int64_t a = c * ntapers > f0 ? c * ntapers : f0, e = (c + 1) * ntapers < f0 + nf ? (c + 1) * ntapers : f0 + nf;
    const int64_t src = kk < nbins_fft ? kk : nfft - kk;
    double* q = acc + c * nout + kk;
    double sum = a > c * ntapers ? *q : 0.0;
    for (int64_t f = a; f < e; ++f) sum += (double)cabs2(X[(f - f0) * nbins_fft + src]);
    *q = sum;
}

// Multitaper cross spectra (src/multitaper.jl:553-616).
// signal is an n_channels x n_samples x n_epochs array (channel index fastest; one epoch: the reference's matrix); xs gets
// one contiguous column per (channel, epoch), column e nchan + c, minus that column's mean when `demean` (:566-570).  One
// block per column.
template <typename T>
__global__ void cs_prep_kernel(const T* __restrict__ signal, int64_t nchan, int64_t n, int demean, T* __restrict__ xs) {
    const int64_t col = blockIdx.x, c = col % nchan;
    signal += (col / nchan) * nchan * n;
    xs += col * n;
    __shared__ double red[32];
    __shared__ T mean_s;
    double acc = 0.0;
    if (demean) {
        for (int64_t i = threadIdx.x; i < n; i += blockDim.x) acc += (double)signal[c + nchan * i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
        __syncthreads();
        if (threadIdx.x == 0) {
            double t = 0.0;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
            mean_s = (T)(t / (double)n);
        }
        __syncthreads();
    }
    const T mu = demean ? mean_s : T(0);
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) xs[i] = signal[c + nchan * i] - mu;
}

__device__ __forceinline__ float fma_rn(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ double fma_rn(double a, double b, double c) { return __fma_rn(a, b, c); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }

// Tile of cs_acc_kernel<T>: F consecutive frequencies x CS_C channels l x CS_C channels m per CTA of CS_THREADS threads;
// thread (fi, tl, tm) owns the RL x RM outputs l = l0 + tl + (CS_C / RL) i, m = m0 + tm + (CS_C / RM) j (strided, so that a
// warp's shared-memory reads hit distinct banks).  Float64 owns half as many outputs per thread as Float32: its 16 complex
// accumulators (partial and epoch sum of 4 x 2 outputs) and 6 operands fit the register file without spills.  The slabs of
// CS_STAGES consecutive (epoch, taper) steps are in flight at once.
constexpr int CS_C = 16, CS_THREADS = 256, CS_STAGES = 4;
template <typename T> struct CsTile {
    static constexpr int RL = 4, RM = sizeof(T) == 4 ? 4 : 2, TL = CS_C / RL, TM = CS_C / RM, F = CS_THREADS / (TL * TM);
};

// out[l, m, fi] over the g epochs of one group whose raw spectra x hold, for taper t, channel c of epoch e at column
// e nchan + c of the t-th nout x (nchan g) slab.  With f = f_lo + fi, each taper adds the term c_f * x[f, l] * conj(x[f, m])
// (rows pre-scaled by 1/sqrt(r_t), so the reference's weight 2/r_t and its 1/sqrt(2) on the DC / Nyquist rows become c_f =
// 2, or 1 there), with the FMA placement of re = fma(a.x, b.x, a.y b.y), im = fma(a.y, b.x, -(a.x b.y)), tapers 0 .. K-1 in
// order into the epoch's partial (the first assigns c_f (re, im), later ones add fma(c_f, re, p.x), fma(c_f, im, p.y)), and
// the partials of the epochs in order into the epoch sum (in the output eltype).  fresh: the first epoch's partial is the
// sum; else the sum continues from out.  divisor > 1: the sum's parts are then divided by it (the last group of E > 1
// epochs).  Every (l, m) is computed: a mirrored triangle would carry the other FMA placement in its imaginary part.
// The two frequency-by-channel slabs of each (epoch, taper) are loaded by cp.async, coalesced along frequency, into a ring of
// CS_STAGES buffers, CS_STAGES - 1 steps ahead of the one being summed; each output is written once.  Block b: l tile b % ct, m tile (b / ct) % ct, frequency tile
// b / ct^2 (ct = ceil(nchan / CS_C)), so the CTAs that share a slab run side by side.
template <typename T>
__global__ void __launch_bounds__(CS_THREADS) cs_acc_kernel(cx<T>* __restrict__ out, const cx<T>* __restrict__ x, int64_t nout,
                                                            int64_t nchan, int64_t g, int64_t ntapers, int64_t f_lo, int64_t nf,
                                                            int nyquist_row, int fresh, int64_t divisor) {
    using Tile = CsTile<T>;
    constexpr int RL = Tile::RL, RM = Tile::RM, TL = Tile::TL, TM = Tile::TM, F = Tile::F, LD = F + 1;
    __shared__ cx<T> slab[CS_STAGES][2][CS_C][LD];            // [buffer][l slab, m slab][channel][frequency], padded rows
    const int64_t ct = (nchan + CS_C - 1) / CS_C, b = blockIdx.x;
    const int64_t l0 = (b % ct) * CS_C, m0 = ((b / ct) % ct) * CS_C, fi0 = (b / (ct * ct)) * F;
    const int tid = threadIdx.x, fi = tid / (TL * TM), tl = tid % TL, tm = (tid / TL) % TM;
    // loads: thread tid copies frequency tid % F of channels tid / F (+ CS_THREADS / F) of both slabs
    constexpr int LROWS = CS_THREADS / F;                     // channels per copy pass: CS_C (Float32) or 2 CS_C / 2 (Float64)
    const int lf = tid % F, lc = tid / F;
    const bool fin = fi0 + lf < nf;
    const cx<T>* const src = x + (f_lo + fi0 + lf);
    const int64_t tstride = nout * nchan * g;
    int64_t ne = 0, nt = 0;                                   // the next (epoch, taper) to stage
    auto stage = [&](int buf) {                               // one commit group per step, empty past the last step
        if (ne < g) {
            const int64_t off = nout * nchan * ne + tstride * nt;
#pragma unroll
            for (int c = lc; c < CS_C; c += LROWS) {
                if (fin && l0 + c < nchan) cp_async<sizeof(cx<T>)>(&slab[buf][0][c][lf], src + off + nout * (l0 + c));
                if (fin && m0 + c < nchan) cp_async<sizeof(cx<T>)>(&slab[buf][1][c][lf], src + off + nout * (m0 + c));
            }
            if (++nt == ntapers) { nt = 0; ++ne; }
        }
        cp_async_commit();
    };
    const int64_t f = f_lo + fi0 + fi;
    const T cf = (f == 0 || (nyquist_row && f == nout - 1)) ? T(1) : T(2);
    const bool fout = fi0 + fi < nf;
    cx<T>* const o = out + nchan * nchan * (fi0 + fi);
    cx<T> p[RL][RM], sum[RL][RM];
    if (!fresh && fout) {
#pragma unroll
        for (int i = 0; i < RL; ++i)
#pragma unroll
            for (int j = 0; j < RM; ++j) {
                const int64_t l = l0 + tl + TL * i, m = m0 + tm + TM * j;
                if (l < nchan && m < nchan) sum[i][j] = o[l + nchan * m];
            }
    }
#pragma unroll
    for (int k = 0; k < CS_STAGES - 1; ++k) stage(k);
    int buf = 0;
    for (int64_t e = 0; e < g; ++e) {
        for (int64_t t = 0; t < ntapers; ++t) {
            cp_async_wait<CS_STAGES - 2>();                   // this step's group has landed (this thread's copies) ...
            __syncthreads();                                  // ... everyone's; and the buffer of the last step is free
            stage(buf == 0 ? CS_STAGES - 1 : buf - 1);
            cx<T> a[RL], bb[RM];
#pragma unroll
            for (int i = 0; i < RL; ++i) a[i] = slab[buf][0][tl + TL * i][fi];
#pragma unroll
            for (int j = 0; j < RM; ++j) bb[j] = slab[buf][1][tm + TM * j][fi];
            if (t == 0) {
#pragma unroll
                for (int i = 0; i < RL; ++i)
#pragma unroll
                    for (int j = 0; j < RM; ++j) {
                        const T re = fma_rn(a[i].x, bb[j].x, mul_rn(a[i].y, bb[j].y));
                        const T im = fma_rn(a[i].y, bb[j].x, -mul_rn(a[i].x, bb[j].y));
                        p[i][j] = mkc<T>(mul_rn(cf, re), mul_rn(cf, im));
                    }
            } else {
#pragma unroll
                for (int i = 0; i < RL; ++i)
#pragma unroll
                    for (int j = 0; j < RM; ++j) {
                        const T re = fma_rn(a[i].x, bb[j].x, mul_rn(a[i].y, bb[j].y));
                        const T im = fma_rn(a[i].y, bb[j].x, -mul_rn(a[i].x, bb[j].y));
                        p[i][j] = mkc<T>(fma_rn(cf, re, p[i][j].x), fma_rn(cf, im, p[i][j].y));
                    }
            }
            if (t + 1 == ntapers) {
                const bool first = fresh && e == 0;
#pragma unroll
                for (int i = 0; i < RL; ++i)
#pragma unroll
                    for (int j = 0; j < RM; ++j)
                        sum[i][j] = first ? p[i][j] : mkc<T>(sum[i][j].x + p[i][j].x, sum[i][j].y + p[i][j].y);
            }
            buf = buf + 1 == CS_STAGES ? 0 : buf + 1;
        }
    }
    if (!fout) return;
    const T d = (T)divisor;
#pragma unroll
    for (int i = 0; i < RL; ++i)
#pragma unroll
        for (int j = 0; j < RM; ++j) {
            const int64_t l = l0 + tl + TL * i, m = m0 + tm + TM * j;
            if (l < nchan && m < nchan) o[l + nchan * m] = divisor > 1 ? mkc<T>(sum[i][j].x / d, sum[i][j].y / d) : sum[i][j];
        }
}

// coherence_from_cs!, src/multitaper.jl:672-693: |S_lm| / sqrt(real(S_ll * S_mm)) from the lower triangle, unit diagonal
template <typename T>
__global__ void coherence_kernel(T* __restrict__ out, const cx<T>* __restrict__ cs, int64_t nchan, int64_t nf) {
    const int64_t total = nf * nchan * nchan;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t l = i % nchan, m = (i / nchan) % nchan, f = i / (nchan * nchan);
        if (l == m) { out[i] = T(1); continue; }
        const int64_t hi = l > m ? l : m, lo = l > m ? m : l;
        const cx<T>* S = cs + f * nchan * nchan;
        const cx<T> s = S[hi + lo * nchan], d1 = S[hi + hi * nchan], d2 = S[lo + lo * nchan];
        out[i] = sqrt(s.x * s.x + s.y * s.y) / sqrt(d1.x * d2.x - d1.y * d2.y);
    }
}

// 2-D periodogram (src/periodograms.jl:175-232, 473-509).  X is the half spectrum of the zero-padded real matrix,
// (n1/2+1) x n2 column-major (first dimension halved, as rfft does).
// ptype 0: out[i, j] = |X_full[i, j]|^2 * m1 over the full n1 x n2 grid (fft2pow2!), conjugate symmetry for i > n1/2.
template <typename T>
__global__ void per2_full_kernel(const cx<T>* __restrict__ X, int64_t n1, int64_t n2, T m1, T* __restrict__ out) {
    const int64_t h = n1 / 2 + 1, total = n1 * n2;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = idx % n1, j = idx / n1;
        const cx<T> v = i < h ? X[i + h * j] : X[(n1 - i) + h * ((n2 - j) % n2)];
        out[idx] = cabs2(v) * m1;
    }
}
// radial forms (fft2pow2radial!): every half-spectrum bin adds |X|^2 * m to its integer wavenumber ring, m = 1/r on the
// rows i = 1 and (n1 even) i = n1/2+1 that have no mirror image, 2/r elsewhere; rings and ring populations are
// accumulated with atomics in Float64 / Int64 (the reference adds in the signal precision, column by column).
template <typename T>
__global__ void per2_radial_kernel(const cx<T>* __restrict__ X, int64_t n1, int64_t n2, double c1, double c2, double m1, double m2,
                                   int64_t kmax, double* __restrict__ acc, unsigned long long* __restrict__ wc) {
    const int64_t h = n1 / 2 + 1, total = h * n2;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = idx % h, j = idx / h;                      // 0-based
        const int64_t kj1 = j <= n2 / 2 ? j : j - n2;
        const double kj = (double)kj1 * c2, a = c1 * (double)i;
        const int64_t wavenum = (int64_t)rint(sqrt(fma(a, a, kj * kj)));    // round(Int, .), ties to even; 0-based ring
        if (wavenum >= kmax) continue;
        const bool single = (i == 0) || (i == h - 1 && n1 % 2 == 0);
        atomicAdd(&acc[wavenum], (double)cabs2(X[idx]) * (single ? m1 : m2));
        atomicAdd(&wc[wavenum], single ? 1ull : 2ull);
    }
}
template <typename T>
__global__ void per2_radial_finish_kernel(const double* __restrict__ acc, const unsigned long long* __restrict__ wc, int64_t kmax,
                                          int average, T* __restrict__ out) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < kmax) out[k] = (T)(average ? acc[k] / (double)wc[k] : acc[k]);
}
// zero-padded copy of the n1 x n2 signal into the nfft1 x nfft2 transform buffer
template <typename T>
__global__ void per2_pad_kernel(const T* __restrict__ s, int64_t n1, int64_t n2, T* __restrict__ dst, int64_t f1, int64_t f2) {
    const int64_t total = f1 * f2;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = idx % f1, j = idx / f1;
        dst[idx] = (i < n1 && j < n2) ? s[i + n1 * j] : T(0);
    }
}

// ---------------------------------------------------------------------------------------------- streaming Welch
// Fused sizes: the partial rows of one call's two batched transform launches (welch_fused_kernel<..., BATCH = true>),
// channel blockIdx.y, summed in Float64 and written (add = 0) or added to column blockIdx.y of acc (nout x nchan).  The
// interior launch's ri rows are summed in welch_finalize_kernel's order -- warp sl of nw = min(ri, 32) sums rows sl, sl + nw,
// ..., then the warps' sums are added in order -- and then the seam launch's rs rows the same way, and the two sums are added.
// So a call with no seam rows puts into acc exactly the sum the one-shot finalize kernel scales.  Real input: bin k sums
// rows k and N - k of the two-for-one transform; welch_stream_power_kernel applies the factor 1/2.
template <typename T, int N>
__global__ void __launch_bounds__(1024) welch_stream_reduce_kernel(const T* __restrict__ seam_rows, int rs,
                                                                   const T* __restrict__ rows, int ri, double* __restrict__ acc,
                                                                   int nout, int real_in, int add) {
    __shared__ double red[2][32][33];
    const int b = threadIdx.x & 31, sl = threadIdx.x >> 5;
    const int k = blockIdx.x * 32 + b;
    auto part = [&](const T* base, int nrows, int which) {
        const int nw = nrows < 32 ? nrows : 32;
        double sum = 0.0;
        if (k < nout && sl < nw) {
            const T* chan = base + (int64_t)blockIdx.y * nrows * N;
            const T* c0 = chan + k;
            const T* c1 = chan + ((N - k) & (N - 1));
            if (real_in) {
                for (int c = sl; c < nrows; c += nw) sum += (double)c0[(int64_t)c * N] + (double)c1[(int64_t)c * N];
            } else {
                for (int c = sl; c < nrows; c += nw) sum += (double)c0[(int64_t)c * N];
            }
        }
        red[which][sl][b] = sum;
    };
    part(rows, ri, 0);
    part(seam_rows, rs, 1);
    __syncthreads();
    if (sl == 0 && k < nout) {
        const int nwi = ri < 32 ? ri : 32, nws = rs < 32 ? rs : 32;
        double sum = red[0][0][b];
        for (int i = 1; i < nwi; ++i) sum += red[0][i][b];
        if (rs > 0) {
            double s2 = red[1][0][b];
            for (int i = 1; i < nws; ++i) s2 += red[1][i][b];
            sum += s2;
        }
        double* q = acc + (int64_t)blockIdx.y * nout + k;
        *q = add ? *q + sum : sum;
    }
}

// cuFFT sizes: the spectra of (channel, segment) pairs f0 .. f0 + nf - 1 (f = c k + j, batch slot f - f0) into acc.  Thread
// (bin kk, channel f0 / k + blockIdx.y) sums |X|^2 over its channel's slots in segment order, then writes the sum (add = 0
// and the channel's first pair is in this batch) or adds it.  Two-sided real output: bin kk >= nbins_fft reads nfft - kk.
template <typename T>
__global__ void welch_stream_acc_kernel(const cx<T>* __restrict__ X, int64_t nbins_fft, int64_t nfft, int64_t nout, int64_t f0,
                                        int64_t nf, int64_t k, int add, double* __restrict__ acc) {
    const int64_t kk = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (kk >= nout) return;
    const int64_t c = f0 / k + blockIdx.y;
    const int64_t a = c * k > f0 ? c * k : f0, e = (c + 1) * k < f0 + nf ? (c + 1) * k : f0 + nf;
    const int64_t src = kk < nbins_fft ? kk : nfft - kk;
    double sum = 0.0;
    for (int64_t f = a; f < e; ++f) sum += (double)cabs2(X[(f - f0) * nbins_fft + src]);
    double* q = acc + c * nout + kk;
    *q = (add || a > c * k) ? *q + sum : sum;
}

// Power of a Float64 accumulation, column blockIdx.y: the fft2pow! scale (m1 = 1/r, m2 = 2/r; :142-172) of welch_finalize_kernel
// (half: fused real plans, whose acc holds twice the power); every cuFFT-size Welch and mt_pgram ends here
template <typename T>
__global__ void welch_stream_power_kernel(const double* __restrict__ acc, int64_t nout, int64_t nfft, int onesided, int half,
                                          double m1, double m2, T* __restrict__ out) {
    const int64_t kk = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (kk >= nout) return;
    const int64_t i = (int64_t)blockIdx.y * nout + kk;
    double sum = acc[i];
    if (half) sum *= 0.5;
    const double m = (onesided && kk != 0 && 2 * kk != nfft) ? m2 : m1;
    out[i] = (T)(sum * m);
}

// ---------------------------------------------------------------------------------------------- dispatch
static bool fused_size_ok(int64_t nfft, bool f64) {
    if (nfft < 256 || (nfft & (nfft - 1))) return false;
    return nfft <= (f64 ? 8192 : 16384);
}

// Calls f(T(), std::integral_constant<int, N>()) with T the plan's real eltype and N = nfft, for the sizes that have fused
// kernels (fused_size_ok); otherwise sets the "no fused <what> kernel" error
template <typename T, typename F> static int fused_size_dispatch(const SpecPlanImpl* p, const char* what, F&& f) {
    switch (p->nfft) {
#define X(NN)                                                                                               \
    case NN:                                                                                                \
        if constexpr (sizeof(T) == 8 && NN > 8192) break;                                                   \
        else return f(T(0), std::integral_constant<int, NN>());
        X(256) X(512) X(1024) X(2048) X(4096) X(8192) X(16384)
#undef X
    }
    set_error("no fused %s kernel for nfft=%lld", what, (long long)p->nfft);
    return DSPB200_EUNSUPPORTED;
}
template <typename F> static int fused_dispatch(const SpecPlanImpl* p, const char* what, F&& f) {
    return p->f64 ? fused_size_dispatch<double>(p, what, f) : fused_size_dispatch<float>(p, what, f);
}

template <typename K> static int set_smem(K kernel, size_t bytes) {
    if (bytes > 48 * 1024) DSP_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    return DSPB200_OK;
}

template <typename T, bool BATCH>
using welch_kern_t = void (*)(const void*, welch_arg<BATCH, int64_t>, welch_arg<!BATCH, int64_t>, int64_t,
                              welch_arg<BATCH, int64_t>, welch_arg<BATCH, int64_t>, welch_arg<BATCH, int>,
                              welch_arg<BATCH, int64_t>, int64_t, int, welch_arg<!BATCH, int64_t>,
                              const typename win_t<T>::type*, const cx<T>*, const cx<T>*, const cx<T>*, T*,
                              welch_arg<!BATCH, int>);

// The fused Welch instances (MODE: staging / window placement, G: thread groups per CTA) in order of preference (measured
// sweep): f(kernel, shared-memory bytes, MODE, G) for each one that may run on TMA-`aligned` segments with(out) a window, the
// direct-load instance last.  These are all the instances there are; dspb200_spec_plan_pin_welch names them from this list.
// TAPERS (mt_pgram): a window row per unit, which MODE 2 / 3 (one window, staged once per CTA) cannot address.
template <typename T, int N, bool CPLX, bool BATCH, bool TAPERS, typename F>
static int welch_candidates(const SpecPlanImpl* p, bool aligned, bool windowed, F&& f) {
    constexpr bool MULTI = sizeof(T) == 4 && N >= 1024 && N <= 4096;       // sizes that get multi-group variants
    constexpr bool WREGOK = sizeof(T) == 4 && N <= 4096;                   // window in registers: 32 extra registers per thread
#define DSP_WELCH_CAND(MODE_, G_)                                                                                   \
    DSP_TRY(f(welch_kern_t<T, BATCH>(welch_fused_kernel<T, N, CPLX, MODE_, G_, BATCH, TAPERS>),                     \
              welch_layout<T, N, CPLX, MODE_>::total(p->n, p->hop, G_), MODE_, G_))
    if (aligned) {
        if constexpr (!TAPERS) {
            if (windowed) {
                if constexpr (CPLX) {
                    // complex: two CTAs per SM with the window in registers, then in shared memory
                    if constexpr (WREGOK) DSP_WELCH_CAND(3, 1);
                    DSP_WELCH_CAND(2, 1);
                    if constexpr (MULTI) { DSP_WELCH_CAND(3, 2); DSP_WELCH_CAND(2, 2); }
                } else {
                    // real: three thread groups sharing tables + window, then two, then two CTAs
                    if constexpr (MULTI) { DSP_WELCH_CAND(2, 3); DSP_WELCH_CAND(2, 2); }
                    DSP_WELCH_CAND(2, 1);
                    if constexpr (WREGOK) DSP_WELCH_CAND(3, 1);
                }
            }
        }
        if constexpr (MULTI && !CPLX) DSP_WELCH_CAND(1, 3);
        DSP_WELCH_CAND(1, 1);
        if constexpr (MULTI) DSP_WELCH_CAND(1, 2);
    }
    DSP_WELCH_CAND(0, 1);
#undef DSP_WELCH_CAND
    return DSPB200_OK;
}

// Resident CTAs per SM of a G-group instance; row_cap > 0 bounds one wave to that many virtual CTAs
template <typename K>
static int welch_per_sm(const SpecPlanImpl* p, K k, int threads, int g, size_t smem, int64_t row_cap, int* per_sm) {
    DSP_TRY(set_smem(k, smem));
    DSP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, k, threads, smem));
    if (row_cap > 0 && (int64_t)*per_sm * g * p->sm_count > row_cap) *per_sm = (int)(row_cap / ((int64_t)g * p->sm_count));
    return DSPB200_OK;
}

// Launch configuration of the fused Welch kernel, chosen once per (plan, path, alignment class) into `cfg`: every candidate
// that fits is rated by the warps it keeps resident per SM (occupancy calculator x G); the first one that keeps at least 12
// is taken, otherwise the one with the most, and the direct-load instance only when no other fits.  The selection walks up
// to nine instances through cudaFuncSetAttribute + the occupancy calculator (tens of microseconds), hence the cache.
// row_cap: the single-signal path's `nparts` (one wave never has more virtual CTAs than `partial` has rows), 0 for a batch.
template <typename T, int N, bool CPLX, bool BATCH, bool TAPERS = false>
static int welch_select(SpecPlanImpl* p, SpecPlanImpl::WelchCfg& cfg, bool aligned, int64_t row_cap) {
    if (cfg.kern != nullptr) return DSPB200_OK;
    constexpr int NT = fft_threads<N>::value;
    using Kern = welch_kern_t<T, BATCH>;
    struct Cand { Kern k; size_t smem; int mode, g, warps, per_sm; };
    Cand best{nullptr, 0, 0, 0, -1, 0};
    auto consider = [&](Kern k, size_t smem, int mode, int g) -> int {
        if (best.warps >= 12 || (mode == 0 && best.k != nullptr)) return DSPB200_OK;
        if (smem > p->smem_optin) return DSPB200_OK;
        int per_sm = 0;
        DSP_TRY(welch_per_sm(p, k, NT * g, g, smem, row_cap, &per_sm));
        if (per_sm < 1) return DSPB200_OK;
        const int warps = per_sm * g * NT / 32;
        if (warps > best.warps) best = Cand{k, smem, mode, g, warps, per_sm};
        return DSPB200_OK;
    };
    DSP_TRY((welch_candidates<T, N, CPLX, BATCH, TAPERS>(p, aligned, p->d_window != nullptr, consider)));
    DSP_REQUIRE(best.k != nullptr, "no %sWelch kernel configuration fits (nfft=%lld)", BATCH ? "batched " : "", (long long)p->nfft);
    DSP_TRY(set_smem(best.k, best.smem));              // (the last candidate examined may have left a different limit)
    cfg.kern = reinterpret_cast<void*>(best.k); cfg.smem = best.smem; cfg.g = best.g; cfg.per_sm = best.per_sm;
    cfg.threads = NT * best.g; cfg.mode = best.mode;
    return DSPB200_OK;
}

// CTAs of one resident wave of the chosen instance, or the pinned number of virtual CTAs / G
static int64_t welch_wave(const SpecPlanImpl* p, const SpecPlanImpl::WelchCfg& cfg) {
    return cfg.vctas ? cfg.vctas / cfg.g : (int64_t)p->sm_count * cfg.per_sm;
}

// Launch the chosen instance on the CTAs that `work` units (one signal) or items (batch) need at G per CTA, at most one wave
template <typename T, bool BATCH>
static int welch_launch(SpecPlanImpl* p, SpecPlanImpl::WelchCfg& cfg, int64_t work, const void* s,
                        welch_arg<BATCH, int64_t> chan_stride, welch_arg<!BATCH, int64_t> seg0, int64_t nseg,
                        welch_arg<BATCH, int64_t> upc, welch_arg<BATCH, int64_t> per, welch_arg<BATCH, int> slices,
                        welch_arg<BATCH, int64_t> nitems, welch_arg<!BATCH, int64_t> sample_offset, void* partial,
                        welch_arg<!BATCH, int> fresh_from, cudaStream_t st) {
    const int64_t wave = welch_wave(p, cfg), want = cdiv(work, cfg.g);
    const int grid = (int)(want < wave ? want : wave);
    DSP_CUDA(launch_pdl(reinterpret_cast<welch_kern_t<T, BATCH>>(cfg.kern), (unsigned)grid, (unsigned)cfg.threads, cfg.smem, st,
                        s, chan_stride, seg0, nseg, upc, per, slices, nitems, p->hop, (int)p->n, sample_offset,
                        reinterpret_cast<const typename win_t<T>::type*>(p->d_window), reinterpret_cast<const cx<T>*>(p->d_tw),
                        reinterpret_cast<const cx<T>*>(p->d_t16), reinterpret_cast<const cx<T>*>(p->d_t256),
                        reinterpret_cast<T*>(partial), fresh_from));
    DSP_LAUNCH_OK();
    cfg.used = (int64_t)grid * cfg.g;
    return DSPB200_OK;
}

// One signal: segments seg0 .. seg0 + nseg - 1 of the buffer s (whose first sample is the signal's sample_offset), added to
// the partial rows of the accumulation open since welch_begin
template <typename T, int N, bool CPLX>
static int launch_welch_fused(SpecPlanImpl* p, const void* s, int64_t seg0, int64_t nseg, int64_t sample_offset,
                              cudaStream_t st) {
    using In = typename in_type<T, CPLX>::type;
    // TMA staging needs 16-byte aligned segment starts and sizes
    const uintptr_t first = (uintptr_t)s + (uintptr_t)((seg0 * p->hop - sample_offset) * (int64_t)sizeof(In));
    const bool aligned = (first % 16 == 0) && ((p->hop * sizeof(In)) % 16 == 0) && ((p->n * sizeof(In)) % 16 == 0);
    const int64_t units = CPLX ? nseg : (nseg + 1) / 2;
    if (units < 1) return DSPB200_OK;
    SpecPlanImpl::WelchCfg& cfg = p->welch_cfg[aligned ? 1 : 0];
    DSP_TRY((welch_select<T, N, CPLX, false>(p, cfg, aligned, p->nparts)));
    // a pinned number of virtual CTAs runs in full, past the units if need be
    DSP_TRY((welch_launch<T, false>(p, cfg, cfg.vctas ? cfg.vctas : units, s, Nil(), seg0, nseg, Nil(), Nil(), Nil(), Nil(),
                                    sample_offset, p->partial.p, p->rows_used, st)));
    if (cfg.used > p->rows_used) p->rows_used = (int)cfg.used;
    return DSPB200_OK;
}

template <typename T, int N>
static int launch_welch_finalize(SpecPlanImpl* p, double r, void* out, cudaStream_t st) {
    // one channel, 32 warps
    DSP_CUDA(launch_pdl(welch_finalize_kernel<T, N>, (unsigned)cdiv(p->nout, 32), 1024u, (size_t)0, st,
                        reinterpret_cast<const T*>(p->partial.p), p->rows_used, reinterpret_cast<T*>(out), (int)p->nout,
                        p->cplx ? 0 : 1, (int)p->onesided, 1.0 / r, 2.0 / r));
    DSP_LAUNCH_OK();
    return DSPB200_OK;
}

// Partial rows of the batched Welch path: at most this many bytes per plan, in a buffer of its own (a streaming accumulation
// open on the plan keeps its rows).  A batch whose channels need more rows runs in channel groups.
static constexpr size_t WELCH_BATCH_SCRATCH = (size_t)32 << 20;

// Slices per channel for `gc` channels of `upc` units on `nv` virtual CTAs: the split whose busiest virtual CTA runs the fewest
// units (items per virtual CTA x units per item), the fewest slices on ties, at most `max_slices`.  Every slice is non-empty.
static int64_t welch_batch_slices(int64_t gc, int64_t upc, int64_t nv, int64_t max_slices) {
    int64_t lim = upc < max_slices ? upc : max_slices;
    if (lim > 2 * nv) lim = 2 * nv;
    int64_t best = 1, best_cost = cdiv(gc, nv) * upc;
    for (int64_t sl = 2; sl <= lim; ++sl) {
        const int64_t per = cdiv(upc, sl);
        if (cdiv(upc, per) != sl) continue;                  // same split as a smaller slice count
        const int64_t cost = cdiv(gc * sl, nv) * per;
        if (cost < best_cost) { best = sl; best_cost = cost; }
    }
    return best;
}

// TMA staging of a batched launch needs every unit start 16-byte aligned: the base, the channel stride (launch_stft_fused's
// rule), hop and n
static bool welch_batch_aligned(const SpecPlanImpl* p, const void* s, int64_t stride, int64_t nchan, size_t esz) {
    return ((uintptr_t)s % 16 == 0) && ((stride * (int64_t)esz) % 16 == 0 || nchan == 1) && ((p->hop * (int64_t)esz) % 16 == 0) &&
           ((p->n * (int64_t)esz) % 16 == 0);
}

// One batched transform launch (welch_fused_kernel<..., BATCH = true>) over gc channels of k segments each: the channels are
// sliced for the resident virtual CTAs of `cfg`, at most max_slices slices per channel, one partial row per (channel, slice)
struct WelchBatchWork { int64_t k = 0, upc = 0, slices = 0, per = 0, nitems = 0; };
static WelchBatchWork welch_batch_work(const SpecPlanImpl* p, const SpecPlanImpl::WelchCfg& cfg, bool cplx, int64_t gc, int64_t k,
                                       int64_t max_slices) {
    WelchBatchWork w;
    w.k = k;
    w.upc = cplx ? k : (k + 1) / 2;
    w.slices = welch_batch_slices(gc, w.upc, welch_wave(p, cfg) * cfg.g, max_slices);
    w.per = cdiv(w.upc, w.slices);
    w.nitems = gc * w.slices;
    return w;
}
// channel c's first sample at s + c * stride; rows: w.nitems rows of N
template <typename T, bool CPLX>
static int welch_batch_launch(SpecPlanImpl* p, SpecPlanImpl::WelchCfg& cfg, const WelchBatchWork& w, const void* s, int64_t stride,
                              void* rows, cudaStream_t st) {
    return welch_launch<T, true>(p, cfg, w.nitems, s, stride, Nil(), w.k, w.upc, w.per, (int)w.slices, w.nitems, Nil(), rows, Nil(),
                                 st);
}

// Batched Welch over the nchan columns of a len x nchan matrix (k segments each): one kernel and one finalize launch per
// channel group
template <typename T, int N, bool CPLX>
static int launch_welch_batch(SpecPlanImpl* p, const void* s, int64_t len, int64_t nchan, int64_t k, double r, void* out,
                              cudaStream_t st) {
    using In = typename in_type<T, CPLX>::type;
    const bool aligned = welch_batch_aligned(p, s, len, nchan, sizeof(In));
    SpecPlanImpl::WelchCfg& cfg = p->welch_batch_cfg[aligned ? 1 : 0];
    DSP_TRY((welch_select<T, N, CPLX, true>(p, cfg, aligned, 0)));
    const int64_t rows_cap = (int64_t)(WELCH_BATCH_SCRATCH / ((size_t)N * sizeof(T)));
    const int64_t gc_max = nchan < rows_cap ? nchan : rows_cap;
    for (int64_t c0 = 0; c0 < nchan; c0 += gc_max) {
        const int64_t gc = nchan - c0 < gc_max ? nchan - c0 : gc_max;
        const WelchBatchWork w = welch_batch_work(p, cfg, CPLX, gc, k, rows_cap / gc);
        const int64_t slices = w.slices;
        DSP_TRY(p->bpartial.reserve((size_t)w.nitems * N * sizeof(T)));
        DSP_TRY((welch_batch_launch<T, CPLX>(p, cfg, w, (const In*)s + c0 * len, len, p->bpartial.p, st)));
        const int nw = slices < 32 ? (int)slices : 32;
        welch_finalize_kernel<T, N><<<dim3((unsigned)cdiv(p->nout, 32), (unsigned)gc), 32 * nw, 0, st>>>(
            reinterpret_cast<const T*>(p->bpartial.p), (int)slices, reinterpret_cast<T*>(out) + c0 * p->nout, (int)p->nout,
            CPLX ? 0 : 1, (int)p->onesided, 1.0 / r, 2.0 / r);
        DSP_LAUNCH_OK();
    }
    return DSPB200_OK;
}

// The history side of an STFT call (dspb200_stft_stream_exec_dev); a one-shot call has none and ldo = k
// (seam, lds: the copy of every channel's first virtual-column samples that the edge kernel wrote; fused sizes only).
// keep_plan: run the instance an aligned call of the plan runs, whatever the alignment of this call (streams)
// ntapers > 0: an mt_spectrogram call -- PSD columns summed over the plan's taper rows in one launch (WIN == 2 instances).
struct StftStreamArgs {
    const void* hist = nullptr; int64_t h = 0, ldh = 0, ldo = 0; const void* seam = nullptr; int64_t lds = 0;
    bool keep_plan = false;
    int ntapers = 0;
};

// k segments of each channel's virtual column [history; s], s being the len x nchan chunk (one-shot: the whole matrix).  A
// stream keeps its plan's instance (sa.keep_plan): stft_w1k_kernel rounds differently from stft_fused_kernel, and the two
// TMA / direct instances of stft_fused_kernel round alike.  A one-shot Float32 1024-point call runs stft_w1k_kernel only
// when it meets the TMA alignment conditions.
template <typename T, int N, bool CPLX>
static int launch_stft_fused(SpecPlanImpl* p, const void* s, int64_t len, int64_t nchan, int64_t k, double r,
                             int psd_only, void* out, cudaStream_t st, const StftStreamArgs& sa) {
    constexpr int NT = fft_threads<N>::value;
    using In = typename in_type<T, CPLX>::type;
    using SS = StftStream<In>;
    const size_t base = (size_t)fft_smem_elems<T, N>() * sizeof(cx<T>);
    const size_t stage = (size_t)(CPLX ? p->n : p->hop + p->n) * sizeof(In) + 16;
    // Float32, N = 1024: every call that meets the TMA alignment conditions runs stft_w1k_kernel (its shared memory is at
    // most about 84 KB), so the fallback below is the direct-load instance alone
    constexpr bool W1K = sizeof(T) == 4 && N == 1024;
    const bool plan_aligned = ((p->hop * sizeof(In)) % 16 == 0) && ((p->n * sizeof(In)) % 16 == 0);
    // the TMA alignment conditions: 16-byte aligned unit starts (streaming: x + start - h) and sizes
    const bool aligned = plan_aligned && ((uintptr_t)s % 16 == 0) && ((len * sizeof(In)) % 16 == 0 || nchan == 1) &&
                         (sa.h * sizeof(In)) % 16 == 0;
    const bool tma = !W1K && aligned &&
                     (base + stage <= p->smem_optin) && (base + stage <= 100 * 1024 || N >= 8192);   // N >= 8192: one CTA per SM anyway
    const size_t smem = tma ? base + stage : base;
    const int64_t upc = CPLX ? k : (k + 1) / 2;
    const int64_t units = upc * nchan;
    if (units < 1) return DSPB200_OK;
    const SS ss{reinterpret_cast<const In*>(sa.seam), sa.lds, sa.h, sa.ldo, (W1K ? aligned : tma) ? 1 : 0, sa.ntapers};
    const auto* w = reinterpret_cast<const typename win_t<T>::type*>(p->d_window);
    const bool mt = sa.ntapers > 0;
    if constexpr (W1K) {
        // one warp per unit (stft_w1k_kernel): a one-shot call needs the TMA alignment conditions, a stream those of its plan
        if ((sa.keep_plan ? plan_aligned : aligned) && p->d_t32 != nullptr) {
            constexpr int WARPS = 4;
            const size_t smem1 = (size_t)w1k::T32_LEN * sizeof(cx<float>) + (w && !mt ? (size_t)p->n * sizeof(float2) : 0) +
                                 (size_t)WARPS * w1k::warp_bytes(CPLX ? p->n : p->hop + p->n, sizeof(In));
            using K1 = void (*)(const void*, int64_t, int64_t, int64_t, int64_t, int64_t, int, const float2*, const cx<float>*, void*, int,
                                int, int, float, float, SS);
            K1 k1 = mt ? (K1)stft_w1k_kernel<CPLX, 2, WARPS> : w ? (K1)stft_w1k_kernel<CPLX, 1, WARPS> : (K1)stft_w1k_kernel<CPLX, 0, WARPS>;
            if (smem1 <= p->smem_optin) {
                DSP_TRY(set_smem(k1, smem1));
                int per = 1;
                DSP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, k1, 32 * WARPS, smem1));
                const int64_t cap1 = (int64_t)p->sm_count * (per < 1 ? 1 : per);
                const int64_t want = cdiv(units, WARPS);
                const unsigned grid1 = (unsigned)(want < cap1 ? want : cap1);
                k1<<<grid1, 32 * WARPS, smem1, st>>>(s, len, k, upc, units, p->hop, (int)p->n, reinterpret_cast<const float2*>(w),
                                                      reinterpret_cast<const cx<float>*>(p->d_t32), out, (int)p->nout, psd_only,
                                                      p->onesided, (float)(1.0 / r), (float)(2.0 / r), ss);
                DSP_LAUNCH_OK();
                return DSPB200_OK;
            }
        }
    }
    const auto* tw = reinterpret_cast<const cx<T>*>(p->d_tw);
    const auto* g16 = reinterpret_cast<const cx<T>*>(p->d_t16);
    const auto* g256 = reinterpret_cast<const cx<T>*>(p->d_t256);
    using Kern = void (*)(const void*, int64_t, int64_t, int64_t, int64_t, int64_t, int, const typename win_t<T>::type*, const cx<T>*,
                          const cx<T>*, const cx<T>*, void*, int, int, int, T, T, SS);
    // window presence is a compile-time property of the Float32 kernels (predicated-off window products still issue)
    constexpr bool SPEC = sizeof(T) == 4;
    Kern kern;
    if (mt) {
        if constexpr (W1K) kern = (Kern)stft_fused_kernel<T, N, CPLX, false, 2>;
        else kern = tma ? (Kern)stft_fused_kernel<T, N, CPLX, true, 2> : (Kern)stft_fused_kernel<T, N, CPLX, false, 2>;
    } else if constexpr (W1K) {
        kern = w ? (Kern)stft_fused_kernel<T, N, CPLX, false, 1> : (Kern)stft_fused_kernel<T, N, CPLX, false, 0>;
    } else if constexpr (SPEC) {
        if (tma) kern = w ? (Kern)stft_fused_kernel<T, N, CPLX, true, 1> : (Kern)stft_fused_kernel<T, N, CPLX, true, 0>;
        else kern = w ? (Kern)stft_fused_kernel<T, N, CPLX, false, 1> : (Kern)stft_fused_kernel<T, N, CPLX, false, 0>;
    } else {
        kern = tma ? (Kern)stft_fused_kernel<T, N, CPLX, true, -1> : (Kern)stft_fused_kernel<T, N, CPLX, false, -1>;
    }
    DSP_TRY(set_smem(kern, smem));
    int per_sm = 1;
    DSP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, NT, smem));
    const int64_t cap = (int64_t)p->sm_count * (per_sm < 1 ? 1 : per_sm);
    const unsigned grid = (unsigned)(units < cap ? units : cap);
    kern<<<grid, NT, smem, st>>>(s, len, k, upc, units, p->hop, (int)p->n, w, tw, g16, g256, out, (int)p->nout, psd_only,
                                 p->onesided, (T)(1.0 / r), (T)(2.0 / r), ss);
    DSP_LAUNCH_OK();
    return DSPB200_OK;
}

// Pinned Welch launch configuration (dspb200_spec_plan_pin_welch, a testing aid): any instance of welch_candidates.  Fills
// both alignment classes of the cache: aligned calls get (mode, g), unaligned ones MODE 0, G = 1; both `vctas`.
template <typename T, int N, bool CPLX, bool BATCH, bool TAPERS = false>
static int welch_pin(SpecPlanImpl* p, int mode, int g, int64_t vctas) {
    constexpr int NT = fft_threads<N>::value;
    using Kern = welch_kern_t<T, BATCH>;
    SpecPlanImpl::WelchCfg pinned[2];
    for (int a = 0; a < 2; ++a) {
        const int m = a ? mode : 0, gg = a ? g : 1;
        Kern k = nullptr;
        size_t smem = 0;
        DSP_TRY((welch_candidates<T, N, CPLX, BATCH, TAPERS>(p, true, true, [&](Kern kc, size_t sc, int mc, int gc) -> int {
            if (mc == m && gc == gg) { k = kc; smem = sc; }
            return DSPB200_OK;
        })));
        if (k == nullptr) {
            set_error("no Welch kernel instance MODE %d, G %d for this plan (nfft=%lld)", m, gg, (long long)N);
            return DSPB200_EUNSUPPORTED;
        }
        if (m >= 2 && p->d_window == nullptr) {           // MODE 2 / 3 stage the window table
            set_error("Welch MODE %d needs a window", m);
            return DSPB200_EUNSUPPORTED;
        }
        if (smem > p->smem_optin) {
            set_error("Welch MODE %d, G %d needs %zu bytes of shared memory (limit %zu)", m, gg, smem, p->smem_optin);
            return DSPB200_EUNSUPPORTED;
        }
        int per_sm = 0;
        DSP_TRY(welch_per_sm(p, k, NT * gg, gg, smem, !BATCH && vctas == 0 ? p->nparts : 0, &per_sm));
        if (per_sm < 1) {
            set_error("Welch MODE %d, G %d does not fit an SM", m, gg);
            return DSPB200_EUNSUPPORTED;
        }
        pinned[a].kern = reinterpret_cast<void*>(k); pinned[a].smem = smem; pinned[a].g = gg; pinned[a].per_sm = per_sm;
        pinned[a].threads = NT * gg; pinned[a].mode = m; pinned[a].vctas = vctas;
    }
    SpecPlanImpl::WelchCfg* cfg = TAPERS ? p->welch_mt_cfg : BATCH ? p->welch_batch_cfg : p->welch_cfg;
    cfg[0] = pinned[0];
    cfg[1] = pinned[1];
    return DSPB200_OK;
}

// ---------------------------------------------------------------------------------------------- generic path
static int generic_prepare(SpecPlanImpl* p) {
    if (p->fft_ok) return DSPB200_OK;
    int64_t b = (int64_t(1) << 22) / p->nfft;
    if (b < 1) b = 1;
    if (b > 8192) b = 8192;
    p->batch = b;
    DSP_TRY(fft_plan_1d(&p->fft, p->cplx, p->f64, CUFFT_FORWARD, p->nfft, b));
    p->fft_ok = true;
    const size_t esz = dtype_size(p->dtype);
    DSP_TRY(p->segbuf.reserve((size_t)(b * p->nfft) * esz));
    DSP_TRY(p->specbuf.reserve((size_t)(b * p->nbins_fft) * (p->f64 ? 16 : 8)));
    DSP_TRY(p->acc.reserve((size_t)p->nout * sizeof(double)));
    return DSPB200_OK;
}

// Streaming calls, cuFFT sizes: blocks along one grid row per batch slot, enough for about 16 waves of the whole batch
static unsigned stream_generic_cols(const SpecPlanImpl* p, int64_t len, int threads) {
    const int64_t want = cdiv(len, threads), cap = cdiv((int64_t)p->sm_count * 16, p->batch);
    return (unsigned)(want < cap ? want : cap);
}

// seg_window_kernel of the plan's element type (T: its real type) into buf, 256 threads per block
template <typename T> static int seg_window_launch(const SpecPlanImpl* p, dim3 grid, const void* hist, int64_t h, int64_t ldh,
                                                    const void* x, int64_t nx, int64_t f0, int64_t nf, int64_t k, int64_t hop,
                                                    int64_t wstride, void* buf, cudaStream_t st) {
    const auto* w = reinterpret_cast<const typename win_t<T>::type*>(p->d_window);
    if (p->cplx)
        seg_window_kernel<T, true><<<grid, 256, 0, st>>>(hist, h, ldh, x, nx, f0, nf, k, hop, p->n, p->nfft, w, wstride, buf);
    else
        seg_window_kernel<T, false><<<grid, 256, 0, st>>>(hist, h, ldh, x, nx, f0, nf, k, hop, p->n, p->nfft, w, wstride, buf);
    DSP_LAUNCH_OK();
    return DSPB200_OK;
}

// The spectra of (channel, segment) pairs f0 .. f0 + nf - 1 of the virtual columns [hist; x] (f = c k + j) in the plan's
// batch buffer: seg_window_kernel (segments hop samples apart, windows wstride values apart), then the plan's cuFFT transform
template <typename T> static int stream_generic_fft(SpecPlanImpl* p, const void* hist, int64_t h, int64_t ldh, const void* x,
                                                     int64_t nx, int64_t f0, int64_t nf, int64_t k, int64_t hop,
                                                     int64_t wstride, cudaStream_t st) {
    const dim3 gseg(stream_generic_cols(p, p->nfft, 256), (unsigned)p->batch);
    DSP_TRY(seg_window_launch<T>(p, gseg, hist, h, ldh, x, nx, f0, nf, k, hop, wstride, p->segbuf.p, st));
    return fft_exec(p->fft, p->cplx, p->f64, CUFFT_FORWARD, p->segbuf.p, p->specbuf.p, st);
}

// STFT call, cuFFT sizes: the nchan x k (channel, segment) pairs fill the plan's batch in order, three launches per batch
template <typename T> static int stft_generic(SpecPlanImpl* p, const StftStreamArgs& sa, const void* x, int64_t nx,
                                               int64_t nchan, int64_t k, double r, int psd_only, void* out, cudaStream_t st) {
    const int64_t pairs = nchan * k;
    const int threads = 256;
    for (int64_t f0 = 0; f0 < pairs; f0 += p->batch) {
        const int64_t nf = pairs - f0 < p->batch ? pairs - f0 : p->batch;
        DSP_TRY(stream_generic_fft<T>(p, sa.hist, sa.h, sa.ldh, x, nx, f0, nf, k, p->hop, 0, st));
        const dim3 gout(stream_generic_cols(p, p->nout, threads), (unsigned)nf);
        stft_store_kernel<T><<<gout, threads, 0, st>>>(reinterpret_cast<const cx<T>*>(p->specbuf.p), p->nbins_fft, p->nfft,
                                                       p->nout, f0, k, sa.ldo, psd_only, p->onesided, (T)(1.0 / r), (T)(2.0 / r),
                                                       out);
        DSP_LAUNCH_OK();
    }
    return DSPB200_OK;
}

// ---------------------------------------------------------------------------------------------- streaming calls
// The seam of a streaming call, fused sizes: the nsu units per channel that start in the history (a unit is one complex
// segment or two consecutive real ones) read v[0, ls) of the virtual column, which stft_stream_edge_kernel copies to
// p->seam with column stride lds (16-byte aligned columns, for TMA)
struct StreamSeam { int64_t nsu = 0, ls = 0, lds = 0; };
static StreamSeam stream_seam(const SpecPlanImpl* p, int64_t nhist, int64_t nx, int64_t nseg) {
    StreamSeam sm;
    if (p->fused && nseg > 0 && nhist > 0) {
        const int64_t us = p->cplx ? p->hop : 2 * p->hop, upc = p->cplx ? nseg : (nseg + 1) / 2;
        sm.nsu = cdiv(nhist, us) < upc ? cdiv(nhist, us) : upc;
        const int64_t end = (sm.nsu - 1) * us + (p->cplx ? p->n : p->hop + p->n);
        sm.ls = end < nhist + nx ? end : nhist + nx;
    }
    const int64_t esz = (int64_t)dtype_size(p->dtype);
    sm.lds = cdiv(sm.ls * esz, 16) * 16 / esz;
    return sm;
}

// Launch 1 of a streaming call: the seam copy and the new history v[skip, skip + newh) of every channel
static int stream_edge(SpecPlanImpl* p, const StreamSeam& sm, const void* hist_in, int64_t nhist, int64_t ldh, const void* x,
                       int64_t nx, int64_t nchan, int64_t skip, int64_t newh, void* hist_out, cudaStream_t st) {
    const size_t esz = dtype_size(p->dtype);
    if (sm.ls > 0) DSP_TRY(p->seam.reserve((size_t)(sm.lds * nchan) * esz));
    if (sm.ls + newh == 0) return DSPB200_OK;
    const int64_t total = nchan * (sm.ls + newh);
    const int threads = 256;
    const unsigned grid = (unsigned)(cdiv(total, threads) < (int64_t)p->sm_count * 8 ? cdiv(total, threads) : (int64_t)p->sm_count * 8);
#define DSP_EDGE(E) stft_stream_edge_kernel<E><<<grid, threads, 0, st>>>((const E*)hist_in, nhist, ldh, (const E*)x, nx, nchan, \
                                                                         (E*)p->seam.p, sm.ls, sm.lds, skip, newh, (E*)hist_out)
    switch (esz) {
        case 4: DSP_EDGE(float); break;
        case 8: DSP_EDGE(double); break;
        default: DSP_EDGE(cx<double>); break;
    }
#undef DSP_EDGE
    DSP_LAUNCH_OK();
    return DSPB200_OK;
}

// Streaming Welch, fused sizes: segments 0 .. nseg - 1 of every channel's virtual column [history (h); x] into acc, per channel
// group one batched transform launch over the seam units (in p->seam, column stride lds), one over the rest of x (column
// stride nx) and welch_stream_reduce_kernel.  With no seam units the transform launch is launch_welch_batch's on x: the
// same base, stride, alignment class, slices and instance.  The groups follow launch_welch_batch's scratch rule, with the
// rows of both transform launches of a group in the scratch.
template <typename T, int N, bool CPLX>
static int welch_stream_fused(SpecPlanImpl* p, const StreamSeam& sm, const void* x, int64_t nx, int64_t h, int64_t nchan,
                              int64_t nseg, double* acc, int add, cudaStream_t st) {
    using In = typename in_type<T, CPLX>::type;
    const int64_t spu = CPLX ? 1 : 2;
    const int64_t seg_s = sm.nsu * spu < nseg ? sm.nsu * spu : nseg;           // segments of the seam units
    const int64_t seg_i = nseg - seg_s;
    const In* xi = reinterpret_cast<const In*>(x) + (seg_i ? seg_s * p->hop - h : 0);
    const bool al_s = welch_batch_aligned(p, p->seam.p, sm.lds, nchan, sizeof(In));
    const bool al_i = welch_batch_aligned(p, xi, nx, nchan, sizeof(In));
    SpecPlanImpl::WelchCfg& cs = p->welch_batch_cfg[al_s ? 1 : 0];
    SpecPlanImpl::WelchCfg& ci = p->welch_batch_cfg[al_i ? 1 : 0];
    if (seg_s) DSP_TRY((welch_select<T, N, CPLX, true>(p, cs, al_s, 0)));
    if (seg_i) DSP_TRY((welch_select<T, N, CPLX, true>(p, ci, al_i, 0)));
    const int64_t rows_cap = (int64_t)(WELCH_BATCH_SCRATCH / ((size_t)N * sizeof(T)));
    const int64_t gcap = seg_s && seg_i ? rows_cap / 2 : rows_cap;
    const int64_t gc_max = nchan < gcap ? nchan : gcap;
    for (int64_t c0 = 0; c0 < nchan; c0 += gc_max) {
        const int64_t gc = nchan - c0 < gc_max ? nchan - c0 : gc_max;
        const int64_t budget = rows_cap / gc;                                   // rows per channel
        WelchBatchWork ws, wi;
        if (seg_s) ws = welch_batch_work(p, cs, CPLX, gc, seg_s, seg_i ? budget / 2 : budget);
        if (seg_i) wi = welch_batch_work(p, ci, CPLX, gc, seg_i, budget - ws.slices);
        DSP_TRY(p->bpartial.reserve((size_t)(ws.nitems + wi.nitems) * N * sizeof(T)));
        T* rows_s = reinterpret_cast<T*>(p->bpartial.p);
        T* rows_i = rows_s + ws.nitems * N;
        if (seg_s)
            DSP_TRY((welch_batch_launch<T, CPLX>(p, cs, ws, reinterpret_cast<const In*>(p->seam.p) + c0 * sm.lds, sm.lds, rows_s, st)));
        if (seg_i) DSP_TRY((welch_batch_launch<T, CPLX>(p, ci, wi, xi + c0 * nx, nx, rows_i, st)));
        const int64_t nw = ws.slices > wi.slices ? ws.slices : wi.slices;
        welch_stream_reduce_kernel<T, N><<<dim3((unsigned)cdiv(p->nout, 32), (unsigned)gc), 32 * (unsigned)(nw < 32 ? nw : 32), 0, st>>>(
            rows_s, (int)ws.slices, rows_i, (int)wi.slices, acc + c0 * p->nout, (int)p->nout, CPLX ? 0 : 1, add);
        DSP_LAUNCH_OK();
    }
    return DSPB200_OK;
}

// Welch, cuFFT sizes: the nchan x k (channel, segment) pairs of the virtual columns through the plan's batch, three launches
// per batch.  Streaming calls, and every other Welch form as one channel with no history.
template <typename T> static int welch_stream_generic(SpecPlanImpl* p, const void* hist, int64_t h, int64_t ldh, const void* x,
                                                       int64_t nx, int64_t nchan, int64_t k, double* acc, int add,
                                                       cudaStream_t st) {
    const int64_t pairs = nchan * k;
    const int threads = 128;
    for (int64_t f0 = 0; f0 < pairs; f0 += p->batch) {
        const int64_t nf = pairs - f0 < p->batch ? pairs - f0 : p->batch;
        DSP_TRY(stream_generic_fft<T>(p, hist, h, ldh, x, nx, f0, nf, k, p->hop, 0, st));
        const int64_t nc = (f0 + nf - 1) / k - f0 / k + 1;                  // channels with a pair in this batch
        welch_stream_acc_kernel<T><<<dim3((unsigned)cdiv(p->nout, threads), (unsigned)nc), threads, 0, st>>>(
            reinterpret_cast<const cx<T>*>(p->specbuf.p), p->nbins_fft, p->nfft, p->nout, f0, nf, k, add, acc);
        DSP_LAUNCH_OK();
    }
    return DSPB200_OK;
}

static int welch_generic(SpecPlanImpl* p, const void* hist, int64_t h, int64_t ldh, const void* x, int64_t nx, int64_t nchan,
                         int64_t k, double* acc, int add, cudaStream_t st) {
    DSP_TRY(generic_prepare(p));
    return p->f64 ? welch_stream_generic<double>(p, hist, h, ldh, x, nx, nchan, k, acc, add, st)
                  : welch_stream_generic<float>(p, hist, h, ldh, x, nx, nchan, k, acc, add, st);
}

// The PSD of the nout x nchan Float64 accumulator acc (welch_stream_power_kernel, up to 65535 channels per launch)
static int welch_power(const SpecPlanImpl* p, const double* acc, int64_t nchan, double r, void* out, cudaStream_t st) {
    const int threads = 128;
    const int half = p->fused && !p->cplx;
    for (int64_t c0 = 0; c0 < nchan; c0 += 65535) {
        const int64_t gc = nchan - c0 < 65535 ? nchan - c0 : 65535;
        const dim3 grid((unsigned)cdiv(p->nout, threads), (unsigned)gc);
        if (p->f64)
            welch_stream_power_kernel<double><<<grid, threads, 0, st>>>(acc + c0 * p->nout, p->nout, p->nfft, p->onesided, half,
                                                                       1.0 / r, 2.0 / r, (double*)out + c0 * p->nout);
        else
            welch_stream_power_kernel<float><<<grid, threads, 0, st>>>(acc + c0 * p->nout, p->nout, p->nfft, p->onesided, half,
                                                                      1.0 / r, 2.0 / r, (float*)out + c0 * p->nout);
        DSP_LAUNCH_OK();
    }
    return DSPB200_OK;
}

// Batched Welch, cuFFT sizes: channel after channel, each written (add = 0) into the batch's own accumulator -- an
// accumulation open on the plan (acc) is left as it was -- and scaled into its column.  The channels are not packed into
// shared cuFFT batches (as a stream packs them): a channel's batch boundaries would then depend on the channels before it,
// and its sum would round differently from the vector call's.
static int welch_batch_generic(SpecPlanImpl* p, const void* s, int64_t len, int64_t nchan, int64_t k, double r, void* out,
                               cudaStream_t st) {
    DSP_TRY(p->bacc.reserve((size_t)p->nout * sizeof(double)));
    double* acc = reinterpret_cast<double*>(p->bacc.p);
    const size_t esz = dtype_size(p->dtype), osz = p->f64 ? 8 : 4;
    for (int64_t c = 0; c < nchan; ++c) {
        DSP_TRY(welch_generic(p, nullptr, 0, 0, (const char*)s + (size_t)(c * len) * esz, len, 1, k, acc, 0, st));
        DSP_TRY(welch_power(p, acc, 1, r, (char*)out + (size_t)(c * p->nout) * osz, st));
    }
    return DSPB200_OK;
}

// ---------------------------------------------------------------------------------------------- plan-level ops
static int welch_begin(SpecPlanImpl* p, cudaStream_t st) {
    if (p->fused) {
        p->rows_used = 0;            // the first launch writes its rows, later ones add (welch_fused_kernel, `fresh_from`)
    } else {
        DSP_TRY(generic_prepare(p));
        DSP_CUDA(cudaMemsetAsync(p->acc.p, 0, (size_t)p->nout * sizeof(double), st));
    }
    return DSPB200_OK;
}

static int welch_accumulate(SpecPlanImpl* p, const void* s, int64_t sample_offset, int64_t seg_begin, int64_t seg_end,
                            cudaStream_t st) {
    if (seg_end <= seg_begin) return DSPB200_OK;
    if (p->fused) {
        return fused_dispatch(p, "Welch", [&](auto t, auto nn) {
            using T = decltype(t);
            constexpr int N = decltype(nn)::value;
            return p->cplx ? launch_welch_fused<T, N, true>(p, s, seg_begin, seg_end - seg_begin, sample_offset, st)
                           : launch_welch_fused<T, N, false>(p, s, seg_begin, seg_end - seg_begin, sample_offset, st);
        });
    }
    // one channel, no history, its first segment at x[0] (welch_range_check: seg_begin hop >= sample_offset), added to acc;
    // the channel's column stride is never read
    const int64_t first = seg_begin * p->hop - sample_offset;
    return welch_generic(p, nullptr, 0, 0, (const char*)s + (size_t)first * dtype_size(p->dtype), 0, 1, seg_end - seg_begin,
                         reinterpret_cast<double*>(p->acc.p), 1, st);
}

static int welch_finalize(SpecPlanImpl* p, double r, void* out, cudaStream_t st) {
    if (p->fused)
        return fused_dispatch(p, "Welch", [&](auto t, auto nn) { return launch_welch_finalize<decltype(t), decltype(nn)::value>(p, r, out, st); });
    return welch_power(p, reinterpret_cast<const double*>(p->acc.p), 1, r, out, st);
}

static int64_t nsegments(const SpecPlanImpl* p, int64_t len) {
    return len >= p->n ? (len - p->n) / p->hop + 1 : 0;   // src/periodograms.jl:49-50
}

static int ensure_streams(SpecPlanImpl* p) { return p->pipe.ensure(p->device); }

}  // namespace dspb200

using namespace dspb200;

struct dspb200_spec_plan {
    SpecPlanImpl impl;
};

static size_t win_row_bytes(const SpecPlanImpl* p) { return (size_t)p->n * sizeof(double); }   // float2 pairs are 8 B too

// Runs f(t) for the tapers t = 0 .. ntapers - 1 of a multitaper plan, with the plan's window set to taper t's row, until one
// fails; the window is restored on every exit.
template <class F> static int for_each_taper(SpecPlanImpl* p, F&& f) {
    void* const base = p->d_window;
    int rc = DSPB200_OK;
    for (int64_t t = 0; t < p->ntapers && rc == DSPB200_OK; ++t) {
        p->d_window = (char*)base + (size_t)t * win_row_bytes(p);
        rc = f(t);
    }
    p->d_window = base;
    return rc;
}

static bool smooth7(int64_t v) {
    for (int64_t q : {2, 3, 5, 7})
        while (v % q == 0) v /= q;
    return v == 1;
}

// Epochs per group of a multitaper cross-spectra call: the raw spectra of all tapers of a group's epochs (nout x nchan x K
// per epoch) stay within MT_CROSS_SCRATCH bytes, and a group holds at least one epoch.
static constexpr size_t MT_CROSS_SCRATCH = (size_t)1 << 30;
static int64_t mt_cross_group(const SpecPlanImpl* p, int64_t nchan, int64_t nepochs) {
    const size_t per_epoch = (size_t)(p->nout * nchan * p->ntapers) * (p->f64 ? 16 : 8);
    const int64_t g = (int64_t)(MT_CROSS_SCRATCH / per_epoch);
    return g < 1 ? 1 : (g < nepochs ? g : nepochs);
}

// mt_cross_power_spectra! / mt_coherence! of the epoch mean, src/multitaper.jl:553-603, 722-790, device pointers; queues the
// work on st (the caller waits for it: the plan's scratch is reused by the next call).  signal is n_channels x n x nepochs.
// Per group of epochs (mt_cross_group): cs_prep_kernel over its (channel, epoch) columns, one raw-spectra STFT call per
// taper over those columns into the taper's slab of p->tmp (per_epoch: one per taper and epoch), and one cs_acc_kernel
// launch, which sums every taper and epoch of the group into the spectra.  The spectra are written to `out`, or, for
// coherence, to pipe.out[0], from which coherence_kernel writes `out`.
template <typename T>
static int mt_cross_run(dspb200_spec_plan* plan, const void* signal, int64_t nchan, int64_t nepochs, int demean, int64_t f_lo,
                        int64_t nf, int coherence, void* out, cudaStream_t st) {
    SpecPlanImpl* p = &plan->impl;
    const int64_t n = p->n, cnt = nchan * nchan * nf, G = mt_cross_group(p, nchan, nepochs);
    const int64_t ctiles = cdiv(nchan, CS_C), ctas = ctiles * ctiles * cdiv(nf, CsTile<T>::F);
    // At odd or non-7-smooth cuFFT sizes a column's transform is not independent of its neighbours in the cuFFT batch (a
    // 3-channel Float32 nfft 1031 call differed from the matrix calls when two epochs shared a batch), so each epoch is
    // transformed by a call of its own, in the batch slots the matrix call gives it.
    const bool per_epoch = !p->fused && (p->nfft % 2 != 0 || !smooth7(p->nfft));
    DSP_REQUIRE(ctas <= INT32_MAX, "too many output tiles (%lld)", (long long)ctas);
    DSP_TRY(p->pipe.in[1].reserve((size_t)(n * nchan * G) * sizeof(T)));
    DSP_TRY(p->tmp.reserve((size_t)(p->nout * nchan * G * p->ntapers) * sizeof(cx<T>)));
    if (coherence) DSP_TRY(p->pipe.out[0].reserve((size_t)cnt * sizeof(cx<T>)));
    cx<T>* const cs = (cx<T>*)(coherence ? p->pipe.out[0].p : out);
    for (int64_t e0 = 0; e0 < nepochs; e0 += G) {
        const int64_t g = nepochs - e0 < G ? nepochs - e0 : G, cols = nchan * g;
        cs_prep_kernel<T><<<(unsigned)cols, 256, 0, st>>>((const T*)signal + e0 * nchan * n, nchan, n, demean, (T*)p->pipe.in[1].p);
        DSP_LAUNCH_OK();
        DSP_TRY(for_each_taper(p, [&](int64_t t) -> int {                  // raw spectra of taper t, nout x cols
            cx<T>* const slab = (cx<T>*)p->tmp.p + t * p->nout * cols;
            if (!per_epoch) return dspb200_stft_exec_dev(plan, p->pipe.in[1].p, n, cols, 1.0, 0, slab, st);
            for (int64_t e = 0; e < g; ++e)
                DSP_TRY(dspb200_stft_exec_dev(plan, (const T*)p->pipe.in[1].p + e * nchan * n, n, nchan, 1.0, 0,
                                              slab + e * nchan * p->nout, st));
            return DSPB200_OK;
        }));
        cs_acc_kernel<T><<<(unsigned)ctas, CS_THREADS, 0, st>>>(cs, (const cx<T>*)p->tmp.p, p->nout, nchan, g, p->ntapers, f_lo, nf,
                                                               (p->nfft % 2 == 0) ? 1 : 0, e0 == 0 ? 1 : 0,
                                                               e0 + g == nepochs ? nepochs : 1);
        DSP_LAUNCH_OK();
    }
    if (coherence) {
        const int threads = 256;
        const int grid = (int)(cdiv(cnt, threads) < device_sm_count() * 32 ? cdiv(cnt, threads) : device_sm_count() * 32);
        coherence_kernel<T><<<grid, threads, 0, st>>>((T*)out, cs, nchan, nf);
        DSP_LAUNCH_OK();
    }
    return DSPB200_OK;
}

// mt_pgram of the nchan columns of a len x nchan matrix (len = n), fused sizes: per channel group, one batched Welch launch
// whose work items are the channels and whose units are a channel's tapers (welch_fused_kernel<..., TAPERS = true>: the
// tapers' |X_t|^2 summed in registers in taper order, one partial row per channel -- a channel's tapers are never split, so a
// column's bits do not depend on the other columns), then welch_finalize_kernel.  The groups follow launch_welch_batch's
// scratch rule.
template <typename T, int N, bool CPLX>
static int launch_mt_pgram(SpecPlanImpl* p, const void* s, int64_t len, int64_t nchan, void* out, cudaStream_t st) {
    using In = typename in_type<T, CPLX>::type;
    const bool aligned = welch_batch_aligned(p, s, len, nchan, sizeof(In));
    SpecPlanImpl::WelchCfg& cfg = p->welch_mt_cfg[aligned ? 1 : 0];
    DSP_TRY((welch_select<T, N, CPLX, true, true>(p, cfg, aligned, 0)));
    const int64_t rows_cap = (int64_t)(WELCH_BATCH_SCRATCH / ((size_t)N * sizeof(T)));
    const int64_t gc_max = nchan < rows_cap ? nchan : rows_cap;
    for (int64_t c0 = 0; c0 < nchan; c0 += gc_max) {
        WelchBatchWork w;                                // one item per channel: its ntapers units, one segment
        w.k = 1;
        w.upc = w.per = p->ntapers;
        w.slices = 1;
        w.nitems = nchan - c0 < gc_max ? nchan - c0 : gc_max;
        DSP_TRY(p->bpartial.reserve((size_t)w.nitems * N * sizeof(T)));
        DSP_TRY((welch_batch_launch<T, CPLX>(p, cfg, w, (const In*)s + c0 * len, len, p->bpartial.p, st)));
        welch_finalize_kernel<T, N><<<dim3((unsigned)cdiv(p->nout, 32), (unsigned)w.nitems), 32, 0, st>>>(
            reinterpret_cast<const T*>(p->bpartial.p), 1, reinterpret_cast<T*>(out) + c0 * p->nout, (int)p->nout, CPLX ? 0 : 1,
            (int)p->onesided, 1.0, 2.0);
        DSP_LAUNCH_OK();
    }
    return DSPB200_OK;
}

// mt_pgram, cuFFT sizes: the nchan x ntapers (channel, taper) pairs through the plan's batch -- seg_window_kernel (pair
// (c, t): channel c's n samples under taper row t), cuFFT, mt_pow_acc_kernel: three launches per batch -- into a Float64
// nout x nchan accumulator, then the fft2pow! scaling (r = 1) of welch_power.
template <typename T> static int mt_pgram_generic(SpecPlanImpl* p, const void* s, int64_t len, int64_t nchan, void* out,
                                                   cudaStream_t st) {
    DSP_TRY(generic_prepare(p));
    DSP_TRY(p->bacc.reserve((size_t)(p->nout * nchan) * sizeof(double)));
    double* acc = reinterpret_cast<double*>(p->bacc.p);
    const int64_t nt = p->ntapers, pairs = nchan * nt;
    for (int64_t f0 = 0; f0 < pairs; f0 += p->batch) {
        const int64_t nf = pairs - f0 < p->batch ? pairs - f0 : p->batch;
        DSP_TRY(stream_generic_fft<T>(p, nullptr, 0, 0, s, len, f0, nf, nt, 0, p->n, st));
        const int64_t nc = (f0 + nf - 1) / nt - f0 / nt + 1;                 // channels with a pair in this batch
        mt_pow_acc_kernel<T><<<dim3((unsigned)cdiv(p->nout, 128), (unsigned)nc), 128, 0, st>>>(
            reinterpret_cast<const cx<T>*>(p->specbuf.p), p->nbins_fft, p->nfft, p->nout, f0, nf, nt, acc);
        DSP_LAUNCH_OK();
    }
    return welch_power(p, acc, nchan, 1.0, out, st);
}

// periodogram(s::AbstractMatrix; nfft, fs, radialsum, radialavg), src/periodograms.jl:473-509, device pointers: queues the
// work on st (cached plan + scratch arena: the caller goes through convenience_call)
template <typename T>
static int periodogram2_run(const void* s, int64_t n1, int64_t n2, int64_t f1, int64_t f2, double r, int ptype, void* out,
                            cudaStream_t st) {
    const int64_t h = f1 / 2 + 1, nmin = f1 < f2 ? f1 : f2, kmax = nmin / 2 + 1;
    const int threads = 256;
    auto grid = [&](int64_t total) { const int64_t g = cdiv(total, threads); const int64_t cap = (int64_t)device_sm_count() * 32; return (int)(g < cap ? g : cap); };
    DevBuf &dpad = scratch_buf(1), &dX = scratch_buf(2), &dacc = scratch_buf(4);
    DSP_TRY(dpad.reserve((size_t)(f1 * f2) * sizeof(T)));
    DSP_TRY(dX.reserve((size_t)(h * f2) * sizeof(cx<T>)));
    per2_pad_kernel<T><<<grid(f1 * f2), threads, 0, st>>>((const T*)s, n1, n2, (T*)dpad.p, f1, f2);
    DSP_LAUNCH_OK();
    const bool f64 = sizeof(T) == 8;
    long long nn[2] = {(long long)f2, (long long)f1};            // cuFFT is row-major: slowest dimension first
    int hp = 0;
    DSP_TRY(plan_cache_get(&hp, 2, nn, false, 0, 0, fft_type(false, f64, CUFFT_FORWARD), 1));
    DSP_TRY(fft_exec((cufftHandle)hp, false, f64, CUFFT_FORWARD, dpad.p, dX.p, st));
    if (ptype == 0) {
        per2_full_kernel<T><<<grid(f1 * f2), threads, 0, st>>>((const cx<T>*)dX.p, f1, f2, (T)(1.0 / r), (T*)out);
        DSP_LAUNCH_OK();
        return DSPB200_OK;
    }
    DSP_TRY(dacc.reserve((size_t)kmax * 16));
    DSP_CUDA(cudaMemsetAsync(dacc.p, 0, (size_t)kmax * 16, st));
    double* acc = (double*)dacc.p;
    unsigned long long* wc = (unsigned long long*)(acc + kmax);
    double c1 = 1.0, c2 = 1.0;                                   // wavevector scaling for non-square transforms, :193-199
    if (f1 == nmin) c2 = (double)f1 / (double)f2; else c1 = (double)f2 / (double)f1;
    const T m1 = (T)(1.0 / r), m2 = (T)(2.0 / r);                // rounded to the signal precision as in the reference
    per2_radial_kernel<T><<<grid(h * f2), threads, 0, st>>>((const cx<T>*)dX.p, f1, f2, c1, c2, (double)m1, (double)m2, kmax, acc, wc);
    DSP_LAUNCH_OK();
    per2_radial_finish_kernel<T><<<(unsigned)cdiv(kmax, threads), threads, 0, st>>>(acc, wc, kmax, ptype == 2, (T*)out);
    DSP_LAUNCH_OK();
    return DSPB200_OK;
}

extern "C" {

static int spec_plan_create_impl(dspb200_spec_plan** plan, int dtype, int64_t n, int64_t noverlap, int64_t nfft,
                                 int onesided, const double* window_host, int64_t nrows) {
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    *plan = nullptr;
    DSP_REQUIRE(dtype_valid(dtype), "invalid dtype %d", dtype);
    DSP_REQUIRE(n >= 1, "n must be >= 1 (got %lld)", (long long)n);
    DSP_REQUIRE(noverlap >= 0 && noverlap < n, "noverlap must be between zero and n");   // DomainError :44
    DSP_REQUIRE(nfft >= n, "nfft must be >= n");                                           // DomainError :45
    DSP_REQUIRE(!(onesided && dtype_is_cplx(dtype)), "cannot compute one-sided FFT of a complex signal");  // :564
    DSP_REQUIRE(nfft < (int64_t(1) << 31), "nfft too large");
    dspb200_spec_plan* h = new (std::nothrow) dspb200_spec_plan();
    DSP_REQUIRE(h != nullptr, "out of host memory");
    SpecPlanImpl* p = &h->impl;
    p->dtype = dtype; p->cplx = dtype_is_cplx(dtype); p->f64 = dtype_is_f64(dtype);
    p->n = n; p->noverlap = noverlap; p->hop = n - noverlap; p->nfft = nfft; p->onesided = onesided ? 1 : 0;
    p->nout = onesided ? nfft / 2 + 1 : nfft;
    p->nbins_fft = p->cplx ? nfft : nfft / 2 + 1;
    p->fused = fused_size_ok(nfft, p->f64);
    int rc = DSPB200_OK;
    do {
        if (cudaGetDevice(&p->device) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "cudaGetDevice", __FILE__, __LINE__); break; }
        p->sm_count = device_sm_count();
        if (window_host) {
            const int64_t nw = n * (nrows < 1 ? 1 : nrows);
            p->ntapers = nrows;
            if (p->f64) {
                rc = upload(&p->d_window, window_host, (size_t)nw * sizeof(double));
            } else {                                       // hi/lo float pairs (same 8 bytes per value)
                std::vector<float> pairs((size_t)nw * 2);
                for (int64_t j = 0; j < nw; ++j) {
                    const float hi = (float)window_host[j];
                    pairs[2 * j] = hi;
                    pairs[2 * j + 1] = (float)(window_host[j] - (double)hi);
                }
                rc = upload(&p->d_window, pairs.data(), pairs.size() * sizeof(float));
            }
            if (rc != DSPB200_OK) break;
        }
        if (p->fused) {
            const size_t csz = p->f64 ? 16 : 8;
            rc = upload_fft_tables(nfft, p->f64, &p->d_tw, &p->d_t16, &p->d_t256);
            if (rc == DSPB200_OK && !p->f64 && nfft == 1024) {                 // table of the warp-per-unit STFT kernel
                std::vector<cx<float>> t32(w1k::T32_LEN);
                w1k::fill_t32(t32.data());
                rc = upload(&p->d_t32, t32.data(), t32.size() * sizeof(cx<float>));
            }
            if (rc != DSPB200_OK) break;
            int optin = 0;
            const cudaError_t e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, p->device);
            if (e != cudaSuccess) { rc = cuda_fail(e, "cudaDeviceGetAttribute", __FILE__, __LINE__); break; }
            p->smem_optin = (size_t)optin;
            // persistent Welch grid: CTAs per SM bounded by shared memory (228 KB/SM on H100) and 2048 threads
            // (data + tables + TMA staging for 50 % overlap) per CTA
            const size_t smem = (size_t)(p->f64 ? padded_len<double>((int)nfft) : padded_len<float>((int)nfft)) * csz + (size_t)(fft_tw16_len(nfft) + fft_tw256_len(nfft)) * csz +
                                (size_t)(p->hop + p->n) * (csz / 2);
            int per_sm = (int)((220 * 1024) / (smem + 1024));
            if (per_sm < 4) per_sm = 4;            // up to (CTAs per SM) x (thread groups per CTA) virtual CTAs
            if (per_sm > 8) per_sm = 8;
            p->nparts = p->sm_count * per_sm;      // upper bound; launches use the occupancy API
            rc = p->partial.reserve((size_t)p->nparts * nfft * (p->f64 ? 8 : 4));
            if (rc != DSPB200_OK) break;
        }
    } while (0);
    if (rc != DSPB200_OK) { dspb200_spec_plan_destroy(h); return rc; }
    *plan = h;
    return DSPB200_OK;
}

int dspb200_spec_plan_create(dspb200_spec_plan** plan, int dtype, int64_t n, int64_t noverlap, int64_t nfft,
                             int onesided, const double* window_host) {
    DSP_RANGE("dspb200_spec_plan_create");
    return spec_plan_create_impl(plan, dtype, n, noverlap, nfft, onesided, window_host, 0);
}

int dspb200_mt_plan_create(dspb200_spec_plan** plan, int dtype, int64_t n, int64_t noverlap, int64_t nfft, int onesided,
                           const double* tapers_host, int64_t ntapers) {
    DSP_RANGE("dspb200_mt_plan_create");
    DSP_REQUIRE(tapers_host != nullptr && ntapers >= 1, "tapers must be a non-empty ntapers x n matrix");
    return spec_plan_create_impl(plan, dtype, n, noverlap, nfft, onesided, tapers_host, ntapers);
}

int dspb200_spec_plan_info(const dspb200_spec_plan* plan, int64_t* nout, int* fused) {
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    if (nout) *nout = plan->impl.nout;
    if (fused) *fused = plan->impl.fused ? 1 : 0;
    return DSPB200_OK;
}

int dspb200_spec_plan_geometry(const dspb200_spec_plan* plan, int* dtype, int64_t* n, int64_t* hop, int64_t* nout) {
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    if (dtype) *dtype = plan->impl.dtype;
    if (n) *n = plan->impl.n;
    if (hop) *hop = plan->impl.hop;
    if (nout) *nout = plan->impl.nout;
    return DSPB200_OK;
}

int64_t dspb200_spec_nsegments(const dspb200_spec_plan* plan, int64_t len) {
    if (!plan) return -1;
    return nsegments(&plan->impl, len);
}

// The index domain of the segment-range forms (dspb200.h): every sum and product below stays under 2^63 in this order
static int welch_range_check(const SpecPlanImpl* p, int64_t len, int64_t sample_offset, int64_t seg_begin, int64_t seg_end) {
    DSP_REQUIRE(seg_begin >= 0 && seg_end >= seg_begin, "bad segment range");
    DSP_REQUIRE(len >= 0 && index_in_domain(len) && index_in_domain(sample_offset) && index_in_domain(sample_offset + len) &&
                    (seg_end == seg_begin || seg_end - 1 <= (DSPB200_INDEX_LIMIT - p->n) / p->hop),
                "segment range outside the index domain: len %lld, sample_offset %lld, segments [%lld, %lld) (limit 2^61)",
                (long long)len, (long long)sample_offset, (long long)seg_begin, (long long)seg_end);
    if (seg_end == seg_begin) return DSPB200_OK;
    DSP_REQUIRE(seg_begin * p->hop >= sample_offset, "segment range starts before the local buffer");
    DSP_REQUIRE((seg_end - 1) * p->hop + p->n <= sample_offset + len, "segment range runs past the local buffer");
    return DSPB200_OK;
}

int dspb200_welch_exec_range_dev(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t sample_offset,
                                 int64_t seg_begin, int64_t seg_end, double r, void* out, void* stream) {
    DSP_RANGE("dspb200_welch_exec_range_dev");
    DSP_REQUIRE(plan && out, "NULL argument");
    DSP_REQUIRE(r != 0.0, "r must be nonzero");
    SpecPlanImpl* p = &plan->impl;
    cudaStream_t st = (cudaStream_t)stream;
    DSP_TRY(welch_range_check(p, len, sample_offset, seg_begin, seg_end));
    DSP_REQUIRE(seg_end == seg_begin || s != nullptr, "s is NULL");
    DSP_TRY(welch_begin(p, st));
    DSP_TRY(welch_accumulate(p, s, sample_offset, seg_begin, seg_end, st));
    return welch_finalize(p, r, out, st);
}

// Streaming form of welch_pgram_helper! (src/periodograms.jl:746-759): begin (zero the accumulator), accumulate any number
// of segment ranges -- each from a buffer that holds at least its own samples -- then finalize (fft2pow! scaling).  This is
// what dspb200_welch_exec_range_dev does in one call; the split lets a pipeline feed the segments chunk by chunk.
int dspb200_welch_begin_dev(dspb200_spec_plan* plan, void* stream) {
    DSP_RANGE("dspb200_welch_begin_dev");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    return welch_begin(&plan->impl, (cudaStream_t)stream);
}
int dspb200_welch_accumulate_dev(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t sample_offset,
                                 int64_t seg_begin, int64_t seg_end, void* stream) {
    DSP_RANGE("dspb200_welch_accumulate_dev");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    SpecPlanImpl* p = &plan->impl;
    DSP_TRY(welch_range_check(p, len, sample_offset, seg_begin, seg_end));
    if (seg_end == seg_begin) return DSPB200_OK;
    DSP_REQUIRE(s != nullptr, "s is NULL");
    return welch_accumulate(p, s, sample_offset, seg_begin, seg_end, (cudaStream_t)stream);
}
int dspb200_welch_finalize_dev(dspb200_spec_plan* plan, double r, void* out, void* stream) {
    DSP_RANGE("dspb200_welch_finalize_dev");
    DSP_REQUIRE(plan && out, "NULL argument");
    DSP_REQUIRE(r != 0.0, "r must be nonzero");
    return welch_finalize(&plan->impl, r, out, (cudaStream_t)stream);
}

// Testing aid: run one chosen fused Welch instance on a chosen number of virtual CTAs (the kernels have no grid-wide
// synchronisation, so a grid larger than one resident wave is as correct as one wave)
int dspb200_spec_plan_pin_welch(dspb200_spec_plan* plan, int batched, int mode, int groups, int64_t vctas) {
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    SpecPlanImpl* p = &plan->impl;
    SpecPlanImpl::WelchCfg* cfg = batched ? p->welch_batch_cfg : p->welch_cfg;
    // batched, multitaper plan: mt_pgram's taper-row instance of MODE 0 / 1 is pinned too (MODE 2 / 3 have none: it selects)
    const bool mt = batched && p->ntapers >= 1;
    if (mt) p->welch_mt_cfg[0] = p->welch_mt_cfg[1] = SpecPlanImpl::WelchCfg{};
    if (mode < 0) {                                      // unpin: the next call selects as before
        cfg[0] = SpecPlanImpl::WelchCfg{};
        cfg[1] = SpecPlanImpl::WelchCfg{};
        return DSPB200_OK;
    }
    if (!p->fused || groups < 1) {
        set_error("no fused Welch kernel instance MODE %d, G %d for this plan", mode, groups);
        return DSPB200_EUNSUPPORTED;
    }
    DSP_REQUIRE(vctas >= 0 && vctas % groups == 0, "vctas (%lld) must be a non-negative multiple of groups (%d)",
                (long long)vctas, groups);
    DSP_REQUIRE(batched || vctas <= p->nparts, "vctas (%lld) exceeds the plan's %d partial rows", (long long)vctas, p->nparts);
    DSP_CUDA(cudaSetDevice(p->device));
    return fused_dispatch(p, "Welch", [&](auto t, auto nn) {
        using T = decltype(t);
        constexpr int N = decltype(nn)::value;
        if (batched) {
            DSP_TRY((p->cplx ? welch_pin<T, N, true, true>(p, mode, groups, vctas) : welch_pin<T, N, false, true>(p, mode, groups, vctas)));
            if (!mt || mode >= 2) return (int)DSPB200_OK;
            return p->cplx ? welch_pin<T, N, true, true, true>(p, mode, groups, vctas) : welch_pin<T, N, false, true, true>(p, mode, groups, vctas);
        }
        return p->cplx ? welch_pin<T, N, true, false>(p, mode, groups, vctas) : welch_pin<T, N, false, false>(p, mode, groups, vctas);
    });
}

int dspb200_spec_plan_welch_config(const dspb200_spec_plan* plan, int batched, int aligned, int* mode, int* groups,
                                   int64_t* vctas) {
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    const SpecPlanImpl::WelchCfg& c = (batched == 2 ? plan->impl.welch_mt_cfg : batched ? plan->impl.welch_batch_cfg
                                                                                        : plan->impl.welch_cfg)[aligned ? 1 : 0];
    const bool ran = c.kern != nullptr && c.used > 0;
    if (mode) *mode = ran ? c.mode : -1;
    if (groups) *groups = ran ? c.g : 0;
    if (vctas) *vctas = ran ? c.used : 0;
    return DSPB200_OK;
}

int dspb200_welch_exec_dev(dspb200_spec_plan* plan, const void* s, int64_t len, double r, void* out, void* stream) {
    DSP_RANGE("dspb200_welch_exec_dev");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    const int64_t k = nsegments(&plan->impl, len);
    return dspb200_welch_exec_range_dev(plan, s, len, 0, 0, k, r, out, stream);
}

// Batched welch_pgram: the nchan columns of the column-major len x nchan matrix `s` are independent signals, each Welch-averaged
// with the plan's configuration; out is nout x nchan.  Fused sizes: one launch over (channel, slice) work items plus one
// finalize launch per channel group (welch_fused_kernel<..., BATCH = true>); cuFFT sizes: channel by channel.
int dspb200_welch_batch_exec_dev(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t nchan, double r, void* out,
                                 void* stream) {
    DSP_RANGE("dspb200_welch_batch_exec_dev");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    DSP_REQUIRE(nchan >= 0 && len >= 0, "negative size");
    SpecPlanImpl* p = &plan->impl;
    cudaStream_t st = (cudaStream_t)stream;
    if (nchan == 0) return DSPB200_OK;
    DSP_REQUIRE(out != nullptr, "out is NULL");
    const int64_t k = nsegments(p, len);
    if (k == 0) {                                        // fill!(out, 0), src/periodograms.jl:747
        DSP_CUDA(cudaMemsetAsync(out, 0, (size_t)(p->nout * nchan) * (p->f64 ? 8 : 4), st));
        return DSPB200_OK;
    }
    DSP_REQUIRE(s != nullptr, "s is NULL");
    DSP_REQUIRE(r != 0.0, "r must be nonzero");
    if (p->fused)
        return fused_dispatch(p, "Welch", [&](auto t, auto nn) {
            using T = decltype(t);
            constexpr int N = decltype(nn)::value;
            return p->cplx ? launch_welch_batch<T, N, true>(p, s, len, nchan, k, r, out, st)
                           : launch_welch_batch<T, N, false>(p, s, len, nchan, k, r, out, st);
        });
    return welch_batch_generic(p, s, len, nchan, k, r, out, st);
}

int dspb200_welch_batch_exec(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t nchan, double r, void* out) {
    DSP_RANGE("dspb200_welch_batch_exec");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    DSP_REQUIRE(nchan >= 0 && len >= 0, "negative size");
    SpecPlanImpl* p = &plan->impl;
    if (nchan == 0) return DSPB200_OK;
    DSP_REQUIRE(out != nullptr, "out is NULL");
    const bool any = nsegments(p, len) > 0;                // otherwise out is zeroed and s is not read
    DSP_REQUIRE(!any || s != nullptr, "s is NULL");
    DSP_TRY(ensure_streams(p));
    const size_t in_bytes = any ? (size_t)(len * nchan) * dtype_size(p->dtype) : 0;
    return run_staged(p->pipe.s_exec, {{s, in_bytes, &p->pipe.in[0]}}, {{out, (size_t)(p->nout * nchan) * (p->f64 ? 8 : 4), &p->pipe.out[0]}},
                      [&] { return dspb200_welch_batch_exec_dev(plan, p->pipe.in[0].p, len, nchan, r, p->pipe.out[0].p, p->pipe.s_exec); });
}

// The tail of the chunked host-pointer Welch calls: the PSD into out[0] (reserved before the first chunk), then to the host.
static int welch_finalize_host(SpecPlanImpl* p, double r, void* out) {
    HostPipe& hp = p->pipe;
    DSP_TRY(welch_finalize(p, r, hp.out[0].p, hp.s_exec));
    DSP_CUDA(cudaMemcpyAsync(out, hp.out[0].p, (size_t)p->nout * (p->f64 ? 8 : 4), cudaMemcpyDeviceToHost, hp.s_exec));
    return DSPB200_OK;
}

// Host-pointer Welch: the signal is streamed through the plan's two slots in segment-aligned chunks (run_chunked), so the
// H2D copy of chunk c+1 overlaps the kernel of chunk c (effective when `s` is pinned).
int dspb200_welch_exec(dspb200_spec_plan* plan, const void* s, int64_t len, double r, void* out) {
    DSP_RANGE("dspb200_welch_exec");
    DSP_REQUIRE(plan && out, "NULL argument");
    DSP_REQUIRE(r != 0.0, "r must be nonzero");
    SpecPlanImpl* p = &plan->impl;
    HostPipe& hp = p->pipe;
    const int64_t k = nsegments(p, len);
    DSP_REQUIRE(k == 0 || s != nullptr, "s is NULL");
    DSP_TRY(ensure_streams(p));
    const size_t esz = dtype_size(p->dtype);
    int64_t chunk_segs = ((int64_t(32) << 20) / (int64_t)esz) / p->hop;   // ~32 MiB of new samples per chunk
    if (chunk_segs < 64) chunk_segs = 64;
    if (chunk_segs > k) chunk_segs = k;
    DSP_TRY(hp.out[0].reserve((size_t)p->nout * (p->f64 ? 8 : 4)));
    DSP_TRY(welch_begin(p, hp.s_exec));
    auto chunk = [&](int64_t c) -> Chunk {
        const int64_t b0 = c * chunk_segs, b1 = b0 + chunk_segs < k ? b0 + chunk_segs : k;
        const int64_t first = b0 * p->hop, cnt = (b1 - 1 - b0) * p->hop + p->n;
        auto accumulate = [=, &hp](const void* in, void*) { return welch_accumulate(p, in, first, b0, b1, hp.s_exec); };
        return {(const char*)s + (size_t)first * esz, (size_t)cnt * esz, accumulate};
    };
    return run_chunked(hp, k > 0 ? cdiv(k, chunk_segs) : 0, (size_t)((chunk_segs - 1) * p->hop + p->n) * esz, 0, chunk,
                       [&] { return welch_finalize_host(p, r, out); });
}

// welch_pgram(filt(b, x), config) (src/dspbase.jl:14-15, src/periodograms.jl:702-759) for a stream that lives in host
// memory.  The filter output y never crosses PCIe: chunk c's samples (plus the nv - 1 sample halo) are copied into a slot
// while the execute stream runs, for chunk c - 1, the overlap-save convolution of its output range into y
// (dspb200_os_exec_range_dev) and then the Welch accumulation of the segments that range completes.  The slot is free
// once the convolution has read it, so the next copy in does not wait for the Welch kernel.
int dspb200_filt_welch_exec(dspb200_os_plan* os, dspb200_spec_plan* spec, const void* x_host, int64_t n, double r,
                            void* out_host) {
    DSP_RANGE("dspb200_filt_welch_exec");
    DSP_REQUIRE(os && spec && out_host, "NULL argument");
    DSP_REQUIRE(n >= 0, "n must be >= 0");
    DSP_REQUIRE(r != 0.0, "r must be nonzero");
    SpecPlanImpl* p = &spec->impl;
    HostPipe& hp = p->pipe;
    int64_t nv = 0, nfft = 0;
    int dt_os = 0;
    DSP_TRY(dspb200_os_plan_geometry(os, &dt_os, &nv, &nfft));
    DSP_REQUIRE(dt_os == p->dtype, "filter plan dtype (%d) and Welch plan dtype (%d) differ", dt_os, p->dtype);
    const int64_t k = nsegments(p, n);
    DSP_REQUIRE(k == 0 || x_host != nullptr, "x is NULL");
    DSP_TRY(ensure_streams(p));
    const size_t esz = dtype_size(p->dtype);
    const int64_t halo = nv - 1, L = nfft - nv + 1;
    int64_t chunk = ((int64_t(32) << 20) / (int64_t)esz) / L * L;         // whole overlap-save blocks, ~32 MiB of new samples
    if (chunk < L) chunk = L;
    if (chunk > n) chunk = n;
    DSP_TRY(hp.out[0].reserve((size_t)p->nout * (p->f64 ? 8 : 4)));
    if (k > 0) DSP_TRY(p->y.reserve((size_t)n * esz));
    DSP_TRY(welch_begin(p, hp.s_exec));
    auto chunk_at = [&](int64_t c) -> Chunk {
        const int64_t c0 = c * chunk, c1 = c0 + chunk < n ? c0 + chunk : n, in0 = c0 - halo > 0 ? c0 - halo : 0;
        char* y = (char*)p->y.p;
        auto filter = [=, &hp](const void* in, void*) {    // y[c0, c1) = (b * x)[c0, c1); the slot holds x[in0, c1)
            return dspb200_os_exec_range_dev(os, in, in0, c1 - in0, y + (size_t)c0 * esz, c0, c1 - c0, hp.s_exec);
        };
        auto accumulate = [=, &hp] {                       // the segments that end in [c0, c1)
            return welch_accumulate(p, y, 0, nsegments(p, c0), nsegments(p, c1), hp.s_exec);
        };
        return {(const char*)x_host + (size_t)in0 * esz, (size_t)(c1 - in0) * esz, filter, accumulate};
    };
    return run_chunked(hp, k > 0 ? cdiv(n, chunk) : 0, (size_t)(chunk + halo) * esz, 0, chunk_at,
                       [&] { return welch_finalize_host(p, r, out_host); });
}

// arraysplit / ArraySplit (src/periodograms.jl:32-73, 134-137): all k windowed, zero-padded segments as a k x nfft
// matrix (row = segment; the reference yields them one at a time into a reused buffer).
int dspb200_arraysplit_exec(dspb200_spec_plan* plan, const void* s, int64_t len, void* out) {
    DSP_RANGE("dspb200_arraysplit_exec");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    SpecPlanImpl* p = &plan->impl;
    const int64_t k = nsegments(p, len);
    if (k == 0) return DSPB200_OK;
    DSP_REQUIRE(s && out, "NULL argument");
    DSP_TRY(ensure_streams(p));
    const size_t esz = dtype_size(p->dtype);
    return run_staged(p->pipe.s_exec, {{s, (size_t)len * esz, &p->pipe.in[0]}}, {{out, (size_t)(k * p->nfft) * esz, &p->pipe.out[0]}}, [&]() -> int {
        // one channel, no history; segment f in row f - f0 of a launch of at most 65535 grid rows
        for (int64_t f0 = 0; f0 < k; f0 += 65535) {
            const int64_t nf = k - f0 < 65535 ? k - f0 : 65535;
            const dim3 grid((unsigned)cdiv(p->nfft, 256), (unsigned)nf);
            void* buf = (char*)p->pipe.out[0].p + (size_t)(f0 * p->nfft) * esz;
            DSP_TRY(p->f64 ? seg_window_launch<double>(p, grid, nullptr, 0, 0, p->pipe.in[0].p, len, f0, nf, k, p->hop, 0, buf, p->pipe.s_exec)
                           : seg_window_launch<float>(p, grid, nullptr, 0, 0, p->pipe.in[0].p, len, f0, nf, k, p->hop, 0, buf, p->pipe.s_exec));
        }
        return DSPB200_OK;
    });
}

// Segments 0 .. k - 1 of every channel's virtual column [history (sa); x (the nx x nchan chunk)], one-shot or streaming
static int stft_launch(SpecPlanImpl* p, const StftStreamArgs& sa, const void* x, int64_t nx, int64_t nchan, int64_t k, double r,
                       int psd_only, void* out, cudaStream_t st) {
    if (p->fused)
        return fused_dispatch(p, "STFT", [&](auto t, auto nn) {
            using T = decltype(t);
            constexpr int N = decltype(nn)::value;
            return p->cplx ? launch_stft_fused<T, N, true>(p, x, nx, nchan, k, r, psd_only, out, st, sa)
                           : launch_stft_fused<T, N, false>(p, x, nx, nchan, k, r, psd_only, out, st, sa);
        });
    DSP_TRY(generic_prepare(p));
    return p->f64 ? stft_generic<double>(p, sa, x, nx, nchan, k, r, psd_only, out, st)
                  : stft_generic<float>(p, sa, x, nx, nchan, k, r, psd_only, out, st);
}

int dspb200_stft_exec_dev(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t nchan, double r, int psd_only,
                          void* out, void* stream) {
    DSP_RANGE("dspb200_stft_exec_dev");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    DSP_REQUIRE(r != 0.0 || !psd_only, "r must be nonzero");
    DSP_REQUIRE(nchan >= 0 && len >= 0, "negative size");
    SpecPlanImpl* p = &plan->impl;
    const int64_t k = nsegments(p, len);
    if (k == 0 || nchan == 0) return DSPB200_OK;
    DSP_REQUIRE(s && out, "NULL argument");
    if (r == 0.0) r = 1.0;
    StftStreamArgs sa;                                   // no history; columns k apart
    sa.ldo = k;
    return stft_launch(p, sa, s, len, nchan, k, r, psd_only, out, (cudaStream_t)stream);
}

int dspb200_stft_exec(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t nchan, double r, int psd_only,
                      void* out) {
    DSP_RANGE("dspb200_stft_exec");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    SpecPlanImpl* p = &plan->impl;
    const int64_t k = nsegments(p, len);
    if (k == 0 || nchan == 0) return DSPB200_OK;
    DSP_REQUIRE(s && out, "NULL argument");
    DSP_TRY(ensure_streams(p));
    const size_t oel = psd_only ? (p->f64 ? 8 : 4) : (p->f64 ? 16 : 8);
    return run_staged(p->pipe.s_exec, {{s, (size_t)len * nchan * dtype_size(p->dtype), &p->pipe.in[0]}}, {{out, (size_t)p->nout * k * nchan * oel, &p->pipe.out[0]}},
                      [&] { return dspb200_stft_exec_dev(plan, p->pipe.in[0].p, len, nchan, r, psd_only, p->pipe.out[0].p, p->pipe.s_exec); });
}

// Streaming calls (STFT and Welch).  Checks shared by every form: sizes, the history, the segments and, device form, the
// overlaps of the written buffers (hist_out, and `out` of obytes bytes, named `oname`) with the others.  *newh = samples of
// the new history.  Returns with *launch = false when the call has nothing to do (no channel, or no sample and no segment:
// the history stays in hist_in).
static int stream_check(const SpecPlanImpl* p, const void* hist_in, int64_t nhist, const void* hist_out, int64_t ldh,
                        const void* x, int64_t nx, int64_t nchan, int64_t nseg, const void* out, size_t obytes, const char* oname,
                        bool dev, int64_t* newh, bool* launch) {
    *launch = false;
    DSP_REQUIRE(hist_in != nullptr || nhist == 0, "hist_in is NULL but nhist = %lld", (long long)nhist);
    DSP_REQUIRE(nhist <= ldh, "nhist (%lld) exceeds ldh (%lld)", (long long)nhist, (long long)ldh);
    DSP_REQUIRE(nseg == 0 || (nseg - 1) * p->hop + p->n <= nhist + nx, "segment %lld runs past the virtual column (%lld samples)",
                (long long)(nseg - 1), (long long)(nhist + nx));
    *newh = nhist + nx - nseg * p->hop;
    DSP_REQUIRE(*newh <= ldh, "the new history (%lld samples) exceeds ldh (%lld)", (long long)*newh, (long long)ldh);
    if (dev) {
        const size_t esz = dtype_size(p->dtype);
        const size_t hbytes = (size_t)(ldh * nchan) * esz, xbytes = (size_t)(nx * nchan) * esz;
        // the kernels read the samples and history of other channels' CTAs: no written buffer may overlap another buffer
        DSP_REQUIRE(!ranges_overlap(hist_out, hbytes, hist_in, hbytes) && !ranges_overlap(hist_out, hbytes, x, xbytes) &&
                    !ranges_overlap(hist_out, hbytes, out, obytes), "hist_out overlaps hist_in, x or %s", oname);
        DSP_REQUIRE(!ranges_overlap(out, obytes, x, xbytes) && !ranges_overlap(out, obytes, hist_in, hbytes),
                    "%s overlaps x or a history buffer", oname);
    }
    if (nchan == 0 || (nx == 0 && nseg == 0)) return DSPB200_OK;
    DSP_REQUIRE((x != nullptr || nx == 0) && (out != nullptr || nseg == 0) && (hist_out != nullptr || *newh == 0), "NULL argument");
    *launch = true;
    return DSPB200_OK;
}

static int stft_stream_check(const SpecPlanImpl* p, const void* hist_in, int64_t nhist, const void* hist_out, int64_t ldh,
                             const void* x, int64_t nx, int64_t nchan, int64_t nseg, double r, int psd_only, const void* out,
                             int64_t ldo, bool dev, int64_t* newh, bool* launch) {
    *launch = false;
    DSP_REQUIRE(nhist >= 0 && nx >= 0 && nchan >= 0 && nseg >= 0 && ldh >= 0, "negative size");
    DSP_REQUIRE(psd_only == 0 || psd_only == 1, "psd_only must be 0 (raw spectra) or 1 (PSD columns)");
    DSP_REQUIRE(r != 0.0 || !psd_only, "r must be nonzero");
    // a multitaper plan's rows carry 1/sqrt(r_t): PSD columns with r = 1 only (raw spectra of a taper sum are not defined)
    DSP_REQUIRE(p->ntapers == 0 || (psd_only == 1 && r == 1.0), "a multitaper plan streams PSD columns (psd_only = 1) with r = 1");
    DSP_REQUIRE(ldo >= nseg, "output column stride ldo < nseg");
    const size_t oel = (psd_only ? 1 : 2) * (p->f64 ? 8 : 4);
    const size_t obytes = (nchan && nseg) ? (size_t)(((nchan - 1) * ldo + nseg) * p->nout) * oel : 0;
    return stream_check(p, hist_in, nhist, hist_out, ldh, x, nx, nchan, nseg, out, obytes, "out", dev, newh, launch);
}

extern "C++" {
// out[c ldc + i] + add[c per + i], rounded once, for i < per and c < nchan: the taper add of a streaming mt_spectrogram, whose
// channels are ldc values apart in `out` (ldo columns) and per apart in the plan's scratch (nseg columns)
template <typename T>
__global__ void acc_add_cols_kernel(T* __restrict__ out, int64_t ldc, const T* __restrict__ add, int64_t per, int64_t nchan) {
    const int64_t total = per * nchan;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t c = i / per;
        T* o = out + c * ldc + (i - c * per);
        *o = add_rn(*o, add[i]);
    }
}

// mt_spectrogram, cuFFT sizes, one-shot (no history in sa) or streaming: taper 0's PSD columns into out, every later taper's
// into the plan's scratch and then added to out, each through the generic stream STFT
template <typename T>
static int mt_stream_generic(SpecPlanImpl* p, const StftStreamArgs& sa, const void* x, int64_t nx, int64_t nchan, int64_t nseg,
                             void* out, cudaStream_t st) {
    DSP_TRY(generic_prepare(p));
    const int64_t per = p->nout * nseg;
    DSP_TRY(p->tmp.reserve((size_t)(per * nchan) * sizeof(T)));
    StftStreamArgs st_tmp = sa;
    st_tmp.ldo = nseg;
    return for_each_taper(p, [&](int64_t t) -> int {
        DSP_TRY(stft_generic<T>(p, t == 0 ? sa : st_tmp, x, nx, nchan, nseg, 1.0, 1, t == 0 ? out : p->tmp.p, st));
        if (t == 0) return DSPB200_OK;
        const int threads = 256;
        const int64_t want = cdiv(per * nchan, threads), cap = (int64_t)p->sm_count * 32;
        acc_add_cols_kernel<T><<<(unsigned)(want < cap ? want : cap), threads, 0, st>>>((T*)out, sa.ldo * p->nout,
                                                                                       (const T*)p->tmp.p, per, nchan);
        DSP_LAUNCH_OK();
        return DSPB200_OK;
    });
}
}  // extern "C++"

// Segments 0 .. nseg - 1 of every channel's virtual column [hist_in (nhist); x (nx)] into out (column s of channel c at
// out + (c ldo + s) nout), then the new history v[nseg hop, nhist + nx) into hist_out.  Fused sizes: at most two launches.
int dspb200_stft_stream_exec_dev(dspb200_spec_plan* plan, const void* hist_in, int64_t nhist, void* hist_out, int64_t ldh,
                                 const void* x, int64_t nx, int64_t nchan, int64_t nseg, double r, int psd_only, void* out,
                                 int64_t ldo, void* stream) {
    DSP_RANGE("dspb200_stft_stream_exec_dev");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    SpecPlanImpl* p = &plan->impl;
    int64_t newh = 0;
    bool launch = false;
    DSP_TRY(stft_stream_check(p, hist_in, nhist, hist_out, ldh, x, nx, nchan, nseg, r, psd_only, out, ldo, true, &newh, &launch));
    if (!launch) return DSPB200_OK;
    if (r == 0.0) r = 1.0;
    cudaStream_t st = (cudaStream_t)stream;
    StftStreamArgs sa{hist_in, nhist, ldh, ldo};
    sa.keep_plan = true;                                 // the same rounding whatever the chunking
    // launch 1: the seam copy (fused sizes: v[0, ls) of every channel, the samples of the units that start in the history)
    // and the new history
    const StreamSeam sm = stream_seam(p, nhist, nx, nseg);
    DSP_TRY(stream_edge(p, sm, hist_in, nhist, ldh, x, nx, nchan, nseg * p->hop, newh, hist_out, st));
    sa.seam = p->seam.p;
    sa.lds = sm.lds;
    if (nseg == 0) return DSPB200_OK;
    // launch 2 (fused sizes; cuFFT sizes: three per batch): the transforms -- a multitaper plan's every taper row in the one
    // fused launch, or its tapers one after another through cuFFT
    if (p->ntapers >= 1) {
        if (!p->fused)
            return p->f64 ? mt_stream_generic<double>(p, sa, x, nx, nchan, nseg, out, st)
                          : mt_stream_generic<float>(p, sa, x, nx, nchan, nseg, out, st);
        sa.ntapers = (int)p->ntapers;
    }
    return stft_launch(p, sa, x, nx, nchan, nseg, r, psd_only, out, st);
}

// Host twin (returns when the work is done): the chunk and the ldh x nchan histories are staged; the rows of hist_out past
// the new history are unspecified
int dspb200_stft_stream_exec(dspb200_spec_plan* plan, const void* hist_in, int64_t nhist, void* hist_out, int64_t ldh,
                             const void* x, int64_t nx, int64_t nchan, int64_t nseg, double r, int psd_only, void* out,
                             int64_t ldo) {
    DSP_RANGE("dspb200_stft_stream_exec");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    SpecPlanImpl* p = &plan->impl;
    int64_t newh = 0;
    bool launch = false;
    DSP_TRY(stft_stream_check(p, hist_in, nhist, hist_out, ldh, x, nx, nchan, nseg, r, psd_only, out, ldo, false, &newh, &launch));
    if (!launch) return DSPB200_OK;
    DSP_TRY(ensure_streams(p));
    const size_t esz = dtype_size(p->dtype), oel = (psd_only ? 1 : 2) * (p->f64 ? 8 : 4);
    const size_t hbytes = (size_t)(ldh * nchan) * esz;
    const size_t obytes = nseg ? (size_t)(((nchan - 1) * ldo + nseg) * p->nout) * oel : 0;
    return run_staged(p->pipe.s_exec, {{x, (size_t)(nx * nchan) * esz, &p->pipe.in[0]}, {hist_in, hist_in ? hbytes : 0, &p->hin}},
                      {{out, obytes, &p->pipe.out[0]}, {hist_out, newh ? hbytes : 0, &p->hout}}, [&] {
                          return dspb200_stft_stream_exec_dev(plan, hist_in ? p->hin.p : nullptr, nhist, p->hout.p, ldh, p->pipe.in[0].p,
                                                              nx, nchan, nseg, r, psd_only, p->pipe.out[0].p, ldo, p->pipe.s_exec);
                      });
}

// Streaming Welch.  Checks shared by both forms (those of the STFT stream, acc in place of out)
static int welch_stream_check(const SpecPlanImpl* p, const void* hist_in, int64_t nhist, const void* hist_out, int64_t ldh,
                              const void* x, int64_t nx, int64_t nchan, int64_t nseg, const double* acc, int add, bool dev,
                              int64_t* newh, bool* launch) {
    *launch = false;
    DSP_REQUIRE(nhist >= 0 && nx >= 0 && nchan >= 0 && nseg >= 0 && ldh >= 0, "negative size");
    DSP_REQUIRE(add == 0 || add == 1, "add must be 0 (write acc) or 1 (add to acc)");
    const size_t abytes = nseg ? (size_t)(p->nout * nchan) * sizeof(double) : 0;
    return stream_check(p, hist_in, nhist, hist_out, ldh, x, nx, nchan, nseg, acc, abytes, "acc", dev, newh, launch);
}

// Segments 0 .. nseg - 1 of every channel's virtual column [hist_in (nhist); x (nx)] into acc, then the new history
// v[nseg hop, nhist + nx) into hist_out.  Fused sizes: at most four launches per channel group, one without segments.
int dspb200_welch_stream_exec_dev(dspb200_spec_plan* plan, const void* hist_in, int64_t nhist, void* hist_out, int64_t ldh,
                                  const void* x, int64_t nx, int64_t nchan, int64_t nseg, double* acc, int add, void* stream) {
    DSP_RANGE("dspb200_welch_stream_exec_dev");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    SpecPlanImpl* p = &plan->impl;
    int64_t newh = 0;
    bool launch = false;
    DSP_TRY(welch_stream_check(p, hist_in, nhist, hist_out, ldh, x, nx, nchan, nseg, acc, add, true, &newh, &launch));
    if (!launch) return DSPB200_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const StreamSeam sm = stream_seam(p, nhist, nx, nseg);
    DSP_TRY(stream_edge(p, sm, hist_in, nhist, ldh, x, nx, nchan, nseg * p->hop, newh, hist_out, st));
    if (nseg == 0) return DSPB200_OK;
    if (p->fused)
        return fused_dispatch(p, "Welch", [&](auto t, auto nn) {
            using T = decltype(t);
            constexpr int N = decltype(nn)::value;
            return p->cplx ? welch_stream_fused<T, N, true>(p, sm, x, nx, nhist, nchan, nseg, acc, add, st)
                           : welch_stream_fused<T, N, false>(p, sm, x, nx, nhist, nchan, nseg, acc, add, st);
        });
    return welch_generic(p, hist_in, nhist, ldh, x, nx, nchan, nseg, acc, add, st);
}

// Host twin (returns when the work is done): the chunk, the histories and acc are staged
int dspb200_welch_stream_exec(dspb200_spec_plan* plan, const void* hist_in, int64_t nhist, void* hist_out, int64_t ldh,
                              const void* x, int64_t nx, int64_t nchan, int64_t nseg, double* acc, int add) {
    DSP_RANGE("dspb200_welch_stream_exec");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    SpecPlanImpl* p = &plan->impl;
    int64_t newh = 0;
    bool launch = false;
    DSP_TRY(welch_stream_check(p, hist_in, nhist, hist_out, ldh, x, nx, nchan, nseg, acc, add, false, &newh, &launch));
    if (!launch) return DSPB200_OK;
    DSP_TRY(ensure_streams(p));
    const size_t esz = dtype_size(p->dtype);
    const size_t hbytes = (size_t)(ldh * nchan) * esz, abytes = nseg ? (size_t)(p->nout * nchan) * sizeof(double) : 0;
    return run_staged(p->pipe.s_exec, {{x, (size_t)(nx * nchan) * esz, &p->pipe.in[0]}, {hist_in, hist_in ? hbytes : 0, &p->hin}, {acc, add ? abytes : 0, &p->pipe.out[0]}},
                      {{acc, abytes, &p->pipe.out[0]}, {hist_out, newh ? hbytes : 0, &p->hout}}, [&] {
                          return dspb200_welch_stream_exec_dev(plan, hist_in ? p->hin.p : nullptr, nhist, p->hout.p, ldh, p->pipe.in[0].p,
                                                               nx, nchan, nseg, reinterpret_cast<double*>(p->pipe.out[0].p), add, p->pipe.s_exec);
                      });
}

int dspb200_welch_stream_power_dev(dspb200_spec_plan* plan, const double* acc, int64_t nchan, double r, void* out, void* stream) {
    DSP_RANGE("dspb200_welch_stream_power_dev");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    DSP_REQUIRE(nchan >= 0, "negative size");
    DSP_REQUIRE(r != 0.0, "r must be nonzero");
    SpecPlanImpl* p = &plan->impl;
    if (nchan == 0) return DSPB200_OK;
    DSP_REQUIRE(acc && out, "NULL argument");
    DSP_REQUIRE(!ranges_overlap(out, (size_t)(p->nout * nchan) * (p->f64 ? 8 : 4), acc, (size_t)(p->nout * nchan) * sizeof(double)),
                "out overlaps acc");
    return welch_power(p, acc, nchan, r, out, (cudaStream_t)stream);
}

int dspb200_welch_stream_power(dspb200_spec_plan* plan, const double* acc, int64_t nchan, double r, void* out) {
    DSP_RANGE("dspb200_welch_stream_power");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    DSP_REQUIRE(nchan >= 0, "negative size");
    DSP_REQUIRE(r != 0.0, "r must be nonzero");
    SpecPlanImpl* p = &plan->impl;
    if (nchan == 0) return DSPB200_OK;
    DSP_REQUIRE(acc && out, "NULL argument");
    DSP_TRY(ensure_streams(p));
    const size_t n = (size_t)(p->nout * nchan);
    return run_staged(p->pipe.s_exec, {{acc, n * sizeof(double), &p->pipe.in[0]}}, {{out, n * (p->f64 ? 8 : 4), &p->pipe.out[0]}}, [&] {
        return dspb200_welch_stream_power_dev(plan, reinterpret_cast<const double*>(p->pipe.in[0].p), nchan, r, p->pipe.out[0].p, p->pipe.s_exec);
    });
}

// Multitaper (SURVEY.md 8f rank 1; src/multitaper.jl:117-242, 262-404).  The plan's window holds `ntapers` rows of n
// samples, each PRE-SCALED by 1/sqrt(r_t) (r_t = fs * sum|w_t|^2 / weight_t, :135-139), so that
//   mt_pgram       = sum_t fft2pow!(FFT(w_t .* s), 1)
//   mt_spectrogram = sum_t spectrogram(s; window = w_t, r = 1)
// of each of the nchan columns of a len x nchan matrix, every channel's tapers summed in taper order (the vector forms are
// nchan = 1).  Fused sizes: mt_pgram is launch_mt_pgram (two launches per channel group), mt_spectrogram ONE launch of the
// STFT kernels' taper-row instances (WIN == 2).  cuFFT sizes: mt_pgram_generic; mt_spectrogram is mt_stream_generic with no
// history (one batched STFT over all channels per taper, each after the first followed by acc_add_cols_kernel).  A stream of
// mt_spectrogram is the STFT stream call on a multitaper plan (dspb200_stft_stream_exec_dev: the same WIN == 2 launch, or
// mt_stream_generic).
static size_t mt_out_bytes(const SpecPlanImpl* p, int64_t nchan, int64_t k) {
    return (size_t)(p->nout * k * nchan) * (p->f64 ? 8 : 4);
}
// The checks of every form, before any launch.  *k: columns per channel (mt_pgram: 1); *launch = false when there is nothing
// to do (no channel, or no segment).
static int mt_batch_check(const dspb200_spec_plan* plan, const void* s, int64_t len, int64_t nchan, const void* out, bool pgram,
                          bool dev, int64_t* k, bool* launch) {
    *launch = false;
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    const SpecPlanImpl* p = &plan->impl;
    DSP_REQUIRE(p->ntapers >= 1, "not a multitaper plan");
    DSP_REQUIRE(len >= 0 && nchan >= 0, "negative size");
    if (pgram) DSP_REQUIRE(len == p->n, "Expected `signal` to be of length `config.n_samples`");    // DimensionMismatch :226
    *k = pgram ? 1 : nsegments(p, len);
    if (nchan == 0 || *k == 0) return DSPB200_OK;
    DSP_REQUIRE(s && out, "NULL argument");
    // the kernels read every channel's samples while other CTAs write `out`
    DSP_REQUIRE(!dev || !ranges_overlap(out, mt_out_bytes(p, nchan, *k), s, (size_t)(len * nchan) * dtype_size(p->dtype)),
                "out overlaps s");
    *launch = true;
    return DSPB200_OK;
}

static int mt_pgram_queue(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t nchan, void* out, cudaStream_t st) {
    SpecPlanImpl* p = &plan->impl;
    if (p->fused)
        return fused_dispatch(p, "Welch", [&](auto t, auto nn) {
            using T = decltype(t);
            constexpr int N = decltype(nn)::value;
            return p->cplx ? launch_mt_pgram<T, N, true>(p, s, len, nchan, out, st) : launch_mt_pgram<T, N, false>(p, s, len, nchan, out, st);
        });
    return p->f64 ? mt_pgram_generic<double>(p, s, len, nchan, out, st) : mt_pgram_generic<float>(p, s, len, nchan, out, st);
}

static int mt_spectrogram_queue(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t nchan, int64_t k, void* out,
                                cudaStream_t st) {
    SpecPlanImpl* p = &plan->impl;
    StftStreamArgs sa;                                   // no history; columns k apart
    sa.ldo = k;
    if (!p->fused)
        return p->f64 ? mt_stream_generic<double>(p, sa, s, len, nchan, k, out, st)
                      : mt_stream_generic<float>(p, sa, s, len, nchan, k, out, st);
    sa.ntapers = (int)p->ntapers;                        // every taper row in the one launch
    return stft_launch(p, sa, s, len, nchan, k, 1.0, 1, out, st);
}

int dspb200_mt_pgram_batch_exec_dev(dspb200_spec_plan* plan, const void* d_s, int64_t len, int64_t nchan, void* d_out,
                                    void* stream) {
    DSP_RANGE("dspb200_mt_pgram_batch_exec_dev");
    int64_t k = 0;
    bool launch = false;
    DSP_TRY(mt_batch_check(plan, d_s, len, nchan, d_out, true, true, &k, &launch));
    if (!launch) return DSPB200_OK;
    DSP_CUDA(cudaSetDevice(plan->impl.device));
    cudaStream_t st = (cudaStream_t)stream;
    return settle(st, mt_pgram_queue(plan, d_s, len, nchan, d_out, st));
}
int dspb200_mt_pgram_batch_exec(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t nchan, void* out) {
    DSP_RANGE("dspb200_mt_pgram_batch_exec");
    int64_t k = 0;
    bool launch = false;
    DSP_TRY(mt_batch_check(plan, s, len, nchan, out, true, false, &k, &launch));
    if (!launch) return DSPB200_OK;
    SpecPlanImpl* p = &plan->impl;
    DSP_TRY(ensure_streams(p));
    return run_staged(p->pipe.s_exec, {{s, (size_t)(len * nchan) * dtype_size(p->dtype), &p->pipe.in[0]}},
                      {{out, mt_out_bytes(p, nchan, k), &p->pipe.out[0]}},
                      [&] { return dspb200_mt_pgram_batch_exec_dev(plan, p->pipe.in[0].p, len, nchan, p->pipe.out[0].p, p->pipe.s_exec); });
}
int dspb200_mt_pgram_exec_dev(dspb200_spec_plan* plan, const void* d_s, int64_t len, void* d_out, void* stream) {
    return dspb200_mt_pgram_batch_exec_dev(plan, d_s, len, 1, d_out, stream);
}
int dspb200_mt_pgram_exec(dspb200_spec_plan* plan, const void* s, int64_t len, void* out) {
    return dspb200_mt_pgram_batch_exec(plan, s, len, 1, out);
}

int dspb200_mt_spectrogram_batch_exec_dev(dspb200_spec_plan* plan, const void* d_s, int64_t len, int64_t nchan, void* d_out,
                                          void* stream) {
    DSP_RANGE("dspb200_mt_spectrogram_batch_exec_dev");
    int64_t k = 0;
    bool launch = false;
    DSP_TRY(mt_batch_check(plan, d_s, len, nchan, d_out, false, true, &k, &launch));
    if (!launch) return DSPB200_OK;
    DSP_CUDA(cudaSetDevice(plan->impl.device));
    cudaStream_t st = (cudaStream_t)stream;
    return settle(st, mt_spectrogram_queue(plan, d_s, len, nchan, k, d_out, st));
}
int dspb200_mt_spectrogram_batch_exec(dspb200_spec_plan* plan, const void* s, int64_t len, int64_t nchan, void* out) {
    DSP_RANGE("dspb200_mt_spectrogram_batch_exec");
    int64_t k = 0;
    bool launch = false;
    DSP_TRY(mt_batch_check(plan, s, len, nchan, out, false, false, &k, &launch));
    if (!launch) return DSPB200_OK;
    SpecPlanImpl* p = &plan->impl;
    DSP_TRY(ensure_streams(p));
    return run_staged(p->pipe.s_exec, {{s, (size_t)(len * nchan) * dtype_size(p->dtype), &p->pipe.in[0]}},
                      {{out, mt_out_bytes(p, nchan, k), &p->pipe.out[0]}},
                      [&] { return dspb200_mt_spectrogram_batch_exec_dev(plan, p->pipe.in[0].p, len, nchan, p->pipe.out[0].p, p->pipe.s_exec); });
}
int dspb200_mt_spectrogram_exec_dev(dspb200_spec_plan* plan, const void* d_s, int64_t len, void* d_out, void* stream) {
    return dspb200_mt_spectrogram_batch_exec_dev(plan, d_s, len, 1, d_out, stream);
}
int dspb200_mt_spectrogram_exec(dspb200_spec_plan* plan, const void* s, int64_t len, void* out) {
    return dspb200_mt_spectrogram_batch_exec(plan, s, len, 1, out);
}

static int mt_cross_check(dspb200_spec_plan* plan, const void* signal, int64_t nchan, int64_t f_lo, int64_t nf, void* out) {
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    SpecPlanImpl* p = &plan->impl;
    DSP_REQUIRE(p->ntapers >= 1, "not a multitaper plan");
    DSP_REQUIRE(!p->cplx && p->onesided,
                "Only real data is supported (with the default choice of `onesided=true`) for this operation.");   // :411-416
    DSP_REQUIRE(nchan >= 1, "n_channels must be positive");
    DSP_REQUIRE(f_lo >= 0 && nf >= 0 && f_lo + nf <= p->nout, "frequency range outside the spectrum");
    DSP_REQUIRE(nf == 0 || (signal && out), "NULL argument");
    return DSPB200_OK;
}
// The epoch form's checks on top of mt_cross_check: nepochs >= 1, every index and byte count of the signal and the output
// inside DSPB200_INDEX_LIMIT, and (device form) an output that does not overlap the signal
static int mt_cross_epochs_check(dspb200_spec_plan* plan, const void* signal, int64_t nchan, int64_t nepochs, int64_t f_lo,
                                 int64_t nf, int coherence, void* out, bool dev) {
    DSP_TRY(mt_cross_check(plan, signal, nchan, f_lo, nf, out));
    DSP_REQUIRE(nepochs >= 1, "n_epochs must be positive");
    const SpecPlanImpl* p = &plan->impl;
    const int64_t lim = DSPB200_INDEX_LIMIT / 16, esz = p->f64 ? 8 : 4;
    DSP_REQUIRE(nchan <= INT32_MAX && p->n <= lim / nchan && nepochs <= lim / (nchan * p->n) &&
                (nf == 0 || nchan <= lim / nchan / nf), "signal or output past DSPB200_INDEX_LIMIT");
    if (dev) {
        const size_t sbytes = (size_t)(nchan * p->n * nepochs * esz);
        const size_t obytes = (size_t)(nchan * nchan * nf * esz * (coherence ? 1 : 2));
        DSP_REQUIRE(!ranges_overlap(signal, sbytes, out, obytes), "out overlaps the signal");
    }
    return DSPB200_OK;
}
static int mt_cross_dev(dspb200_spec_plan* plan, const void* d_signal, int64_t nchan, int64_t nepochs, int demean, int64_t f_lo,
                        int64_t nf, int coherence, void* d_out, void* stream) {
    if (nf == 0) return DSPB200_OK;
    SpecPlanImpl* p = &plan->impl;
    DSP_TRY(ensure_streams(p));
    cudaStream_t st = (cudaStream_t)stream;
    return settle(st, p->f64 ? mt_cross_run<double>(plan, d_signal, nchan, nepochs, demean, f_lo, nf, coherence, d_out, st)
                             : mt_cross_run<float>(plan, d_signal, nchan, nepochs, demean, f_lo, nf, coherence, d_out, st));
}
int dspb200_mt_cross_spectra_exec_dev(dspb200_spec_plan* plan, const void* d_signal, int64_t nchan, int demean, int64_t f_lo,
                                      int64_t nf, int coherence, void* d_out, void* stream) {
    DSP_RANGE("dspb200_mt_cross_spectra_exec_dev");
    DSP_TRY(mt_cross_check(plan, d_signal, nchan, f_lo, nf, d_out));
    return mt_cross_dev(plan, d_signal, nchan, 1, demean, f_lo, nf, coherence, d_out, stream);
}
int dspb200_mt_cross_spectra_epochs(dspb200_spec_plan* plan, const void* d_signal, int64_t nchan, int64_t nepochs, int demean,
                                    int64_t f_lo, int64_t nf, int coherence, void* d_out, void* stream) {
    DSP_RANGE("dspb200_mt_cross_spectra_epochs");
    DSP_TRY(mt_cross_epochs_check(plan, d_signal, nchan, nepochs, f_lo, nf, coherence, d_out, true));
    return mt_cross_dev(plan, d_signal, nchan, nepochs, demean, f_lo, nf, coherence, d_out, stream);
}
// Host pointers: the signal is staged in pipe.in[0] and the result in pipe.out[1], which the device form does not use.
int dspb200_mt_cross_spectra_epochs_exec(dspb200_spec_plan* plan, const void* signal, int64_t nchan, int64_t nepochs, int demean,
                                         int64_t f_lo, int64_t nf, int coherence, void* out) {
    DSP_RANGE("dspb200_mt_cross_spectra_epochs_exec");
    DSP_TRY(mt_cross_epochs_check(plan, signal, nchan, nepochs, f_lo, nf, coherence, out, false));
    if (nf == 0) return DSPB200_OK;
    SpecPlanImpl* p = &plan->impl;
    DSP_TRY(ensure_streams(p));
    HostPipe& hp = p->pipe;
    const size_t esz = p->f64 ? 8 : 4, out_bytes = (size_t)(nchan * nchan * nf) * esz * (coherence ? 1 : 2);
    return run_staged(hp.s_exec, {{signal, (size_t)(p->n * nchan * nepochs) * esz, &hp.in[0]}}, {{out, out_bytes, &hp.out[1]}}, [&] {
        return dspb200_mt_cross_spectra_epochs(plan, hp.in[0].p, nchan, nepochs, demean, f_lo, nf, coherence, hp.out[1].p, hp.s_exec);
    });
}
// Host pointers: the signal is staged in pipe.in[0] and the result in pipe.out[1], which the device form does not use.
int dspb200_mt_cross_spectra_exec(dspb200_spec_plan* plan, const void* signal, int64_t nchan, int demean, int64_t f_lo,
                                  int64_t nf, int coherence, void* out) {
    DSP_RANGE("dspb200_mt_cross_spectra_exec");
    DSP_TRY(mt_cross_check(plan, signal, nchan, f_lo, nf, out));
    if (nf == 0) return DSPB200_OK;
    SpecPlanImpl* p = &plan->impl;
    DSP_TRY(ensure_streams(p));
    HostPipe& hp = p->pipe;
    const size_t esz = p->f64 ? 8 : 4, out_bytes = (size_t)(nchan * nchan * nf) * esz * (coherence ? 1 : 2);
    return run_staged(hp.s_exec, {{signal, (size_t)(p->n * nchan) * esz, &hp.in[0]}}, {{out, out_bytes, &hp.out[1]}}, [&] {
        return dspb200_mt_cross_spectra_exec_dev(plan, hp.in[0].p, nchan, demean, f_lo, nf, coherence, hp.out[1].p, hp.s_exec);
    });
}

// periodogram(s::AbstractMatrix; nfft, fs, radialsum, radialavg), src/periodograms.jl:473-509 (cached plan + scratch arena)
static int periodogram2_check(int dtype, const void* s, int64_t n1, int64_t n2, int64_t nfft1, int64_t nfft2, double r, int ptype,
                              void* out) {
    DSP_REQUIRE(dtype == DSPB200_F32 || dtype == DSPB200_F64, "periodogram of a matrix takes a real signal (dtype %d)", dtype);
    DSP_REQUIRE(s && out, "NULL argument");
    DSP_REQUIRE(n1 > 1 && n2 > 1, "dimensions of s must be > 1");                                   // :478
    DSP_REQUIRE(n1 <= nfft1 && n2 <= nfft2, "nfft must be >= size(s)");                             // :477
    DSP_REQUIRE(nfft1 < (int64_t(1) << 31) && nfft2 < (int64_t(1) << 31), "nfft too large");
    DSP_REQUIRE(ptype >= 0 && ptype <= 2 && r != 0.0, "bad ptype or r");
    return DSPB200_OK;
}
static int periodogram2_queue(int dtype, const void* d_s, int64_t n1, int64_t n2, int64_t nfft1, int64_t nfft2, double r, int ptype,
                              void* d_out, cudaStream_t st) {
    return dtype == DSPB200_F64 ? periodogram2_run<double>(d_s, n1, n2, nfft1, nfft2, r, ptype, d_out, st)
                                : periodogram2_run<float>(d_s, n1, n2, nfft1, nfft2, r, ptype, d_out, st);
}
int dspb200_periodogram2_exec(int dtype, const void* s, int64_t n1, int64_t n2, int64_t nfft1, int64_t nfft2, double r, int ptype,
                              void* out) {
    DSP_RANGE("dspb200_periodogram2_exec");
    DSP_TRY(periodogram2_check(dtype, s, n1, n2, nfft1, nfft2, r, ptype, out));
    const size_t esz = dtype_size(dtype);
    const int64_t nmin = nfft1 < nfft2 ? nfft1 : nfft2, nout = ptype == 0 ? nfft1 * nfft2 : nmin / 2 + 1;
    DevBuf &ds = scratch_buf(0), &dout = scratch_buf(3);
    return convenience_call({{s, (size_t)(n1 * n2) * esz, &ds}}, {{out, (size_t)nout * esz, &dout}}, [&](cudaStream_t st) {
        return periodogram2_queue(dtype, ds.p, n1, n2, nfft1, nfft2, r, ptype, dout.p, st);
    });
}
int dspb200_periodogram2_exec_dev(int dtype, const void* d_s, int64_t n1, int64_t n2, int64_t nfft1, int64_t nfft2, double r,
                                  int ptype, void* d_out, void* stream) {
    DSP_RANGE("dspb200_periodogram2_exec_dev");
    DSP_TRY(periodogram2_check(dtype, d_s, n1, n2, nfft1, nfft2, r, ptype, d_out));
    return convenience_call((cudaStream_t)stream, [&](cudaStream_t st) {
        return periodogram2_queue(dtype, d_s, n1, n2, nfft1, nfft2, r, ptype, d_out, st);
    });
}

int dspb200_spec_plan_destroy(dspb200_spec_plan* plan) {
    if (!plan) return DSPB200_OK;
    SpecPlanImpl* p = &plan->impl;
    if (p->d_window) cudaFree(p->d_window);
    if (p->d_tw) cudaFree(p->d_tw);
    if (p->d_t16) cudaFree(p->d_t16);
    if (p->d_t32) cudaFree(p->d_t32);
    if (p->d_t256) cudaFree(p->d_t256);
    p->partial.release(); p->bpartial.release(); p->bacc.release(); p->segbuf.release(); p->specbuf.release(); p->acc.release();
    p->tmp.release(); p->hin.release(); p->hout.release(); p->seam.release(); p->y.release();
    if (p->fft_ok) cufftDestroy(p->fft);
    p->pipe.release();
    delete plan;
    return DSPB200_OK;
}

}  // extern "C"
