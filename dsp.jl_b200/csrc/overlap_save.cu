// dspb200 -- overlap-save FFT convolution / filtering, single-FFT convolution, direct convolution.
//
// Reference path: unsafe_conv_kern_os! (src/dspbase.jl:490-609), os_prepare_conv / os_filter_transform! /
// os_conv_block! (:299-356), _fftfilt! (src/Filters/filt.jl:479-521), _conv_kern_fft! (src/dspbase.jl:611-644),
// _conv_td! (:646-660).
//
// Fused kernel (power-of-two nfft in shared memory): one CTA per block of L = nfft - nv + 1 outputs
//   global load (nv-1 sample halo, zero outside the signal) -> forward passes -> [last pass, x H, first pass of the
//   second transform in registers] -> remaining passes -> store the valid L samples.
// Each sample is read once and written once from/to HBM; the nv-1 halo re-read comes from L2.  Real signals ride two blocks per complex FFT (z = a + i b; h real => y = a*h + i b*h).
// H carries the 1/nfft of the unnormalised inverse (src/dspbase.jl:516, src/Filters/filt.jl:498).
#include "fft_core.cuh"
#include "async_copy.cuh"
#include "cufft_exec.cuh"
#include <math.h>
#include <stdlib.h>
#include <new>
#include <vector>

namespace dspb200 {

struct OsPlanImpl {
    int dtype = 0;
    bool cplx = false, f64 = false;
    int64_t nv = 0, nfft = 0, L = 0;
    bool fused = false;
    int device = 0;
    void* d_tw = nullptr;   // fused: last-pass twiddle table (fft_fill_tl)
    void* d_t16 = nullptr;  // fused: radix-16 twiddle tables
    void* d_t256 = nullptr;
    void* d_r32 = nullptr;  // fused 16384-point Float32: tables of the 32 · 32 · 16 plan (fft_r32_fill_tables)
    int sm_count = 0;               // device_sm_count() at plan creation
    int fused_per_sm = 0;   // resident CTAs per SM of this plan's fused kernel (occupancy calculator, asked once)
    int fused_state_per_sm = 0;     // the same for its stateful instance
    void* d_H = nullptr;    // natural order; fused: cx<T>[nfft] pre-scaled by 1/nfft; generic: nfft or nfft/2+1 bins
    // generic
    cufftHandle fwd = 0, inv = 0;
    bool fft_ok = false;
    int64_t batch = 0, nbins = 0;
    DevBuf td, fd;
    HostPipe pipe;          // host-pointer calls
};

template <typename T, bool CPLX> struct os_elt { using type = T; };
template <typename T> struct os_elt<T, true> { using type = cx<T>; };

// ---------------------------------------------------------------------------------------------- fused kernel
// Geometry (0-based): block q of a column produces outputs m in [out_begin + q*L, out_begin + (q+1)*L);
// its buffer slot j holds input sample i = out_begin + q*L - (nv-1) + j, and slot j >= nv-1 of the result
// is output m = out_begin + q*L + j - (nv-1).  Input samples outside [u_begin, u_begin+nu_local) are zero.
// Persistent CTAs stride over the units (unit = one complex block or two real blocks), neighbouring CTAs work
// on neighbouring blocks at the same time so the nv-1 sample halo is an L2 hit.
//
// One unit (fft_core.cuh):  first pass (global loads, thread c reads u[i0 + c + r N/16]: coalesced)  | middle passes |
// [last forward pass -> x H -> swap -> first pass of the second transform] in registers | middle passes | last pass ->
// global stores (thread t writes y[t + r N/16]: coalesced).  H is in natural order (the forward transform ends in
// natural order), pre-scaled by 1/N; thread t reads H[t + r N/16]: coalesced, no tiling needed.
// The 16384-point Float32 kernels (os_threads::staged) run the 32 · 32 · 16 plan instead (os_unit_r32: first | radix-32 |
// [last, x H, swap, first] | radix-32 | last), and read an interior unit's input from shared memory: two TMA bulk copies,
// issued during the previous unit, put the span in natural order in front of and at the head of the data buffer (OsStage).
// Probes of that kernel's per-unit transfers (2^26 ComplexF32 samples, 4097 taps, H100 SXM 80 GB at 700 W, before staging):
// conv 0.660 .. 0.667 ms; without the input loads 0.607 .. 0.614, without the H loads 0.628 .. 0.637, without the output
// stores 0.543 .. 0.546.

// Launch shape of the fused kernel per size, from a "resident threads" sweep on an earlier GPU generation; the 16384-point
// Float32 kernels have been measured again on the H100.  On sm_90a the 128-register 8192-point instances spill (Float32
// real / complex 260 / 280 bytes, Float64 232 / 240 bytes), so their shape is the next one to re-measure there:
//  * N = 512 .. 4096 (and the real N = 256 kernel): 1024 resident threads per SM under a 64-register cap, one radix-16
//    butterfly in flight per thread -- the extra warps hide the shared-memory latency (faster than 512 threads with two
//    butterflies in flight under a 128-register cap);
//  * complex N = 16384 (one CTA per SM: its shared memory holds one block): 512 threads, 128 registers, two butterflies in
//    flight: on the H100 it is faster than 1024 threads with one butterfly each under a 64-register cap, the earlier
//    generation's choice (2^26 samples, 4097 taps, H100 80 GB HBM3 at 400 W, alternating: conv 0.695 .. 0.704 against
//    0.795 .. 0.801 ms).  Its transform runs as 32 · 32 · 16 (fft_r32): one radix-32 butterfly per thread in the first and
//    middle passes, two radix-16 ones in the last, no spills; against 16 · 16 · 16 · 4 at the same shape (2^26 samples,
//    4097 taps, H100 80GB HBM3 at 700 W, alternating): conv 0.543 .. 0.548 against 0.589 .. 0.595 ms, and the real
//    one-shot fftfilt of 64 x 2^20 Float32 with 4097 taps 0.380 .. 0.383 against 0.395 .. 0.399 ms.  Splitting the block
//    over a two-CTA cluster so that two 512-thread, 64-register CTAs share each
//    SM does not pay there either: a 512-thread, 64-register 8192-point
//    kernel at two CTAs per SM costs 0.43 of a 16384-point unit per unit (0.46 with the store count of half a
//    16384-point block; transform length alone gives 0.46 .. 0.5), which leaves no room for the exchange.  Its next unit's
//    input is staged by TMA (OsStage), and the last pass reads both butterflies' operands before any math (the copy may
//    overwrite the buffer once they are in registers); an earlier prefetch of those samples into registers spilled;
//  * N = 8192, real N = 16384: 512 resident threads, 128 registers, two butterflies in flight (the 64-register
//    build spilled there when the shape was chosen).  Double precision: one CTA of up to 256 registers per thread.
template <typename T, int N, bool CPLX> struct os_threads {
    static constexpr bool f32 = sizeof(T) == 4;
    static constexpr int value = fft_threads<N>::value;
    static constexpr bool wide = f32 && ((N >= 512 && N <= 4096) || (N == 256 && !CPLX));     // 1024 resident threads
    static constexpr int minblocks = wide ? 1024 / value : fft_minblocks<T, N>::value;
    // the 16384-point Float32 kernels at 512 threads (two butterflies per thread in every pass): the next unit's input is
    // staged in shared memory by TMA while the current one runs (OsStage)
    static constexpr bool staged = f32 && N == 16384;
};
// Staged kernels: the first OS_STAGE_HEAD bytes of a unit's span land in a region of their own right in front of the data
// buffer (32 KB of the 33 KB the 16384-point block leaves free), the rest at the data buffer's head -- contiguous, so the
// first pass reads slot j at head + j.  The head region is free again once the first pass has read it, so its copy for
// the next unit is issued there, a whole unit ahead; only the rest has to arrive during the last pass.  Copying the whole
// span during the last pass instead was slower in both sessions that compared the two (2^26 ComplexF32 samples, 4097 taps,
// H100 SXM 80 GB at 400 W, alternating, 3 runs each): conv 0.655 .. 0.657 against 0.649 .. 0.654 ms, and on another card
// 0.671 .. 0.672 against 0.668 .. 0.671 ms.
constexpr int OS_STAGE_HEAD = 32768;
static_assert(OS_STAGE_HEAD % 16 == 0, "TMA copies move multiples of 16 bytes");
static_assert(OS_STAGE_HEAD < 16384 * 4, "the head region holds less than the shortest staged span (N + 1 floats)");
// data buffer and twiddle tables of the fused kernel, in elements of cx<T>: the staged kernels run the 32 · 32 · 16 plan
template <typename T, int N, bool CPLX> __host__ __device__ constexpr int os_fft_elems() {
    return os_threads<T, N, CPLX>::staged ? fft_r32::SMEM_ELEMS : fft_smem_elems<T, N>();
}
// dynamic shared memory of the fused kernel: (staged kernels) head region, data buffer and twiddle tables, then (staged
// kernels) the copies' mbarrier
template <typename T, int N, bool CPLX> constexpr size_t os_smem_bytes() {
    return (size_t)os_fft_elems<T, N, CPLX>() * sizeof(cx<T>) + (os_threads<T, N, CPLX>::staged ? OS_STAGE_HEAD + 16 : 0);
}

template <typename T> __device__ __forceinline__ cx<T> ldg_cx(const cx<T>* __restrict__ p) {
    if constexpr (sizeof(T) == 4) {
        const float2 v = __ldg(reinterpret_cast<const float2*>(p));
        return mkc<T>(v.x, v.y);
    } else {
        const double2 v = __ldg(reinterpret_cast<const double2*>(p));
        return mkc<T>(v.x, v.y);
    }
}

// Per-unit geometry in slot coordinates j (0 <= j < N, block B of a real pair: j + L), 32-bit: u[j] is the sample in
// slot j, out[j] the output produced by slot j >= nv-1; slot j holds a stored sample iff jlo <= j < jhi, its output is
// wanted iff j < jend and is an exact zero (src/dspbase.jl:733-735) from jzero on.
template <typename E> struct OsUnit {
    const E* u;
    E* out;
    int jlo, jhi, jend, jzero;
    int nvm1, L;
};

// Stateful calls (DF2TFilter, dspb200_os_exec_state_dev): a column's call computes the outputs o in [0, nx + nv - 1) of
// conv(v, x); o < nv - 1 adds the incoming transposed direct-form state si_in[o], o >= nx is the outgoing state
// si_out[o - nx], the rest is out[o].  si_in / si_out hold nv - 1 elements per column; si_in may be NULL (zero state); without
// si_out the call computes only the nx outputs.  Only edge units touch the state: an interior unit's outputs lie in
// [nv - 1, nx).  The stateless instances take the empty struct, so their parameters and code are those of before.
template <typename E, bool STATE> struct OsState {};
template <typename E> struct OsState<E, true> {
    const E* si_in;
    E* si_out;
    int64_t nx;
};
// The state geometry of an edge unit of a stateful call: slot j's output is s0 + j; si_in / si_out are shifted so that index
// j addresses that output's state entry; slots j < jsi take incoming state, slots j >= jnx are outgoing state.  It is
// computed just before the last pass (os_fused_kernel's state_geometry), not carried through the transforms' registers.
template <typename E> struct OsUnitState {
    const E* si_in;
    E* si_out;
    int jsi, jnx;
};
struct OsNoState {};
template <typename E> __device__ __forceinline__ void os_put_state(const OsUnit<E>& g, const OsUnitState<E>& s, int j, E v) {
    if (j < s.jsi) v = v + s.si_in[j];
    if (j < s.jnx) g.out[j] = v;
    else s.si_out[j] = v;
}

__device__ __forceinline__ int os_clamp(int64_t v) {
    return (int)(v < -(int64_t(1) << 30) ? -(int64_t(1) << 30) : (v > (int64_t(1) << 30) ? (int64_t(1) << 30) : v));
}
// clamp(a - b) for a that may be INT64_MAX ("no limit") and |b| < 2^62: no signed overflow
__device__ __forceinline__ int os_clamp_diff(int64_t a, int64_t b) {
    return a >= (int64_t(1) << 62) ? (1 << 30) : os_clamp(a - b);
}

// Sample in slot j of a unit (block A in .x, block B of a real pair in .y).
// INTERIOR: every input sample of the unit is stored and every output is wanted and non-zero -- no bounds tests at all
// (all units but the first and the last few of a column)
template <typename T, bool CPLX, bool INTERIOR>
__device__ __forceinline__ cx<T> os_sample(const OsUnit<typename os_elt<T, CPLX>::type>& g, int j) {
#if DSP_PROBE & 2
    return mkc<T>(T(j), T(1));
#endif
    if constexpr (CPLX) {
        if constexpr (INTERIOR) return g.u[j];
        return (j >= g.jlo && j < g.jhi) ? g.u[j] : mkc<T>(T(0), T(0));
    } else {
        const int jb = j + g.L;
        if constexpr (INTERIOR) return mkc<T>(g.u[j], g.u[jb]);
        const T a = (j >= g.jlo && j < g.jhi) ? g.u[j] : T(0);
        const T b = (jb >= g.jlo && jb < g.jhi) ? g.u[jb] : T(0);
        return mkc<T>(a, b);
    }
}

// TMA staging of a unit's input (os_threads::staged kernels), so that its L2 -> SM transfer does not stand alone at the head
// of the unit.  The NEXT unit's span arrives in two bulk copies completed on one mbarrier phase: its head region part is
// issued right after the current unit's first pass (which has read the head region), the rest in the current unit's
// last pass, once every thread has read its last-pass operands -- the data buffer is dead from there to the next first
// pass, so this copy overlaps the last pass's butterflies and global stores.
struct OsStage {
    unsigned char* head; // slot 0 of a staged span: OS_STAGE_HEAD bytes in front of the data buffer
    uint64_t* bar;       // mbarrier of the copies (shared memory behind the twiddle tables)
    uint32_t bytes;      // length of the span: the unit's input rounded up to 16 bytes
    uint32_t parity;     // phase of the next wait
};

// Output of slot j of a unit (y: swapped domain, result = (y.y, y.x)).  STATE: only the edge units' stores change
// (os_put_state, with the OsUnitState that state_geometry() returns).
template <typename T, bool CPLX, bool INTERIOR, bool STATE, typename SGeom>
__device__ __forceinline__ void os_put(const OsUnit<typename os_elt<T, CPLX>::type>& g, const SGeom& sg, int j, cx<T> y) {
#if DSP_PROBE & 8
    if (y.x != T(123456.75)) return;
#endif
    if (j < g.nvm1) return;
    if constexpr (CPLX) {
        if constexpr (INTERIOR) g.out[j] = mkc<T>(y.y, y.x);
        else if constexpr (STATE) { if (j < g.jend) os_put_state(g, sg, j, mkc<T>(y.y, y.x)); }
        else if (j < g.jend) g.out[j] = (j < g.jzero) ? mkc<T>(y.y, y.x) : mkc<T>(T(0), T(0));
    } else {
        const int jb = j + g.L;
        if constexpr (INTERIOR) {
            g.out[j] = y.y;
            g.out[jb] = y.x;
        } else if constexpr (STATE) {
            if (j < g.jend) os_put_state(g, sg, j, y.y);
            if (jb < g.jend) os_put_state(g, sg, jb, y.x);
        } else {
            if (j < g.jend) g.out[j] = (j < g.jzero) ? y.y : T(0);
            if (jb < g.jend) g.out[jb] = (jb < g.jzero) ? y.x : T(0);
        }
    }
}
template <typename E, bool STATE, bool INTERIOR> using os_sgeom_t = std::conditional_t<STATE && !INTERIOR, OsUnitState<E>, OsNoState>;

// One unit of the kernels that are not staged (fft_plan_traits<N>).
template <typename T, int N, bool CPLX, int NT, bool INTERIOR, int ITERS, bool STATE, typename SG>
__device__ __forceinline__ void os_unit(const FftCtx<T>& ctx, int tid, const OsUnit<typename os_elt<T, CPLX>::type>& g,
                                        const cx<T>* __restrict__ H, const SG& state_geometry) {
    using E = typename os_elt<T, CPLX>::type;
    constexpr int Q = fft_plan_traits<N>::Q;
    static_assert(ITERS == (Q + NT - 1) / NT, "register tile does not match the thread count");
    {
        // global loads; the barrier inside (between the first butterfly and its stores) also ends the previous unit's last
        // pass
        auto ld0 = [&](int j, int, int) -> cx<T> { return os_sample<T, CPLX, INTERIOR>(g, j); };
        fft_first_pass<T, N, NT, true>(ctx, tid, ld0);
    }
    __syncthreads();
    fft_middle<T, N, NT>(ctx, tid);
    // last forward pass, x H, swap, first pass of the second transform -- in registers
    cx<T> v[ITERS][16];
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
        const int tp = tid + it * NT;
        if (Q % NT == 0 || tp < Q) {
            fft_last_pass<T, N, (ITERS == 1 && Q % NT == 0) ? NT : 0>(ctx, tp, v[it], tid);
#pragma unroll
#if DSP_PROBE & 4
            for (int r = 0; r < 16; ++r) v[it][r] = cswap(cmul(v[it][r], mkc<T>(T(0.5), T(r))));
#else
            for (int r = 0; r < 16; ++r) v[it][r] = cswap(cmul(v[it][r], ldg_cx<T>(H + tp + r * Q)));
#endif
            fft_bfly16_plain<T>(v[it]);
        }
    }
    __syncthreads();                                   // every thread has read its last-pass inputs
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
        const int tp = tid + it * NT;
        if (Q % NT == 0 || tp < Q) fft_store_block<T, N>(ctx.sm, tp, v[it]);
    }
    __syncthreads();
    fft_middle<T, N, NT>(ctx, tid);
    constexpr int RL = fft_plan_traits<N>::RL, NBF = 16 / RL;
    os_sgeom_t<E, STATE, INTERIOR> sg{};
    if constexpr (STATE && !INTERIOR) sg = state_geometry();
    // last pass, streamed one radix-RL butterfly at a time -- RL live values instead of 16
    auto chunk = [&](auto a_, int tp) {
        constexpr int A = decltype(a_)::value;
        cx<T> u[RL];
        fft_last_pass_chunk<T, N, A>(ctx, tp, u);
#pragma unroll
        for (int jj = 0; jj < RL; ++jj) os_put<T, CPLX, INTERIOR, STATE>(g, sg, tp + (A + NBF * jj) * Q, u[jj]);
    };
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
        const int tp = tid + it * NT;
        if (Q % NT != 0 && tp >= Q) break;
        chunk(std::integral_constant<int, 0>{}, tp);
        if constexpr (NBF >= 2) chunk(std::integral_constant<int, 1>{}, tp);
        if constexpr (NBF >= 4) { chunk(std::integral_constant<int, 2>{}, tp); chunk(std::integral_constant<int, 3>{}, tp); }
        if constexpr (NBF >= 8) {
            chunk(std::integral_constant<int, 4>{}, tp); chunk(std::integral_constant<int, 5>{}, tp);
            chunk(std::integral_constant<int, 6>{}, tp); chunk(std::integral_constant<int, 7>{}, tp);
        }
    }
}

// One unit of the staged kernels (os_threads::staged: the 16384-point Float32 ones), in the 32 · 32 · 16 plan (fft_r32):
//   first | radix-32 | [last, x H, swap, first] | radix-32 | last
// Thread tid owns residue class tid of both first passes, butterfly tid of both radix-32 passes and the radix-16
// butterflies tid, tid + 512 of both last passes, whose outputs X[tid + 512 m], m < 32, are that residue class.
// staged: the unit's input span is (being) copied to OsStage::head; next_u: slot 0 of the next unit when that one is to be
// staged (os_fused_kernel decides), else null.
template <typename T, bool CPLX, bool INTERIOR, bool STATE, typename SG>
__device__ __forceinline__ void os_unit_r32(const FftR32Ctx<T>& ctx, int tid, const OsUnit<typename os_elt<T, CPLX>::type>& g,
                                            const cx<T>* __restrict__ H, OsStage& st, bool staged,
                                            const typename os_elt<T, CPLX>::type* __restrict__ next_u, const SG& state_geometry) {
    using E = typename os_elt<T, CPLX>::type;
    constexpr int NT = fft_r32::NT, Q = fft_r32::Q;
    cx<T> v[32];
    if (INTERIOR && staged) {
        // the span in natural order from st.head (head region, then the data buffer): lanes read consecutive words
        mbar_wait(st.bar, st.parity);
        st.parity ^= 1;
        const E* s = reinterpret_cast<const E*>(st.head);
#pragma unroll
        for (int m = 0; m < 32; ++m) {
            const int j = tid + m * Q;
            if constexpr (CPLX) v[m] = s[j];
            else v[m] = mkc<T>(s[j], s[j + g.L]);
        }
    } else {
#pragma unroll
        for (int m = 0; m < 32; ++m) v[m] = os_sample<T, CPLX, INTERIOR>(g, tid + m * Q);
    }
    fft_r32_first_bfly<T>(v);
    // every thread has read its samples (the staged ones lie in the data buffer's head) and the previous unit's last pass
    // is over
    __syncthreads();
    fft_r32_store_block<T>(ctx.sm, tid, v);
    __syncthreads();
    if (next_u != nullptr && tid == 0) {
        // the head region has been read: the next unit's head goes there now, its phase completes with the rest
        fence_proxy_async_shared();
        mbar_expect_tx_noarrive(st.bar, OS_STAGE_HEAD);
        tma_load_1d(st.head, next_u, OS_STAGE_HEAD, st.bar);
    }
#if !(DSP_PROBE & 16)
    fft_r32_middle<T, true>(ctx, tid);
#endif
    __syncthreads();
    // last forward pass, x H, swap, first pass of the second transform -- in registers
    {
        cx<T> u[2][16];
#pragma unroll
        for (int it = 0; it < 2; ++it) {
            fft_r32_last_load<T>(ctx, tid + it * NT, u[it]);
            fft_r32_last_bfly<T>(ctx, tid + it * NT, u[it]);
        }
#pragma unroll
#if DSP_PROBE & 4
        for (int m = 0; m < 32; ++m) v[m] = cswap(cmul(u[m & 1][m >> 1], mkc<T>(T(0.5), T(m))));
#else
        for (int m = 0; m < 32; ++m) v[m] = cswap(cmul(u[m & 1][m >> 1], ldg_cx<T>(H + tid + m * Q)));
#endif
    }
    fft_r32_first_bfly<T>(v);
    __syncthreads();                                   // every thread has read its last-pass inputs
    fft_r32_store_block<T>(ctx.sm, tid, v);
    __syncthreads();
#if !(DSP_PROBE & 16)
    fft_r32_middle<T, true>(ctx, tid);
#endif
    __syncthreads();
    os_sgeom_t<E, STATE, INTERIOR> sg{};
    if constexpr (STATE && !INTERIOR) sg = state_geometry();
    // Last pass: every thread reads the operands of both of its butterflies, then -- one barrier later, when nobody reads
    // the data buffer any more -- one thread issues the copy of the rest of the next unit's span into it, and the
    // butterflies and the global stores run while the copy is in flight.
    cx<T> w[2][16];
#pragma unroll
    for (int it = 0; it < 2; ++it) fft_r32_last_load<T>(ctx, tid + it * NT, w[it]);
    if (next_u != nullptr) {
        __syncthreads();
        if (tid == 0) {
            fence_proxy_async_shared();
            mbar_expect_tx(st.bar, st.bytes - OS_STAGE_HEAD);
            tma_load_1d(ctx.sm, reinterpret_cast<const unsigned char*>(next_u) + OS_STAGE_HEAD, st.bytes - OS_STAGE_HEAD, st.bar);
        }
    }
#pragma unroll
    for (int it = 0; it < 2; ++it) {
        const int t = tid + it * NT;
        fft_r32_last_bfly<T>(ctx, t, w[it]);
#pragma unroll
        for (int s = 0; s < 16; ++s) os_put<T, CPLX, INTERIOR, STATE>(g, sg, t + s * fft_r32::QL, w[it][s]);
    }
}

template <typename T, int N, bool CPLX, bool STATE>
__global__ void __launch_bounds__((os_threads<T, N, CPLX>::value), (os_threads<T, N, CPLX>::minblocks))
os_fused_kernel(const void* __restrict__ u_, int64_t u_begin, int64_t nu_local, int64_t u_col_stride,
                void* __restrict__ out_, int64_t out_begin, int64_t out_count, int64_t out_col_stride,
                int64_t zero_from, int nv, int64_t units_per_col, int64_t total_units, const cx<T>* __restrict__ gtl,
                const cx<T>* __restrict__ g16, const cx<T>* __restrict__ g256, const cx<T>* __restrict__ H,
                const OsState<typename os_elt<T, CPLX>::type, STATE> sa) {
    // gtl, g16, g256: the tables of fft_plan_traits<N>; staged kernels: gtl holds those of the 32 · 32 · 16 plan
    constexpr int NT = os_threads<T, N, CPLX>::value;
    constexpr int Q = fft_plan_traits<N>::Q;
    constexpr int ITERS = (Q + NT - 1) / NT;
    constexpr bool STAGED = os_threads<T, N, CPLX>::staged;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int HEAD = STAGED ? OS_STAGE_HEAD : 0;
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw + HEAD);
    using E = typename os_elt<T, CPLX>::type;
    const int tid = threadIdx.x;
    pdl_launch_dependents();
    auto make_ctx = [&]() {
        if constexpr (STAGED) return fft_r32_make_ctx<T>(sm, sm + fft_r32::PADDED_LEN, gtl, tid);
        else return fft_make_ctx<T, N, NT>(sm, g16, g256, gtl, tid);
    };
    const auto ctx = make_ctx();
    OsStage st;
    st.head = smem_raw;
    st.bar = reinterpret_cast<uint64_t*>(smem_raw + HEAD + (size_t)os_fft_elems<T, N, CPLX>() * sizeof(cx<T>));
    st.parity = 0;
    if constexpr (STAGED) {
        if (tid == 0) {
            mbar_init(st.bar, 1);
            mbar_fence_init();
        }
    }
    pdl_wait();                                        // tables staged; from here on data of preceding kernels is touched
    __syncthreads();                                   // (and the barrier initialised)
    const int L = N - nv + 1;
    const int span = CPLX ? N : N + L;                 // input samples / output range (+ nv - 1) of one unit
    st.bytes = (uint32_t)((span * sizeof(E) + 15) & ~(size_t)15);

    // geometry of unit gu; returns whether it is interior.  Recomputed where it is needed instead of carried in registers
    // across the unit
    const bool onecol = units_per_col >= total_units;
    auto geometry = [&](int64_t gu, OsUnit<E>& g) -> bool {
        const int64_t col = onecol ? 0 : gu / units_per_col;
        const int64_t unit = gu - col * units_per_col;
        const int64_t q = CPLX ? unit : 2 * unit;
        const int64_t s0 = out_begin + q * L - (nv - 1);          // global index of the sample in slot 0
        const int64_t i0 = s0 - u_begin;                          // its local index
        g.u = reinterpret_cast<const E*>(u_) + col * u_col_stride + i0;
        g.out = reinterpret_cast<E*>(out_) + col * out_col_stride + (s0 - out_begin);
        g.jlo = os_clamp(-i0);
        g.jhi = os_clamp(nu_local - i0);
        g.jend = os_clamp(out_begin + out_count - s0);
        g.jzero = os_clamp_diff(zero_from, s0);
        g.nvm1 = nv - 1;
        g.L = L;
        return g.jlo <= 0 && g.jhi >= span && g.jend >= span && g.jzero >= span;
    };
    // STATE: the state geometry of (edge) unit gu, in the same coordinates (OsUnitState)
    auto state_geometry = [&](int64_t gu) {
        OsUnitState<E> s{};
        if constexpr (STATE) {
            const int64_t col = onecol ? 0 : gu / units_per_col;
            const int64_t unit = gu - col * units_per_col;
            const int64_t s0 = out_begin + (CPLX ? unit : 2 * unit) * L - (nv - 1);
            s.si_in = sa.si_in + col * (nv - 1) + s0;
            s.si_out = sa.si_out + col * (nv - 1) + (s0 - sa.nx);
            s.jsi = sa.si_in ? os_clamp((nv - 1) - s0) : -(1 << 30);
            s.jnx = os_clamp(sa.nx - s0);
        }
        return s;
    };
    // pull the input range of unit gn into L2 (16-byte aligned sub-range, clipped to the stored signal)
    auto l2_prefetch = [&](int64_t gn) {
        if (tid == 0 && gn < total_units) {
            const int64_t coln = onecol ? 0 : gn / units_per_col;
            const int64_t qn = (CPLX ? 1 : 2) * (gn - coln * units_per_col);
            int64_t lo = out_begin + qn * L - (nv - 1) - u_begin;
            int64_t hi = lo + span;
            if (lo < 0) lo = 0;
            if (hi > nu_local) hi = nu_local;
            const uintptr_t a0 = ((uintptr_t)(reinterpret_cast<const E*>(u_) + coln * u_col_stride + lo) + 15) & ~(uintptr_t)15;
            const uintptr_t a1 = (uintptr_t)(reinterpret_cast<const E*>(u_) + coln * u_col_stride + hi) & ~(uintptr_t)15;
            if (hi > lo && a1 > a0) tma_prefetch_l2(reinterpret_cast<const void*>(a0), (uint32_t)(a1 - a0));
        }
    };
    // slot 0 of unit gn if its input is to be staged in shared memory, else null: staged kernels only, interior units
    // (no predicates on the samples), 16-byte aligned source (TMA), and the copy's round-up to 16 bytes still inside the
    // stored signal.  Every other unit loads its samples from global memory in its first pass.
    auto stage_src = [&](int64_t gn) -> const E* {
        if (!STAGED || gn >= total_units || (DSP_PROBE & 2)) return nullptr;   // (the input-load probe stages nothing)
        OsUnit<E> gl;
        if (!geometry(gn, gl)) return nullptr;
        if ((int64_t)gl.jhi * (int64_t)sizeof(E) < (int64_t)st.bytes || ((uintptr_t)gl.u & 15) != 0) return nullptr;
        return gl.u;
    };
    bool staged = false;
    if constexpr (STAGED) {
        const E* src = stage_src(blockIdx.x);
        staged = src != nullptr;
        if (staged && tid == 0) {
            mbar_expect_tx(st.bar, st.bytes);
            tma_load_1d(st.head, src, OS_STAGE_HEAD, st.bar);
            tma_load_1d(ctx.sm, reinterpret_cast<const unsigned char*>(src) + OS_STAGE_HEAD, st.bytes - OS_STAGE_HEAD, st.bar);
        }
    }

    for (int64_t gu = blockIdx.x; gu < total_units; gu += gridDim.x) {
        // while this unit computes, the next one is pulled into L2, so that its TMA copies read L2 (without this prefetch
        // the staged complex 16384-point conv, whole span copied in the last pass, took 0.664 .. 0.666 ms instead of
        // 0.655 .. 0.659 ms: H100 SXM 80 GB at 400 W)
        l2_prefetch(gu + (int64_t)gridDim.x);
        OsUnit<E> g;
        const bool interior = geometry(gu, g);
        const E* next_u = stage_src(gu + gridDim.x);
        auto sgeom = [&]() { return state_geometry(gu); };
        if constexpr (STAGED) {
            if (interior) os_unit_r32<T, CPLX, true, STATE>(ctx, tid, g, H, st, staged, next_u, sgeom);
            else os_unit_r32<T, CPLX, false, STATE>(ctx, tid, g, H, st, staged, next_u, sgeom);
        } else {
            if (interior) os_unit<T, N, CPLX, NT, true, ITERS, STATE>(ctx, tid, g, H, sgeom);
            else os_unit<T, N, CPLX, NT, false, ITERS, STATE>(ctx, tid, g, H, sgeom);
        }
        staged = next_u != nullptr;
    }
}

// H in natural order: forward transform of the zero-padded taps, scaled by 1/N.
template <typename T, int N, bool CPLX>
__global__ void __launch_bounds__(fft_threads<N>::value, fft_minblocks<T, N>::value)
os_filter_kernel(const void* __restrict__ v_, int nv, const cx<T>* __restrict__ gtl, const cx<T>* __restrict__ g16,
                 const cx<T>* __restrict__ g256, cx<T>* __restrict__ H) {
    constexpr int NT = fft_threads<N>::value;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    using E = typename os_elt<T, CPLX>::type;
    const E* v = reinterpret_cast<const E*>(v_);
    const FftCtx<T> ctx = fft_make_ctx<T, N, NT>(sm, g16, g256, gtl, threadIdx.x);
    __syncthreads();
    const T scale = T(1) / T(N);
    auto ld0 = [&](int j, int, int) -> cx<T> {
        if (j >= nv) return mkc<T>(T(0), T(0));
        if constexpr (CPLX) return v[j]; else return mkc<T>(v[j], T(0));
    };
    auto stl = [&](int k, int, int, cx<T> x) { H[k] = cscale(x, scale); };
    fft_forward<T, N, NT>(ctx, threadIdx.x, ld0, stl);
}

// ---------------------------------------------------------------------------------------------- generic kernels
template <typename T, bool CPLX>
__global__ void os_gather_kernel(const void* __restrict__ u_, int64_t u_begin, int64_t nu_local, int64_t m_first,
                                 int64_t L, int64_t nv, int64_t nfft, int64_t nblk, void* __restrict__ td_) {
    using E = typename os_elt<T, CPLX>::type;
    const E* u = reinterpret_cast<const E*>(u_);
    E* td = reinterpret_cast<E*>(td_);
    const int64_t total = nblk * nfft;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = i / nfft, j = i - b * nfft;
        const int64_t src = m_first + b * L - (nv - 1) + j - u_begin;
        E v;
        if constexpr (CPLX) v = mkc<T>(T(0), T(0)); else v = T(0);
        if (src >= 0 && src < nu_local) v = u[src];
        td[i] = v;
    }
}

template <typename T>
__global__ void os_cmul_kernel(cx<T>* __restrict__ X, const cx<T>* __restrict__ H, int64_t nbins, int64_t nblk) {
    const int64_t total = nblk * nbins;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
        X[i] = cmul(X[i], H[i % nbins]);
}

// ---------------------------------------------------------------------------------------------- hilbert
// hilbert(x), src/util.jl:31-75: X = rfft(x) written into the first n/2+1 bins of a zeroed length-n complex buffer,
// bins 2 .. n/2 + isodd(n) (1-based) doubled, inverse complex FFT with the 1/n normalisation.
template <typename T>
__global__ void hilbert_weight_kernel(cx<T>* __restrict__ X, int64_t n, int64_t ncols, T scale) {
    const int64_t total = n * ncols;
    const int64_t last2 = (n + 1) / 2 - 1;                    // last doubled bin (0-based)
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t k = i % n;
        if (k > n / 2) { X[i] = mkc<T>(T(0), T(0)); continue; }      // never written by the real transform
        const T w = (k >= 1 && k <= last2) ? T(2) * scale : scale;   // DC and (n even) Nyquist keep weight 1
        X[i] = cscale(X[i], w);
    }
}

// ---------------------------------------------------------------------------------------------- N-D conv (rank <= 3)
// Column-major arrays, dim 1 fastest (Julia layout); ranks below 3 carry trailing sizes of 1.
struct Dims3 { int64_t n[3]; };

// dst (size d) = src (size s) zero-padded / cropped at the origin: _zeropad!, src/dspbase.jl:187-256, and the copyto! of
// the valid region, :624-627 / :640-643
template <typename E>
__global__ void nd_copy_kernel(const E* __restrict__ src, Dims3 s, E* __restrict__ dst, Dims3 d, E zero) {
    const int64_t total = d.n[0] * d.n[1] * d.n[2];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i0 = i % d.n[0], i1 = (i / d.n[0]) % d.n[1], i2 = i / (d.n[0] * d.n[1]);
        dst[i] = (i0 < s.n[0] && i1 < s.n[1] && i2 < s.n[2]) ? src[i0 + s.n[0] * (i1 + s.n[1] * i2)] : zero;
    }
}

// _conv_td!, src/dspbase.jl:646-660, N-D: out[k] = sum of u[m] * v[n] over m + n = k, one output per thread.  The reference
// loops `for m in CartesianIndices(u), n in CartesianIndices(v)` when size(u,1) <= size(v,1), else with n outer: every
// output sums its products in the column-major order of the outer array's index (dim 1 fastest), each step
// muladd(u[m], v[n], acc).  The walk below is over that array (w), the other one (o) read at k - j.  RANK1: rank 1, no index
// decomposition (its 64-bit divisions took a 2048 x 31 Float32 call from 0.035 to 0.040 ms: H100 80GB HBM3, 700 W).
template <typename T, bool CPLX, bool RANK1>
__global__ void conv_direct_nd_kernel(const void* __restrict__ u_, Dims3 su, const void* __restrict__ v_, Dims3 sv,
                                      void* __restrict__ out_) {
    using E = typename os_elt<T, CPLX>::type;
    const bool walk_u = su.n[0] <= sv.n[0];
    const E* w = reinterpret_cast<const E*>(walk_u ? u_ : v_);
    const E* o = reinterpret_cast<const E*>(walk_u ? v_ : u_);
    const Dims3 sw = walk_u ? su : sv, so = walk_u ? sv : su;
    E* out = reinterpret_cast<E*>(out_);
    const int64_t o0 = su.n[0] + sv.n[0] - 1, o1 = su.n[1] + sv.n[1] - 1, o2 = su.n[2] + sv.n[2] - 1;
    const int64_t total = o0 * o1 * o2;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t k0 = RANK1 ? i : i % o0, k1 = RANK1 ? 0 : (i / o0) % o1, k2 = RANK1 ? 0 : i / (o0 * o1);
        T ar = T(0), ai = T(0);
        for (int64_t m2 = max(k2 - (so.n[2] - 1), (int64_t)0); m2 <= min(k2, sw.n[2] - 1); ++m2)
            for (int64_t m1 = max(k1 - (so.n[1] - 1), (int64_t)0); m1 <= min(k1, sw.n[1] - 1); ++m1)
                for (int64_t m0 = max(k0 - (so.n[0] - 1), (int64_t)0); m0 <= min(k0, sw.n[0] - 1); ++m0) {
                    const E p = w[m0 + sw.n[0] * (m1 + sw.n[1] * m2)];
                    const E q = o[(k0 - m0) + so.n[0] * ((k1 - m1) + so.n[1] * (k2 - m2))];
                    const E a = walk_u ? p : q, b = walk_u ? q : p;     // a = u[m], b = v[n]: muladd(a, b, acc)
                    if constexpr (CPLX) {
                        ar = fma(a.x, b.x, fma(-a.y, b.y, ar));
                        ai = fma(a.x, b.y, fma(a.y, b.x, ai));
                    } else {
                        ar = fma(a, b, ar);
                    }
                }
        if constexpr (CPLX) out[i] = mkc<T>(ar, ai); else out[i] = ar;
    }
}

// N-D overlap-save blocking: unsafe_conv_kern_os! with its perimeter blocks, src/dspbase.jl:371-609.  Block b = (b0, b1, b2)
// of the nb grid owns the outputs L .* b .. L .* (b + 1) - 1 (L = save_blocksize, :505); its time-domain buffer holds nf
// samples per dimension starting sv - 1 before the block's first output and is zero where that lies outside u (the
// reference's pad_before / pad_after, :449-463; centre blocks, :583-606, are the case without padding).  Blocks are
// transformed `nblk` at a time by ONE batched N-D cuFFT plan; blocks past the end of the grid (last batch) are zeros.
struct OsNd { int64_t su[3], sv[3], so[3], nf[3], L[3], nb[3]; };

template <typename E>
__global__ void nd_os_gather_kernel(const E* __restrict__ u, OsNd g, int64_t blk0, int64_t nblk, E* __restrict__ td, E zero) {
    const int64_t per = g.nf[0] * g.nf[1] * g.nf[2], total = per * nblk, nblocks = g.nb[0] * g.nb[1] * g.nb[2];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = blk0 + i / per, r = i % per;
        E val = zero;
        if (b < nblocks) {
            const int64_t i0 = r % g.nf[0], i1 = (r / g.nf[0]) % g.nf[1], i2 = r / (g.nf[0] * g.nf[1]);
            const int64_t b0 = b % g.nb[0], b1 = (b / g.nb[0]) % g.nb[1], b2 = b / (g.nb[0] * g.nb[1]);
            const int64_t s0 = g.L[0] * b0 - (g.sv[0] - 1) + i0, s1 = g.L[1] * b1 - (g.sv[1] - 1) + i1,
                          s2 = g.L[2] * b2 - (g.sv[2] - 1) + i2;
            if (s0 >= 0 && s0 < g.su[0] && s1 >= 0 && s1 < g.su[1] && s2 >= 0 && s2 < g.su[2])
                val = u[s0 + g.su[0] * (s1 + g.su[1] * s2)];
        }
        td[i] = val;
    }
}

// the valid region sv : nf of every block (:603-606, cropped at the end of the output, :468-482) -> out
template <typename E>
__global__ void nd_os_scatter_kernel(const E* __restrict__ td, OsNd g, int64_t blk0, int64_t nblk, E* __restrict__ out) {
    const int64_t per = g.L[0] * g.L[1] * g.L[2], total = per * nblk, nblocks = g.nb[0] * g.nb[1] * g.nb[2];
    const int64_t nfp = g.nf[0] * g.nf[1] * g.nf[2];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t lb = i / per, b = blk0 + lb, r = i % per;
        if (b >= nblocks) continue;
        const int64_t j0 = r % g.L[0], j1 = (r / g.L[0]) % g.L[1], j2 = r / (g.L[0] * g.L[1]);
        const int64_t b0 = b % g.nb[0], b1 = (b / g.nb[0]) % g.nb[1], b2 = b / (g.nb[0] * g.nb[1]);
        const int64_t o0 = g.L[0] * b0 + j0, o1 = g.L[1] * b1 + j1, o2 = g.L[2] * b2 + j2;
        if (o0 < g.so[0] && o1 < g.so[1] && o2 < g.so[2])
            out[o0 + g.so[0] * (o1 + g.so[1] * o2)] =
                td[lb * nfp + (j0 + g.sv[0] - 1) + g.nf[0] * ((j1 + g.sv[1] - 1) + g.nf[1] * (j2 + g.sv[2] - 1))];
    }
}

// STATE: sa holds one column's state (OsState), and m is that column's output index (out_begin == 0)
template <typename T, bool CPLX, bool STATE>
__global__ void os_scatter_kernel(const void* __restrict__ td_, int64_t m_first, int64_t L, int64_t nv, int64_t nfft,
                                  int64_t nblk, void* __restrict__ out_, int64_t out_begin, int64_t out_end,
                                  int64_t zero_from, const OsState<typename os_elt<T, CPLX>::type, STATE> sa) {
    using E = typename os_elt<T, CPLX>::type;
    const E* td = reinterpret_cast<const E*>(td_);
    E* out = reinterpret_cast<E*>(out_);
    const int64_t total = nblk * L;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = i / L, j = i - b * L;
        const int64_t m = m_first + b * L + j;
        if (m < out_end) {
            E v = td[b * nfft + (nv - 1) + j];
            if (m >= zero_from) { if constexpr (CPLX) v = mkc<T>(T(0), T(0)); else v = T(0); }
            if constexpr (STATE) {
                if (sa.si_in && m < nv - 1) v = v + sa.si_in[m];
                if (m >= sa.nx) {
                    sa.si_out[m - sa.nx] = v;
                    continue;
                }
            }
            out[m - out_begin] = v;
        }
    }
}

template <typename T, bool CPLX>
__global__ void pad_copy_kernel(const void* __restrict__ src_, int64_t n, void* __restrict__ dst_, int64_t nfft, T scale) {
    using E = typename os_elt<T, CPLX>::type;
    const E* src = reinterpret_cast<const E*>(src_);
    E* dst = reinterpret_cast<E*>(dst_);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nfft; i += (int64_t)gridDim.x * blockDim.x) {
        E v;
        if constexpr (CPLX) v = mkc<T>(T(0), T(0)); else v = T(0);
        if (i < n) {
            v = src[i];
            if constexpr (CPLX) v = cscale(v, scale); else v = v * scale;
        }
        dst[i] = v;
    }
}

template <typename T>
__global__ void scale_cplx_kernel(cx<T>* __restrict__ X, int64_t n, T scale) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        X[i] = cscale(X[i], scale);
}

// ---------------------------------------------------------------------------------------------- dispatch
#define DSP_OS_SIZES(X) X(32) X(64) X(128) X(256) X(512) X(1024) X(2048) X(4096) X(8192) X(16384)

static bool os_fused_ok(int64_t nfft, int64_t nv, bool f64) {
    if (nfft < 32 || (nfft & (nfft - 1))) return false;
    if (nfft > (f64 ? 8192 : 16384)) return false;
    return nfft >= nv;
}

template <typename K> static int set_smem(K kernel, size_t bytes) {
    if (bytes > 48 * 1024) DSP_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    return DSPB200_OK;
}

struct OsRange {
    const void* u; int64_t u_begin, nu_local, u_col_stride;
    void* out; int64_t out_begin, out_count, out_col_stride;
    int64_t zero_from, ncols;
};

// state of a stateful call (OsState, untyped): si_in / si_out hold nv - 1 elements per column
struct OsStateArgs {
    const void* si_in;
    void* si_out;
    int64_t nx;
};
// The stateful entry plans with nfft = 0 (auto_nfft), so it reaches the fused sizes from 1024 up only.
constexpr int OS_STATE_MIN_NFFT = 1024;
// the kernel argument for the state entries from element `off` on (a column's state in the generic path)
template <typename E, bool STATE> static OsState<E, STATE> os_state_arg(const OsStateArgs& s, int64_t off) {
    OsState<E, STATE> r{};
    if constexpr (STATE)
        r = {s.si_in ? reinterpret_cast<const E*>(s.si_in) + off : nullptr, s.si_out ? reinterpret_cast<E*>(s.si_out) + off : nullptr, s.nx};
    return r;
}

template <typename T, int N, bool CPLX, bool STATE>
static int launch_os_fused(OsPlanImpl* p, const OsRange& a, const OsStateArgs& s, cudaStream_t st) {
    using E = typename os_elt<T, CPLX>::type;
    constexpr int NT = os_threads<T, N, CPLX>::value;
    const size_t smem = os_smem_bytes<T, N, CPLX>();
    auto kern = os_fused_kernel<T, N, CPLX, STATE>;
    const OsState<E, STATE> sa = os_state_arg<E, STATE>(s, 0);
    const int64_t nblk = cdiv(a.out_count, p->L);
    const int64_t upc = CPLX ? nblk : (nblk + 1) / 2;
    const int64_t units = upc * a.ncols;
    if (units < 1) return DSPB200_OK;
    // persistent grid: one resident wave (CTAs per SM from the occupancy calculator: shared memory and register cap)
    int& per_sm = STATE ? p->fused_state_per_sm : p->fused_per_sm;
    if (per_sm < 1) {
        DSP_TRY(set_smem(kern, smem));
        int per = 1;
        DSP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, kern, NT, smem));
        per_sm = per < 1 ? 1 : per;
    }
    const int64_t cap = (int64_t)p->sm_count * per_sm;
    const int64_t blocks = units < cap ? units : cap;
    DSP_CUDA(launch_pdl(kern, (unsigned)blocks, NT, smem, st, a.u, a.u_begin, a.nu_local, a.u_col_stride, a.out, a.out_begin,
                        a.out_count, a.out_col_stride, a.zero_from, (int)p->nv, upc, units,
                        reinterpret_cast<const cx<T>*>(os_threads<T, N, CPLX>::staged ? p->d_r32 : p->d_tw),
                        reinterpret_cast<const cx<T>*>(p->d_t16), reinterpret_cast<const cx<T>*>(p->d_t256),
                        reinterpret_cast<const cx<T>*>(p->d_H), sa));
    DSP_LAUNCH_OK();
    return DSPB200_OK;
}

template <typename T, bool STATE> static int os_fused_dispatch(OsPlanImpl* p, const OsRange& a, const OsStateArgs& s, cudaStream_t st) {
    switch (p->nfft) {
#define X(NN)                                                                                                       \
    case NN:                                                                                                        \
        if constexpr ((sizeof(T) == 8 && NN > 8192) || (STATE && NN < OS_STATE_MIN_NFFT)) break;                    \
        else return p->cplx ? launch_os_fused<T, NN, true, STATE>(p, a, s, st) : launch_os_fused<T, NN, false, STATE>(p, a, s, st);
        DSP_OS_SIZES(X)
#undef X
    }
    set_error("no fused %soverlap-save kernel for nfft=%lld", STATE ? "stateful " : "", (long long)p->nfft);
    return DSPB200_EUNSUPPORTED;
}

template <typename T, int N, bool CPLX>
static int launch_os_filter(OsPlanImpl* p, const void* d_v) {
    constexpr int NT = fft_threads<N>::value;
    const size_t smem = (size_t)fft_smem_elems<T, N>() * sizeof(cx<T>);
    auto kern = os_filter_kernel<T, N, CPLX>;
    DSP_TRY(set_smem(kern, smem));
    kern<<<1, NT, smem, 0>>>(d_v, (int)p->nv, reinterpret_cast<const cx<T>*>(p->d_tw), reinterpret_cast<const cx<T>*>(p->d_t16),
                             reinterpret_cast<const cx<T>*>(p->d_t256), reinterpret_cast<cx<T>*>(p->d_H));
    DSP_LAUNCH_OK();
    DSP_CUDA(cudaStreamSynchronize(0));
    return DSPB200_OK;
}

template <typename T> static int os_filter_dispatch(OsPlanImpl* p, const void* d_v) {
    switch (p->nfft) {
#define X(NN)                                                                                   \
    case NN:                                                                                    \
        if constexpr (sizeof(T) == 8 && NN > 8192) break;                                       \
        else return p->cplx ? launch_os_filter<T, NN, true>(p, d_v) : launch_os_filter<T, NN, false>(p, d_v);
        DSP_OS_SIZES(X)
#undef X
    }
    return DSPB200_EUNSUPPORTED;
}

static int grid_for(int64_t total, int threads) {
    int64_t g = cdiv(total, threads);
    const int64_t cap = (int64_t)device_sm_count() * 64;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

template <typename T, bool STATE> static int os_generic_run(OsPlanImpl* p, const OsRange& a, const OsStateArgs& s, cudaStream_t st) {
    const int threads = 256;
    for (int64_t c = 0; c < a.ncols; ++c) {
        const char* ucol = (const char*)a.u + (size_t)(c * a.u_col_stride) * dtype_size(p->dtype);
        char* ocol = (char*)a.out + (size_t)(c * a.out_col_stride) * dtype_size(p->dtype);
        const int64_t nblk_total = cdiv(a.out_count, p->L);
        for (int64_t b0 = 0; b0 < nblk_total; b0 += p->batch) {
            const int64_t nblk = nblk_total - b0 < p->batch ? nblk_total - b0 : p->batch;
            const int64_t m_first = a.out_begin + b0 * p->L;
            // gather all `batch` rows (rows >= nblk read past the range and are simply ignored by scatter)
            if (p->cplx) os_gather_kernel<T, true><<<grid_for(p->batch * p->nfft, threads), threads, 0, st>>>(ucol, a.u_begin, a.nu_local, m_first, p->L, p->nv, p->nfft, p->batch, p->td.p);
            else os_gather_kernel<T, false><<<grid_for(p->batch * p->nfft, threads), threads, 0, st>>>(ucol, a.u_begin, a.nu_local, m_first, p->L, p->nv, p->nfft, p->batch, p->td.p);
            DSP_LAUNCH_OK();
            DSP_TRY(fft_exec(p->fwd, p->cplx, p->f64, CUFFT_FORWARD, p->td.p, p->fd.p, st));
            os_cmul_kernel<T><<<grid_for(p->batch * p->nbins, threads), threads, 0, st>>>(reinterpret_cast<cx<T>*>(p->fd.p), reinterpret_cast<const cx<T>*>(p->d_H), p->nbins, p->batch);
            DSP_LAUNCH_OK();
            DSP_TRY(fft_exec(p->inv, p->cplx, p->f64, CUFFT_INVERSE, p->fd.p, p->td.p, st));
            if (p->cplx) os_scatter_kernel<T, true, STATE><<<grid_for(nblk * p->L, threads), threads, 0, st>>>(p->td.p, m_first, p->L, p->nv, p->nfft, nblk, ocol, a.out_begin, a.out_begin + a.out_count, a.zero_from, os_state_arg<cx<T>, STATE>(s, c * (p->nv - 1)));
            else os_scatter_kernel<T, false, STATE><<<grid_for(nblk * p->L, threads), threads, 0, st>>>(p->td.p, m_first, p->L, p->nv, p->nfft, nblk, ocol, a.out_begin, a.out_begin + a.out_count, a.zero_from, os_state_arg<T, STATE>(s, c * (p->nv - 1)));
            DSP_LAUNCH_OK();
        }
    }
    return DSPB200_OK;
}

template <bool STATE> static int os_run(OsPlanImpl* p, const OsRange& a, const OsStateArgs& s, cudaStream_t st) {
    if (a.out_count <= 0 || a.ncols <= 0) return DSPB200_OK;
    if (p->fused) return p->f64 ? os_fused_dispatch<double, STATE>(p, a, s, st) : os_fused_dispatch<float, STATE>(p, a, s, st);
    return p->f64 ? os_generic_run<double, STATE>(p, a, s, st) : os_generic_run<float, STATE>(p, a, s, st);
}
static int os_run(OsPlanImpl* p, const OsRange& a, cudaStream_t st) { return os_run<false>(p, a, OsStateArgs{}, st); }

static int64_t auto_nfft(int64_t nv, bool f64) {
    const int64_t nmax = f64 ? 8192 : 16384;
    int64_t best = 0;
    double best_cost = 0;
    for (int64_t n = 1024; n <= nmax; n <<= 1) {
        if (n - nv + 1 < n / 2) continue;   // at least half of every block must be new output
        const double cost = (double)n * (log2((double)n) + 2.0) / (double)(n - nv + 1);
        if (best == 0 || cost < best_cost) { best = n; best_cost = cost; }
    }
    if (best) return best;
    int64_t n = 4096;
    while (n < 4 * nv) n <<= 1;   // generic path: 75 % of each block is new output
    return n;
}

static int ensure_streams(OsPlanImpl* p) { return p->pipe.ensure(p->device); }

}  // namespace dspb200

using namespace dspb200;

struct dspb200_os_plan {
    OsPlanImpl impl;
};

// conv(u, v) for arrays of rank 1 to 3 on device pointers: _conv_td! (mode 0), _conv_kern_fft! (mode 1: one N-D FFT pair of
// size nffts) or unsafe_conv_kern_os! (mode 2: blocks of nffts, batched).  Plans and scratch come from the cache / arena of
// runtime.cu; the caller holds the ConvenienceLock and synchronises the stream before the arena is reused.
enum { ND_DIRECT = 0, ND_FFT = 1, ND_OS = 2 };
static size_t g_nd_os_budget = (size_t)1 << 30;          // bytes of block buffers per batch (dspb200_conv_nd_os_* entry points)

template <typename T, bool CPLX>
static int conv_nd_dev(int mode, int rank, const int64_t* usize, const void* d_u, const int64_t* vsize, const void* d_v,
                       const int64_t* nffts, void* d_out, cudaStream_t st) {
    using E = typename os_elt<T, CPLX>::type;
    Dims3 su{{1, 1, 1}}, sv{{1, 1, 1}}, so{{1, 1, 1}}, sf{{1, 1, 1}};
    for (int d = 0; d < rank; ++d) {
        su.n[d] = usize[d]; sv.n[d] = vsize[d]; so.n[d] = usize[d] + vsize[d] - 1;
        if (mode != ND_DIRECT) sf.n[d] = nffts[d];
    }
    const int64_t no = so.n[0] * so.n[1] * so.n[2];
    const int threads = 256;
    if (mode == ND_DIRECT) {
        auto kern = rank == 1 ? conv_direct_nd_kernel<T, CPLX, true> : conv_direct_nd_kernel<T, CPLX, false>;
        kern<<<grid_for(no, 128), 128, 0, st>>>(d_u, su, d_v, sv, d_out);
        DSP_LAUNCH_OK();
        return DSPB200_OK;
    }
    DevBuf &tu = scratch_buf(3), &fu = scratch_buf(4), &fv = scratch_buf(5);
    const int64_t nf = sf.n[0] * sf.n[1] * sf.n[2];
    Dims3 sb = sf;                                           // spectrum dims: first (fastest) dim halved for real input
    if (!CPLX) sb.n[0] = sf.n[0] / 2 + 1;
    const int64_t nb = sb.n[0] * sb.n[1] * sb.n[2];
    long long nn[3];                                         // cuFFT is row-major: slowest dimension first
    for (int d = 0; d < rank; ++d) nn[d] = (long long)sf.n[rank - 1 - d];
    const bool f64 = sizeof(T) == 8;
    const int tf = fft_type(CPLX, f64, CUFFT_FORWARD), ti = fft_type(CPLX, f64, CUFFT_INVERSE);
    E zero;
    if constexpr (CPLX) zero = mkc<T>(T(0), T(0)); else zero = T(0);
    int h1f = 0;
    DSP_TRY(plan_cache_get(&h1f, rank, nn, false, 0, 0, tf, 1));
    if (mode == ND_FFT) {
        int h1i = h1f;
        if (!CPLX) DSP_TRY(plan_cache_get(&h1i, rank, nn, false, 0, 0, ti, 1));
        DSP_TRY(tu.reserve((size_t)nf * sizeof(E)));
        DSP_TRY(fu.reserve((size_t)nb * sizeof(cx<T>))); DSP_TRY(fv.reserve((size_t)nb * sizeof(cx<T>)));
        nd_copy_kernel<E><<<grid_for(nf, threads), threads, 0, st>>>((const E*)d_u, su, (E*)tu.p, sf, zero);
        DSP_LAUNCH_OK();
        DSP_TRY(fft_exec((cufftHandle)h1f, CPLX, f64, CUFFT_FORWARD, tu.p, fu.p, st));
        nd_copy_kernel<E><<<grid_for(nf, threads), threads, 0, st>>>((const E*)d_v, sv, (E*)tu.p, sf, zero);
        DSP_LAUNCH_OK();
        DSP_TRY(fft_exec((cufftHandle)h1f, CPLX, f64, CUFFT_FORWARD, tu.p, fv.p, st));
        scale_cplx_kernel<T><<<grid_for(nb, threads), threads, 0, st>>>((cx<T>*)fv.p, nb, T(1) / (T)nf);
        os_cmul_kernel<T><<<grid_for(nb, threads), threads, 0, st>>>((cx<T>*)fu.p, (const cx<T>*)fv.p, nb, 1);
        count_launch(2);
        DSP_TRY(fft_exec((cufftHandle)h1i, CPLX, f64, CUFFT_INVERSE, fu.p, tu.p, st));
        nd_copy_kernel<E><<<grid_for(no, threads), threads, 0, st>>>((const E*)tu.p, sf, (E*)d_out, so, zero);
        DSP_LAUNCH_OK();
        return DSPB200_OK;
    }
    // ND_OS
    OsNd g;
    int64_t nblocks = 1, Lp = 1;
    for (int d = 0; d < 3; ++d) {
        g.su[d] = su.n[d]; g.sv[d] = sv.n[d]; g.so[d] = so.n[d]; g.nf[d] = sf.n[d];
        const int64_t ideal = sf.n[d] - sv.n[d] + 1;                           // :500
        g.L[d] = ideal < so.n[d] ? ideal : so.n[d];                             // save_blocksize = ideal - sout_deficit, :503-505
        g.nb[d] = cdiv(so.n[d], g.L[d]);                                        // :506
        nblocks *= g.nb[d]; Lp *= g.L[d];
    }
    const size_t per_block = (size_t)nf * sizeof(E) + (size_t)nb * sizeof(cx<T>);
    int64_t batch = (int64_t)(g_nd_os_budget / per_block);
    if (batch < 1) batch = 1;
    if (batch > nblocks) batch = nblocks;
    int hbf = h1f, hbi = 0;
    if (batch > 1) DSP_TRY(plan_cache_get(&hbf, rank, nn, false, 0, 0, tf, batch));
    if (CPLX) hbi = hbf; else DSP_TRY(plan_cache_get(&hbi, rank, nn, false, 0, 0, ti, batch));
    DSP_TRY(tu.reserve((size_t)nf * batch * sizeof(E)));
    DSP_TRY(fu.reserve((size_t)nb * batch * sizeof(cx<T>))); DSP_TRY(fv.reserve((size_t)nb * sizeof(cx<T>)));
    // filter spectrum, scaled once by 1/prod(nffts) (:513-516)
    nd_copy_kernel<E><<<grid_for(nf, threads), threads, 0, st>>>((const E*)d_v, sv, (E*)tu.p, sf, zero);
    DSP_LAUNCH_OK();
    DSP_TRY(fft_exec((cufftHandle)h1f, CPLX, f64, CUFFT_FORWARD, tu.p, fv.p, st));
    scale_cplx_kernel<T><<<grid_for(nb, threads), threads, 0, st>>>((cx<T>*)fv.p, nb, T(1) / (T)nf);
    DSP_LAUNCH_OK();
    for (int64_t b0 = 0; b0 < nblocks; b0 += batch) {
        nd_os_gather_kernel<E><<<grid_for(nf * batch, threads), threads, 0, st>>>((const E*)d_u, g, b0, batch, (E*)tu.p, zero);
        DSP_LAUNCH_OK();
        DSP_TRY(fft_exec((cufftHandle)hbf, CPLX, f64, CUFFT_FORWARD, tu.p, fu.p, st));
        os_cmul_kernel<T><<<grid_for(nb * batch, threads), threads, 0, st>>>((cx<T>*)fu.p, (const cx<T>*)fv.p, nb, batch);
        DSP_LAUNCH_OK();
        DSP_TRY(fft_exec((cufftHandle)hbi, CPLX, f64, CUFFT_INVERSE, fu.p, tu.p, st));
        nd_os_scatter_kernel<E><<<grid_for(Lp * batch, threads), threads, 0, st>>>((const E*)tu.p, g, b0, batch, (E*)d_out);
        DSP_LAUNCH_OK();
    }
    return DSPB200_OK;
}

static int conv_nd_check(int dtype, int mode, int rank, const int64_t* usize, const void* u, const int64_t* vsize, const void* v,
                         const int64_t* nffts, void* out) {
    DSP_REQUIRE(dtype_valid(dtype), "invalid dtype %d", dtype);
    DSP_REQUIRE(rank >= 1 && rank <= 3, "rank must be 1, 2 or 3");
    DSP_REQUIRE(usize && vsize && u && v && out, "NULL argument");
    DSP_REQUIRE(mode == ND_DIRECT || nffts, "nffts is NULL");
    for (int d = 0; d < rank; ++d) {
        DSP_REQUIRE(usize[d] >= 1 && vsize[d] >= 1, "empty input");
        if (mode == ND_FFT)
            DSP_REQUIRE(nffts[d] >= usize[d] + vsize[d] - 1 && nffts[d] < (int64_t(1) << 31), "nffts must cover the full output");
        if (mode == ND_OS)
            DSP_REQUIRE(nffts[d] >= vsize[d] && nffts[d] < (int64_t(1) << 31), "overlap-save nffts must be at least size(v)");
    }
    return DSPB200_OK;
}

static int conv_nd_dispatch(int dtype, int mode, int rank, const int64_t* usize, const void* d_u, const int64_t* vsize,
                            const void* d_v, const int64_t* nffts, void* d_out, cudaStream_t st) {
    switch (dtype) {
        case DSPB200_F32: return conv_nd_dev<float, false>(mode, rank, usize, d_u, vsize, d_v, nffts, d_out, st);
        case DSPB200_F64: return conv_nd_dev<double, false>(mode, rank, usize, d_u, vsize, d_v, nffts, d_out, st);
        case DSPB200_C32: return conv_nd_dev<float, true>(mode, rank, usize, d_u, vsize, d_v, nffts, d_out, st);
        default: return conv_nd_dev<double, true>(mode, rank, usize, d_u, vsize, d_v, nffts, d_out, st);
    }
}

// device-pointer form: returns after the work on `stream` has completed (the cached plans and the arena are shared)
static int conv_nd_run_dev(int dtype, int mode, int rank, const int64_t* usize, const void* d_u, const int64_t* vsize, const void* d_v,
                           const int64_t* nffts, void* d_out, cudaStream_t st) {
    return convenience_call(st, [&](cudaStream_t s) {
        return conv_nd_dispatch(dtype, mode, rank, usize, d_u, vsize, d_v, nffts, d_out, s);
    });
}

// host-pointer form
static int conv_nd_run_host(int dtype, int mode, int rank, const int64_t* usize, const void* u, const int64_t* vsize, const void* v,
                            const int64_t* nffts, void* out) {
    int64_t nu = 1, nv = 1, no = 1;
    for (int d = 0; d < rank; ++d) { nu *= usize[d]; nv *= vsize[d]; no *= usize[d] + vsize[d] - 1; }
    const size_t esz = dtype_size(dtype);
    DevBuf &du = scratch_buf(0), &dv = scratch_buf(1), &dout = scratch_buf(2);
    return convenience_call({{u, (size_t)nu * esz, &du}, {v, (size_t)nv * esz, &dv}}, {{out, (size_t)no * esz, &dout}}, [&](cudaStream_t s) {
        return conv_nd_dispatch(dtype, mode, rank, usize, du.p, vsize, dv.p, nffts, dout.p, s);
    });
}

extern "C" {

int dspb200_os_plan_create(dspb200_os_plan** plan, int dtype, const void* v_host, int64_t nv, int64_t nfft) {
    DSP_RANGE("dspb200_os_plan_create");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    *plan = nullptr;
    DSP_REQUIRE(dtype_valid(dtype), "invalid dtype %d", dtype);
    DSP_REQUIRE(v_host != nullptr && nv >= 1, "filter must be non-empty");
    DSP_REQUIRE(nfft == 0 || nfft >= nv, "nfft (%lld) must be >= nv (%lld)", (long long)nfft, (long long)nv);
    DSP_REQUIRE(nfft < (int64_t(1) << 30), "nfft too large");
    dspb200_os_plan* h = new (std::nothrow) dspb200_os_plan();
    DSP_REQUIRE(h != nullptr, "out of host memory");
    OsPlanImpl* p = &h->impl;
    p->dtype = dtype; p->cplx = dtype_is_cplx(dtype); p->f64 = dtype_is_f64(dtype);
    p->nv = nv;
    p->nfft = nfft ? nfft : auto_nfft(nv, p->f64);
    p->L = p->nfft - nv + 1;
    p->fused = os_fused_ok(p->nfft, nv, p->f64);
    const size_t esz = dtype_size(dtype), csz = p->f64 ? 16 : 8;
    int rc = DSPB200_OK;
    void* d_v = nullptr;
    do {
        cudaError_t e = cudaGetDevice(&p->device);
        if (e != cudaSuccess) { rc = cuda_fail(e, "cudaGetDevice", __FILE__, __LINE__); break; }
        rc = upload(&d_v, v_host, (size_t)nv * esz);
        if (rc != DSPB200_OK) break;
        if (p->fused) {
            p->sm_count = device_sm_count();
            rc = upload_fft_tables(p->nfft, p->f64, &p->d_tw, &p->d_t16, &p->d_t256);
            if (rc != DSPB200_OK) break;
            if (!p->f64 && p->nfft == fft_r32::N) {                // the 16384-point Float32 kernels' plan (os_unit_r32)
                std::vector<cx<float>> tab(fft_r32::TABLE_LEN);
                fft_r32_fill_tables<float>(tab.data());
                rc = upload(&p->d_r32, tab.data(), tab.size() * sizeof(cx<float>));
                if (rc != DSPB200_OK) break;
            }
            e = cudaMalloc(&p->d_H, (size_t)p->nfft * csz);
            if (e != cudaSuccess) { rc = cuda_fail(e, "cudaMalloc(H)", __FILE__, __LINE__); break; }
            rc = p->f64 ? os_filter_dispatch<double>(p, d_v) : os_filter_dispatch<float>(p, d_v);
        } else {
            p->nbins = p->cplx ? p->nfft : p->nfft / 2 + 1;
            int64_t b = (int64_t(1) << 22) / p->nfft;   // ~32 MiB (C32) of blocks in flight: stays L2-resident
            if (b < 1) b = 1;
            if (b > 4096) b = 4096;
            p->batch = b;
            rc = fft_plan_1d(&p->fwd, p->cplx, p->f64, CUFFT_FORWARD, p->nfft, b);
            if (rc == DSPB200_OK) rc = fft_plan_1d(&p->inv, p->cplx, p->f64, CUFFT_INVERSE, p->nfft, b);
            if (rc != DSPB200_OK) break;
            p->fft_ok = true;
            rc = p->td.reserve((size_t)(b * p->nfft) * esz);
            if (rc == DSPB200_OK) rc = p->fd.reserve((size_t)(b * p->nbins) * csz);
            if (rc != DSPB200_OK) break;
            e = cudaMalloc(&p->d_H, (size_t)p->nbins * csz);
            if (e != cudaSuccess) { rc = cuda_fail(e, "cudaMalloc(H)", __FILE__, __LINE__); break; }
            // H = FFT(zero-padded v / nfft): reuse the batch plan on row 0 of td (other rows zero)
            e = cudaMemset(p->td.p, 0, (size_t)(b * p->nfft) * esz);
            if (e != cudaSuccess) { rc = cuda_fail(e, "cudaMemset", __FILE__, __LINE__); break; }
            const int threads = 256;
            if (p->f64) {
                if (p->cplx) pad_copy_kernel<double, true><<<grid_for(p->nfft, threads), threads>>>(d_v, nv, p->td.p, p->nfft, 1.0 / (double)p->nfft);
                else pad_copy_kernel<double, false><<<grid_for(p->nfft, threads), threads>>>(d_v, nv, p->td.p, p->nfft, 1.0 / (double)p->nfft);
            } else {
                if (p->cplx) pad_copy_kernel<float, true><<<grid_for(p->nfft, threads), threads>>>(d_v, nv, p->td.p, p->nfft, 1.0f / (float)p->nfft);
                else pad_copy_kernel<float, false><<<grid_for(p->nfft, threads), threads>>>(d_v, nv, p->td.p, p->nfft, 1.0f / (float)p->nfft);
            }
            count_launch(1);
            rc = fft_exec(p->fwd, p->cplx, p->f64, CUFFT_FORWARD, p->td.p, p->fd.p, 0);
            if (rc != DSPB200_OK) break;
            e = cudaMemcpy(p->d_H, p->fd.p, (size_t)p->nbins * csz, cudaMemcpyDeviceToDevice);
            if (e == cudaSuccess) e = cudaDeviceSynchronize();
            if (e != cudaSuccess) { rc = cuda_fail(e, "filter transform", __FILE__, __LINE__); break; }
        }
    } while (0);
    if (d_v) cudaFree(d_v);
    if (rc != DSPB200_OK) { dspb200_os_plan_destroy(h); return rc; }
    *plan = h;
    return DSPB200_OK;
}

int dspb200_os_plan_nfft(const dspb200_os_plan* plan, int64_t* nfft, int* fused) {
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    if (nfft) *nfft = plan->impl.nfft;
    if (fused) *fused = plan->impl.fused ? 1 : 0;
    return DSPB200_OK;
}

int dspb200_os_plan_geometry(const dspb200_os_plan* plan, int* dtype, int64_t* nv, int64_t* nfft) {
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    if (dtype) *dtype = plan->impl.dtype;
    if (nv) *nv = plan->impl.nv;
    if (nfft) *nfft = plan->impl.nfft;
    return DSPB200_OK;
}

int dspb200_os_exec_dev(dspb200_os_plan* plan, const void* u, int64_t nu, int64_t ncols, void* out, int64_t nout,
                        void* stream) {
    DSP_RANGE("dspb200_os_exec_dev");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    DSP_REQUIRE(nu >= 0 && ncols >= 0 && nout >= 0, "negative size");
    if (nout == 0 || ncols == 0) return DSPB200_OK;
    DSP_REQUIRE(out != nullptr && (u != nullptr || nu == 0), "NULL argument");
    OsPlanImpl* p = &plan->impl;
    if (nu == 0) {
        DSP_CUDA(cudaMemsetAsync(out, 0, (size_t)(nout * ncols) * dtype_size(p->dtype), (cudaStream_t)stream));
        return DSPB200_OK;
    }
    OsRange a{u, 0, nu, nu, out, 0, nout, nout, nu + p->nv - 1, ncols};
    return os_run(p, a, (cudaStream_t)stream);
}

int dspb200_os_exec_range_dev(dspb200_os_plan* plan, const void* u_local, int64_t u_begin, int64_t nu_local,
                              void* out_local, int64_t out_begin, int64_t out_count, void* stream) {
    DSP_RANGE("dspb200_os_exec_range_dev");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    DSP_REQUIRE(nu_local >= 0 && out_count >= 0 && out_begin >= 0, "bad range");
    DSP_REQUIRE(index_in_domain(u_begin) && index_in_domain(nu_local) && index_in_domain(out_begin) &&
                    index_in_domain(out_count) && index_in_domain(u_begin + nu_local) && index_in_domain(out_begin + out_count),
                "range outside the index domain: u_begin %lld, nu_local %lld, out_begin %lld, out_count %lld (limit 2^61)",
                (long long)u_begin, (long long)nu_local, (long long)out_begin, (long long)out_count);
    if (out_count == 0) return DSPB200_OK;
    DSP_REQUIRE(out_local != nullptr && (u_local != nullptr || nu_local == 0), "NULL argument");
    OsPlanImpl* p = &plan->impl;
    OsRange a{u_local, u_begin, nu_local, 0, out_local, out_begin, out_count, 0, INT64_MAX, 1};
    return os_run(p, a, (cudaStream_t)stream);
}

// Stateful overlap-save (fftfilt(f::DF2TFilter, x)): outputs [0, nx + nv - 1) of each column, the first nv - 1 plus si_in,
// the last nv - 1 into si_out (OsState).  One fused launch, or the generic path's launches per column.
int dspb200_os_exec_state_dev(dspb200_os_plan* plan, const void* x, int64_t nx, int64_t ncols, const void* si_in, void* si_out,
                              void* out, void* stream) {
    DSP_RANGE("dspb200_os_exec_state_dev");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    OsPlanImpl* p = &plan->impl;
    const int64_t ns = p->nv - 1;
    cudaStream_t st = (cudaStream_t)stream;
    DSP_TRY(state_prologue_dev(x, nx, ncols, si_in, si_out, out, ns, dtype_size(p->dtype), st));
    if (nx == 0 || ncols == 0) return DSPB200_OK;
    if (p->fused && p->nfft < OS_STATE_MIN_NFFT) {
        set_error("no stateful overlap-save kernel for nfft=%lld: the stateful form takes plans with nfft = 0 (library choice)",
                  (long long)p->nfft);
        return DSPB200_EUNSUPPORTED;
    }
    if (ns == 0) { si_in = nullptr; si_out = nullptr; }                  // nv == 1: no state
    OsRange a{x, 0, nx, nx, out, 0, nx + (si_out ? ns : 0), nx, INT64_MAX, ncols};
    return os_run<true>(p, a, OsStateArgs{si_in, si_out, nx}, st);
}

// Host pointers.  One long column is streamed in chunks of whole blocks (run_chunked): chunk c+1 is copied in while chunk
// c is convolved and chunk c-1 is copied out; otherwise copy in -> run -> copy out.
int dspb200_os_exec(dspb200_os_plan* plan, const void* u, int64_t nu, int64_t ncols, void* out, int64_t nout) {
    DSP_RANGE("dspb200_os_exec");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    DSP_REQUIRE(nu >= 0 && ncols >= 0 && nout >= 0, "negative size");
    if (nout == 0 || ncols == 0) return DSPB200_OK;
    DSP_REQUIRE(out != nullptr && (u != nullptr || nu == 0), "NULL argument");
    OsPlanImpl* p = &plan->impl;
    HostPipe& hp = p->pipe;
    DSP_TRY(ensure_streams(p));
    const size_t esz = dtype_size(p->dtype);
    const int64_t chunk_out = ((int64_t(32) << 20) / (int64_t)esz / p->L + 1) * p->L;   // ~32 MiB, whole blocks
    if (ncols == 1 && nout > 2 * chunk_out && nu > 0) {
        const int64_t nfull = nu + p->nv - 1;
        auto chunk = [&](int64_t c) -> Chunk {
            const int64_t m0 = c * chunk_out, cnt = nout - m0 < chunk_out ? nout - m0 : chunk_out;
            int64_t i_lo = m0 - (p->nv - 1); if (i_lo < 0) i_lo = 0;
            int64_t i_hi = m0 + cnt; if (i_hi > nu) i_hi = nu;
            const int64_t ni = i_hi > i_lo ? i_hi - i_lo : 0;
            auto run = [=, &hp](const void* in, void* o) {
                return os_run(p, OsRange{in, i_lo, ni, 0, o, m0, cnt, 0, nfull, 1}, hp.s_exec);
            };
            return {(const char*)u + (size_t)i_lo * esz, (size_t)ni * esz, run, nullptr, (char*)out + (size_t)m0 * esz, (size_t)cnt * esz};
        };
        return run_chunked(hp, cdiv(nout, chunk_out), (size_t)(chunk_out + p->nv - 1) * esz, (size_t)chunk_out * esz, chunk, nullptr);
    }
    return run_staged(hp.s_exec, {{u, (size_t)(nu * ncols) * esz, &hp.in[0]}}, {{out, (size_t)(nout * ncols) * esz, &hp.out[0]}},
                      [&] { return dspb200_os_exec_dev(plan, hp.in[0].p, nu, ncols, hp.out[0].p, nout, hp.s_exec); });
}

// Host pointers: x and the state are staged apart (x in in[0], out in out[0], si_in in in[1], si_out in out[1]).
int dspb200_os_exec_state(dspb200_os_plan* plan, const void* x, int64_t nx, int64_t ncols, const void* si_in, void* si_out,
                          void* out) {
    DSP_RANGE("dspb200_os_exec_state");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    OsPlanImpl* p = &plan->impl;
    HostPipe& hp = p->pipe;
    return exec_state_host(p, hp.s_exec, x, nx, ncols, si_in, si_out, out, p->nv - 1, dtype_size(p->dtype), hp.in[0], hp.out[0],
                           hp.in[1], hp.out[1], [&](const void* d_x, const void* d_si_in, void* d_si_out, void* d_out) {
                               return dspb200_os_exec_state_dev(plan, d_x, nx, ncols, d_si_in, d_si_out, d_out, hp.s_exec);
                           });
}

int dspb200_os_plan_destroy(dspb200_os_plan* plan) {
    if (!plan) return DSPB200_OK;
    OsPlanImpl* p = &plan->impl;
    if (p->d_tw) cudaFree(p->d_tw);
    if (p->d_t16) cudaFree(p->d_t16);
    if (p->d_t256) cudaFree(p->d_t256);
    if (p->d_r32) cudaFree(p->d_r32);
    if (p->d_H) cudaFree(p->d_H);
    if (p->fft_ok) { cufftDestroy(p->fwd); cufftDestroy(p->inv); }
    p->td.release(); p->fd.release();
    p->pipe.release();
    delete plan;
    return DSPB200_OK;
}

// _conv_kern_fft!, src/dspbase.jl:611-644: the rank-1 transform pair of dspb200_conv_nd_exec (host pointers)
int dspb200_conv_fft_exec(int dtype, const void* u, int64_t nu, const void* v, int64_t nv, int64_t nfft, void* out) {
    DSP_RANGE("dspb200_conv_fft_exec");
    DSP_TRY(conv_nd_check(dtype, ND_FFT, 1, &nu, u, &nv, v, &nfft, out));
    return conv_nd_run_host(dtype, ND_FFT, 1, &nu, u, &nv, v, &nfft, out);
}

// conv(u, v) / conv!(out, u, v) for matrices and rank-3 arrays, src/dspbase.jl:611-660, 709-757 (cached plans)
int dspb200_conv_nd_exec(int dtype, int rank, const int64_t* usize, const void* u, const int64_t* vsize, const void* v,
                         const int64_t* nffts, void* out) {
    DSP_RANGE("dspb200_conv_nd_exec");
    const int mode = nffts ? ND_FFT : ND_DIRECT;
    DSP_TRY(conv_nd_check(dtype, mode, rank, usize, u, vsize, v, nffts, out));
    return conv_nd_run_host(dtype, mode, rank, usize, u, vsize, v, nffts, out);
}
int dspb200_conv_nd_exec_dev(int dtype, int rank, const int64_t* usize, const void* d_u, const int64_t* vsize, const void* d_v,
                             const int64_t* nffts, void* d_out, void* stream) {
    DSP_RANGE("dspb200_conv_nd_exec_dev");
    const int mode = nffts ? ND_FFT : ND_DIRECT;
    DSP_TRY(conv_nd_check(dtype, mode, rank, usize, d_u, vsize, d_v, nffts, d_out));
    return conv_nd_run_dev(dtype, mode, rank, usize, d_u, vsize, d_v, nffts, d_out, reinterpret_cast<cudaStream_t>(stream));
}

// conv(u, v; algorithm=:fft_overlapsave) for arrays of rank <= 3: unsafe_conv_kern_os!, src/dspbase.jl:371-609
int dspb200_conv_nd_os_exec(int dtype, int rank, const int64_t* usize, const void* u, const int64_t* vsize, const void* v,
                            const int64_t* nffts, void* out) {
    DSP_RANGE("dspb200_conv_nd_os_exec");
    DSP_TRY(conv_nd_check(dtype, ND_OS, rank, usize, u, vsize, v, nffts, out));
    return conv_nd_run_host(dtype, ND_OS, rank, usize, u, vsize, v, nffts, out);
}
int dspb200_conv_nd_os_exec_dev(int dtype, int rank, const int64_t* usize, const void* d_u, const int64_t* vsize, const void* d_v,
                                const int64_t* nffts, void* d_out, void* stream) {
    DSP_RANGE("dspb200_conv_nd_os_exec_dev");
    DSP_TRY(conv_nd_check(dtype, ND_OS, rank, usize, d_u, vsize, d_v, nffts, d_out));
    return conv_nd_run_dev(dtype, ND_OS, rank, usize, d_u, vsize, d_v, nffts, d_out, reinterpret_cast<cudaStream_t>(stream));
}
int dspb200_conv_nd_os_set_budget(size_t bytes) {
    DSP_REQUIRE(bytes >= 1, "the block-buffer budget must be positive");
    g_nd_os_budget = bytes;
    return DSPB200_OK;
}

// hilbert(x), src/util.jl:31-75 (kernel: hilbert_weight_kernel above)
static int hilbert_check(int dtype, const void* x, int64_t n, int64_t ncols, const void* out) {
    DSP_REQUIRE(dtype == DSPB200_F32 || dtype == DSPB200_F64, "hilbert takes a real signal (dtype %d)", dtype);
    DSP_REQUIRE(x && out && n >= 1 && ncols >= 1, "empty or NULL input");
    DSP_REQUIRE(n < (int64_t(1) << 31), "n too large");
    return DSPB200_OK;
}

// queues the transforms and the weighting on st (cached plans: the caller holds the ConvenienceLock)
static int hilbert_queue(int dtype, const void* d_x, int64_t n, int64_t ncols, void* d_out, cudaStream_t st) {
    const bool f64 = dtype == DSPB200_F64;
    long long nn[1] = {(long long)n};
    int hf = 0, hi = 0;
    // real -> complex, column c: n reals at c*n  ->  n/2+1 bins at the start of the n-bin output column c
    DSP_TRY(plan_cache_get(&hf, 1, nn, true, n, n, fft_type(false, f64, CUFFT_FORWARD), ncols));
    DSP_TRY(plan_cache_get(&hi, 1, nn, false, 0, 0, fft_type(true, f64, CUFFT_INVERSE), ncols));
    DSP_TRY(fft_exec((cufftHandle)hf, false, f64, CUFFT_FORWARD, d_x, d_out, st));
    const int threads = 256, g = grid_for(n * ncols, threads);
    if (f64) hilbert_weight_kernel<double><<<g, threads, 0, st>>>((cx<double>*)d_out, n, ncols, 1.0 / (double)n);
    else hilbert_weight_kernel<float><<<g, threads, 0, st>>>((cx<float>*)d_out, n, ncols, 1.0f / (float)n);
    DSP_LAUNCH_OK();
    return fft_exec((cufftHandle)hi, true, f64, CUFFT_INVERSE, d_out, d_out, st);
}

int dspb200_hilbert_exec_dev(int dtype, const void* d_x, int64_t n, int64_t ncols, void* d_out, void* stream) {
    DSP_RANGE("dspb200_hilbert_exec_dev");
    DSP_TRY(hilbert_check(dtype, d_x, n, ncols, d_out));
    return convenience_call(reinterpret_cast<cudaStream_t>(stream),
                            [&](cudaStream_t st) { return hilbert_queue(dtype, d_x, n, ncols, d_out, st); });
}

int dspb200_hilbert_exec(int dtype, const void* x, int64_t n, int64_t ncols, void* out) {
    DSP_RANGE("dspb200_hilbert_exec");
    DSP_TRY(hilbert_check(dtype, x, n, ncols, out));
    const size_t bytes = (size_t)(n * ncols) * dtype_size(dtype);
    DevBuf &dx = scratch_buf(0), &dout = scratch_buf(1);
    return convenience_call({{x, bytes, &dx}}, {{out, 2 * bytes, &dout}},
                            [&](cudaStream_t st) { return hilbert_queue(dtype, dx.p, n, ncols, dout.p, st); });
}

// _conv_td!, src/dspbase.jl:646-660: the rank-1 direct convolution of dspb200_conv_nd_exec (host pointers)
int dspb200_conv_direct_exec(int dtype, const void* u, int64_t nu, const void* v, int64_t nv, void* out) {
    DSP_RANGE("dspb200_conv_direct_exec");
    DSP_TRY(conv_nd_check(dtype, ND_DIRECT, 1, &nu, u, &nv, v, nullptr, out));
    return conv_nd_run_host(dtype, ND_DIRECT, 1, &nu, u, &nv, v, nullptr, out);
}

}  // extern "C"
