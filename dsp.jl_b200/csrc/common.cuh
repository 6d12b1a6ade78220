// dspb200 -- common device/host helpers (complex type, dtype traits, error plumbing).
#pragma once
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdarg.h>
#include <functional>
#include <initializer_list>
#include <type_traits>

#include "../../include/dspb200.h"

namespace dspb200 {

// ----------------------------------------------------------------------------------------------
// Interleaved complex (layout-identical to Julia's Complex{T}, float2 / double2).
template <typename T>
struct alignas(2 * sizeof(T)) cx {
    T x, y;
};

template <typename T> __host__ __device__ __forceinline__ cx<T> mkc(T a, T b) { cx<T> r; r.x = a; r.y = b; return r; }
template <typename T> __host__ __device__ __forceinline__ cx<T> operator+(cx<T> a, cx<T> b) { return mkc<T>(a.x + b.x, a.y + b.y); }
template <typename T> __host__ __device__ __forceinline__ cx<T> operator-(cx<T> a, cx<T> b) { return mkc<T>(a.x - b.x, a.y - b.y); }
template <typename T> __host__ __device__ __forceinline__ cx<T> cmul(cx<T> a, cx<T> b) {
    return mkc<T>(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
template <typename T> __host__ __device__ __forceinline__ cx<T> cscale(cx<T> a, T s) { return mkc<T>(a.x * s, a.y * s); }
template <typename T> __host__ __device__ __forceinline__ cx<T> cconj(cx<T> a) { return mkc<T>(a.x, -a.y); }
template <typename T> __host__ __device__ __forceinline__ cx<T> cswap(cx<T> a) { return mkc<T>(a.y, a.x); }
// multiply by -i
template <typename T> __host__ __device__ __forceinline__ cx<T> mul_mi(cx<T> a) { return mkc<T>(a.y, -a.x); }
template <typename T> __host__ __device__ __forceinline__ T cabs2(cx<T> a) { return a.x * a.x + a.y * a.y; }

// ----------------------------------------------------------------------------------------------
// dtype traits
template <typename E> struct elt_traits;
template <> struct elt_traits<float>       { using real = float;  static constexpr bool is_cplx = false; };
template <> struct elt_traits<double>      { using real = double; static constexpr bool is_cplx = false; };
template <> struct elt_traits<cx<float>>   { using real = float;  static constexpr bool is_cplx = true; };
template <> struct elt_traits<cx<double>>  { using real = double; static constexpr bool is_cplx = true; };

inline size_t dtype_size(int dt) {
    switch (dt) {
        case DSPB200_F32: return 4;
        case DSPB200_F64: return 8;
        case DSPB200_C32: return 8;
        case DSPB200_C64: return 16;
    }
    return 0;
}
inline bool dtype_is_cplx(int dt) { return dt == DSPB200_C32 || dt == DSPB200_C64; }
inline bool dtype_is_f64(int dt) { return dt == DSPB200_F64 || dt == DSPB200_C64; }
inline bool dtype_valid(int dt) { return dt >= 0 && dt <= 3; }

// ----------------------------------------------------------------------------------------------
// error plumbing (thread-local message; the C ABI never throws)
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define DSP_CUDA(call)                                                              \
    do {                                                                            \
        cudaError_t e__ = (call);                                                   \
        if (e__ != cudaSuccess) return ::dspb200::cuda_fail(e__, #call, __FILE__, __LINE__); \
    } while (0)

#define DSP_REQUIRE(cond, ...)                    \
    do {                                          \
        if (!(cond)) {                            \
            ::dspb200::set_error(__VA_ARGS__);    \
            return DSPB200_EINVALID;              \
        }                                         \
    } while (0)

// A global sample or output index of a range form inside the domain dspb200.h states (|v| <= DSPB200_INDEX_LIMIT): the
// sum and difference of two such indices cannot overflow int64_t.
static inline bool index_in_domain(int64_t v) { return v >= -DSPB200_INDEX_LIMIT && v <= DSPB200_INDEX_LIMIT; }

// NVTX range around every C-ABI entry point that does device work (SURVEY.md section 5: the reference has no tracing; this
// is what makes the library's calls visible on an Nsight timeline).  Header-only NVTX3: a no-op unless a tool is attached.
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};
#define DSP_RANGE(name) ::dspb200::NvtxRange nvtx_range__(name)

#define DSP_TRY(expr)               \
    do {                            \
        int rc__ = (expr);          \
        if (rc__ != DSPB200_OK) return rc__; \
    } while (0)

// Device scratch buffer that only grows (owned by plans).
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    int reserve(size_t bytes) {
        if (bytes <= cap) return DSPB200_OK;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e != cudaSuccess) { set_error("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e)); cudaGetLastError(); return DSPB200_ENOMEM; }
        cap = bytes;
        return DSPB200_OK;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

// *d = a new device copy of h's bytes (plan constructors: taps, twiddle tables)
int upload(void** d, const void* h, size_t bytes);
// the fused FFT kernels' tables for nfft points (fft_core.cuh): last-pass twiddles, radix-16 and radix-256 tables
int upload_fft_tables(int64_t nfft, bool f64, void** d_tw, void** d_t16, void** d_t256);

// Creates *s, a non-blocking stream, unless it exists (the private streams of a plan's host-pointer entry points).
inline int ensure_stream(cudaStream_t* s) {
    if (!*s) DSP_CUDA(cudaStreamCreateWithFlags(s, cudaStreamNonBlocking));
    return DSPB200_OK;
}

// Waits for `st` whether or not `rc` reports a failure, so that no error return leaves work that reads or writes the
// caller's memory in flight.  Returns rc, or the synchronisation's error when rc is DSPB200_OK.
int settle(cudaStream_t st, int rc);

inline bool ranges_overlap(const void* a, size_t na, const void* b, size_t nb) {
    return a && b && na && nb && (const char*)a < (const char*)b + nb && (const char*)b < (const char*)a + na;
}

// Host-pointer entry points are staging around their device-pointer twins: reserve the device buffers (16 bytes at least,
// so that every staged pointer is valid), queue the host-to-device copies on `st`, run dev() (usually the twin, reading
// the buffers' pointers), queue the device-to-host copies, and return once `st` is idle, on success and failure alike.
struct HostIn { const void* src; size_t bytes; DevBuf* buf; };
struct HostOut { void* dst; size_t bytes; DevBuf* buf; };
template <class F>
int run_staged(cudaStream_t st, std::initializer_list<HostIn> in, std::initializer_list<HostOut> out, F&& dev) {
    auto queue = [&]() -> int {
        for (const HostIn& h : in) DSP_TRY(h.buf->reserve(h.bytes ? h.bytes : 16));
        for (const HostOut& h : out) DSP_TRY(h.buf->reserve(h.bytes ? h.bytes : 16));
        for (const HostIn& h : in)
            if (h.bytes) DSP_CUDA(cudaMemcpyAsync(h.buf->p, h.src, h.bytes, cudaMemcpyHostToDevice, st));
        DSP_TRY(dev());
        for (const HostOut& h : out)
            if (h.bytes) DSP_CUDA(cudaMemcpyAsync(h.dst, h.buf->p, h.bytes, cudaMemcpyDeviceToHost, st));
        return DSPB200_OK;
    };
    return settle(st, queue());
}

// The streams, events and device slots of a plan's host-pointer calls.  One-shot calls stage through in[0] / out[0] on
// s_exec (run_staged); chunked calls (run_chunked) give chunk c slot c % 2, copied in on s_in, computed on s_exec and
// drained on s_out, so that chunk c+1's copy in and chunk c-1's copy out overlap chunk c's kernels.
struct HostPipe {
    cudaStream_t s_in = nullptr, s_exec = nullptr, s_out = nullptr;
    cudaEvent_t ev_in[2] = {}, ev_exec[2] = {}, ev_out[2] = {};
    DevBuf in[2], out[2];
    int ensure(int device);   // makes `device` current and creates the streams and events on first use
    void release();
};

// One chunk of run_chunked: `bytes` of host input at `src` are copied into the slot's input buffer, read(in, out) queues on
// s_exec the work that reads the slot's input buffer and writes its output buffer, after() (optional) queues further work
// on s_exec that uses neither buffer, and `out_bytes` (optional) of the output buffer are then copied to `dst`.
struct Chunk {
    const void* src;
    size_t bytes;
    std::function<int(const void* in, void* out)> read;
    std::function<int()> after;
    void* dst = nullptr;
    size_t out_bytes = 0;
};

// Host-pointer calls that stream the caller's buffers through the two slots of `hp`: reserve in_cap (and out_cap, if any)
// bytes per slot used, queue chunk(0) ... chunk(nchunks - 1) and then tail() (optional) on s_exec, and return once all
// three streams are idle, on success and failure alike (the first error is the one reported).  A slot is refilled once its
// last read is done and written once its last output has been drained.
int run_chunked(HostPipe& hp, int64_t nchunks, size_t in_cap, size_t out_cap, const std::function<Chunk(int64_t)>& chunk,
                const std::function<int()>& tail);

// Stateful FIR and overlap-save calls (DF2TFilter): ns state elements of esz bytes per column, in si_in (NULL: zero state)
// and out to si_out (NULL: not wanted).
// Device form: the size and overlap checks -- CTAs read the samples, halo and state behind other CTAs' outputs, so a
// buffer that is written must not overlap one that is read (or the other written one) -- and, for nx == 0, the state
// passed through on `st`.  The caller returns after this when nx == 0 or ncols == 0.
int state_prologue_dev(const void* x, int64_t nx, int64_t ncols, const void* si_in, void* si_out, void* out, int64_t ns,
                       size_t esz, cudaStream_t st);
// Host form, for a plan P with ensure_streams(P*), which creates the plan's execute stream `s_exec` (hence taken by
// reference: it is read after ensure_streams has run): x and the state are staged apart (bx, bout, bsi, bso), so out may
// be x and si_out may be si_in; nx == 0 passes the state through on the host.
// dev(d_x, d_si_in, d_si_out, d_out) runs the device form on s_exec.
template <class P, class F>
int exec_state_host(P* p, const cudaStream_t& s_exec, const void* x, int64_t nx, int64_t ncols, const void* si_in, void* si_out,
                    void* out, int64_t ns, size_t esz, DevBuf& bx, DevBuf& bout, DevBuf& bsi, DevBuf& bso, F&& dev) {
    DSP_REQUIRE(nx >= 0 && ncols >= 0, "negative size");
    if (ncols == 0) return DSPB200_OK;
    DSP_REQUIRE(nx == 0 || (x && out), "NULL argument");
    const size_t bytes = (size_t)(nx * ncols) * esz, sbytes = (size_t)(ns * ncols) * esz;
    if (nx == 0) {
        if (si_out && sbytes && si_out != si_in) {
            if (si_in) memmove(si_out, si_in, sbytes);
            else memset(si_out, 0, sbytes);
        }
        return DSPB200_OK;
    }
    DSP_TRY(ensure_streams(p));
    return run_staged(s_exec, {{x, bytes, &bx}, {si_in, si_in ? sbytes : 0, &bsi}},
                      {{out, bytes, &bout}, {si_out, si_out ? sbytes : 0, &bso}},
                      [&] { return dev(bx.p, si_in ? bsi.p : nullptr, si_out ? bso.p : nullptr, bout.p); });
}

int device_sm_count();
// height rows of width bytes, src + r*spitch -> dst + r*dpitch, device to device on st: one cudaMemcpy2DAsync, or one
// cudaMemcpyAsync per row where a pitch exceeds the device's cudaDevAttrMaxPitch (columns of more than ~2 GiB) or there is
// one row.  Copies, no kernel launch.
int memcpy2d_dd(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t height, cudaStream_t st);
void count_launch(int n = 1);

// cuFFT plans and device scratch of the plan-less convenience entry points (conv_fft, conv_nd, hilbert, periodogram2) are
// cached: round 1 created and destroyed two plans and up to six allocations per call.  `plan_cache_get` returns a handle
// owned by the cache (never destroy it); `embed` selects inembed = onembed = n with the given distances (hilbert's
// real -> complex plan), otherwise the default packed layout.  The cache keeps the 32 most recently used plans per
// process; the calls that use them go through `convenience_call` below, which serialises them (they are synchronous).
int plan_cache_get(int* handle, int rank, const long long* n, bool embed, long long idist, long long odist, int type, long long batch);
DevBuf& scratch_buf(int slot);            // per-process grow-only device buffers, slot 0..7
void scratch_trim(size_t keep_bytes);     // release the buffers larger than keep_bytes
struct ConvenienceLock { ConvenienceLock(); ~ConvenienceLock(); };

// The one exit of the plan-less entry points: under the ConvenienceLock, queue(st) queues the call's work on st, the call
// returns once st is idle, on success and failure alike, and the arena then drops its large buffers (the plans and the
// small buffers stay for the next call).  queue() neither locks nor trims, so that no buffer it uses is freed under it.
// Device-pointer form:
template <class F> int convenience_call(cudaStream_t st, F&& queue) {
    ConvenienceLock lock;
    const int rc = settle(st, queue(st));
    scratch_trim((size_t)256 << 20);
    return rc;
}
// Host-pointer form: queue(0) between the copies of run_staged (the staging buffers are arena slots).
template <class F> int convenience_call(std::initializer_list<HostIn> in, std::initializer_list<HostOut> out, F&& queue) {
    ConvenienceLock lock;
    const int rc = run_staged(0, in, out, [&] { return queue(cudaStream_t(0)); });
    scratch_trim((size_t)256 << 20);
    return rc;
}

// after every kernel launch
#define DSP_LAUNCH_OK()                                                              \
    do {                                                                            \
        ::dspb200::count_launch(1);                                                 \
        cudaError_t e__ = cudaGetLastError();                                       \
        if (e__ != cudaSuccess) return ::dspb200::cuda_fail(e__, "kernel launch", __FILE__, __LINE__); \
    } while (0)
static inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Programmatic dependent launch (sm_90+).  The persistent kernels of a pipeline (overlap-save -> Welch -> finalize -> next
// overlap-save) are launched with programmatic stream serialisation: a kernel's CTAs may become resident as soon as the
// previous kernel's CTAs leave an SM, stage their twiddle tables / window (constants since plan creation) and then block
// in `pdl_wait()` until the previous grid has completed and its memory is visible -- the launch gap and the table prologue
// (49 KB per CTA for the 16384-point Float32 kernel) overlap the previous kernel's tail instead of following it.  EVERY
// thread executes pdl_wait() before its first access to anything a preceding kernel could have written or still be
// reading, so the chain is transitive.  Kernels launched without the attribute execute both instructions as no-ops.
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
template <typename... KA, typename... A>
static inline cudaError_t launch_pdl(void (*kern)(KA...), unsigned grid, unsigned block, size_t smem, cudaStream_t st, A... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, KA(args)...);
}
#endif

}  // namespace dspb200
