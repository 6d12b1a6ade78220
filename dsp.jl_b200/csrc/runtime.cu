// dspb200 -- runtime entry points: errors, device selection, memory helpers.
#include "common.cuh"
#include "cufft_exec.cuh"
#include "fft_core.cuh"
#include <atomic>
#include <mutex>
#include <vector>

namespace dspb200 {

static thread_local char g_err[512] = "";
std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
    set_error("CUDA error %d (%s) in %s at %s:%d", (int)e, cudaGetErrorString(e), what, file, line);
    cudaGetLastError();
    return e == cudaErrorMemoryAllocation ? DSPB200_ENOMEM : DSPB200_ECUDA;
}

int device_sm_count() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
    return n;
}

int memcpy2d_dd(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t height, cudaStream_t st) {
    if (width == 0 || height == 0) return DSPB200_OK;
    int dev = 0, max_pitch = 0;
    DSP_CUDA(cudaGetDevice(&dev));
    DSP_CUDA(cudaDeviceGetAttribute(&max_pitch, cudaDevAttrMaxPitch, dev));
    if (height > 1 && dpitch <= (size_t)max_pitch && spitch <= (size_t)max_pitch) {
        DSP_CUDA(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, height, cudaMemcpyDeviceToDevice, st));
        return DSPB200_OK;
    }
    for (size_t r = 0; r < height; ++r)
        DSP_CUDA(cudaMemcpyAsync((char*)dst + r * dpitch, (const char*)src + r * spitch, width, cudaMemcpyDeviceToDevice, st));
    return DSPB200_OK;
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int cufft_fail(cufftResult r, const char* what) {
    set_error("cuFFT error %d in %s", (int)r, what);
    return DSPB200_ECUFFT;
}

int fft_plan_1d(cufftHandle* h, bool cplx, bool f64, int dir, int64_t n, int64_t batch) {
    long long nn[1] = {(long long)n};
    size_t ws = 0;
    *h = 0;
    DSP_CUFFT(cufftCreate(h));
    const cufftResult r = cufftMakePlanMany64(*h, 1, nn, nullptr, 1, 0, nullptr, 1, 0, fft_type(cplx, f64, dir), (long long)batch, &ws);
    if (r != CUFFT_SUCCESS) {
        cufftDestroy(*h);
        *h = 0;
        return cufft_fail(r, "cufftMakePlanMany64");
    }
    return DSPB200_OK;
}

int fft_exec(cufftHandle h, bool cplx, bool f64, int dir, const void* in, void* out, cudaStream_t st) {
    void* src = const_cast<void*>(in);                              // cuFFT takes non-const input pointers
    DSP_CUFFT(cufftSetStream(h, st));
    if (cplx) {
        if (f64) DSP_CUFFT(cufftExecZ2Z(h, (cufftDoubleComplex*)src, (cufftDoubleComplex*)out, dir));
        else DSP_CUFFT(cufftExecC2C(h, (cufftComplex*)src, (cufftComplex*)out, dir));
    } else if (dir == CUFFT_FORWARD) {
        if (f64) DSP_CUFFT(cufftExecD2Z(h, (cufftDoubleReal*)src, (cufftDoubleComplex*)out));
        else DSP_CUFFT(cufftExecR2C(h, (cufftReal*)src, (cufftComplex*)out));
    } else {
        if (f64) DSP_CUFFT(cufftExecZ2D(h, (cufftDoubleComplex*)src, (cufftDoubleReal*)out));
        else DSP_CUFFT(cufftExecC2R(h, (cufftComplex*)src, (cufftReal*)out));
    }
    count_launch(1);
    return DSPB200_OK;
}

int upload(void** d, const void* h, size_t bytes) {
    DSP_CUDA(cudaMalloc(d, bytes));
    DSP_CUDA(cudaMemcpy(*d, h, bytes, cudaMemcpyHostToDevice));
    return DSPB200_OK;
}

template <typename T>
static int upload_fft_tables(int64_t nfft, void** d_tw, void** d_t16, void** d_t256) {
    std::vector<cx<T>> tw((size_t)fft_tl_len_rt(nfft) + 1), t16((size_t)fft_tw16_len(nfft)), t256((size_t)fft_tw256_len(nfft));
    fft_fill_tl<T>(tw.data(), nfft);
    fft_fill_tables<T>(t16.data(), t256.data(), nfft);
    DSP_TRY(upload(d_tw, tw.data(), tw.size() * sizeof(cx<T>)));
    DSP_TRY(upload(d_t16, t16.data(), t16.size() * sizeof(cx<T>)));
    return upload(d_t256, t256.data(), t256.size() * sizeof(cx<T>));
}
int upload_fft_tables(int64_t nfft, bool f64, void** d_tw, void** d_t16, void** d_t256) {
    return f64 ? upload_fft_tables<double>(nfft, d_tw, d_t16, d_t256) : upload_fft_tables<float>(nfft, d_tw, d_t16, d_t256);
}

int settle(cudaStream_t st, int rc) {
    const cudaError_t e = cudaStreamSynchronize(st);
    if (rc != DSPB200_OK) {
        cudaGetLastError();                             // the first error is the one reported
        return rc;
    }
    return e == cudaSuccess ? DSPB200_OK : cuda_fail(e, "cudaStreamSynchronize", __FILE__, __LINE__);
}

int HostPipe::ensure(int device) {
    DSP_CUDA(cudaSetDevice(device));
    if (s_exec) return DSPB200_OK;                                       // s_exec is created last: it marks the set complete
    DSP_TRY(ensure_stream(&s_in));
    DSP_TRY(ensure_stream(&s_out));
    for (cudaEvent_t* ev : {ev_in, ev_exec, ev_out})
        for (int i = 0; i < 2; ++i)
            if (!ev[i]) DSP_CUDA(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
    return ensure_stream(&s_exec);
}

void HostPipe::release() {
    for (int i = 0; i < 2; ++i) {
        in[i].release(); out[i].release();
        for (cudaEvent_t ev : {ev_in[i], ev_exec[i], ev_out[i]})
            if (ev) cudaEventDestroy(ev);
    }
    for (cudaStream_t st : {s_in, s_exec, s_out})
        if (st) cudaStreamDestroy(st);
}

int run_chunked(HostPipe& hp, int64_t nchunks, size_t in_cap, size_t out_cap, const std::function<Chunk(int64_t)>& chunk,
                const std::function<int()>& tail) {
    auto queue = [&]() -> int {
        for (int s = 0; s < 2 && s < nchunks; ++s) {
            DSP_TRY(hp.in[s].reserve(in_cap));
            if (out_cap) DSP_TRY(hp.out[s].reserve(out_cap));
        }
        bool read[2] = {false, false}, draining[2] = {false, false};
        for (int64_t c = 0; c < nchunks; ++c) {
            const int s = (int)(c & 1);
            const Chunk ch = chunk(c);
            if (read[s]) DSP_CUDA(cudaStreamWaitEvent(hp.s_in, hp.ev_exec[s], 0));
            if (ch.bytes) DSP_CUDA(cudaMemcpyAsync(hp.in[s].p, ch.src, ch.bytes, cudaMemcpyHostToDevice, hp.s_in));
            DSP_CUDA(cudaEventRecord(hp.ev_in[s], hp.s_in));
            DSP_CUDA(cudaStreamWaitEvent(hp.s_exec, hp.ev_in[s], 0));
            if (draining[s]) DSP_CUDA(cudaStreamWaitEvent(hp.s_exec, hp.ev_out[s], 0));
            DSP_TRY(ch.read(hp.in[s].p, hp.out[s].p));
            DSP_CUDA(cudaEventRecord(hp.ev_exec[s], hp.s_exec));
            read[s] = true;
            if (ch.after) DSP_TRY(ch.after());
            if (ch.out_bytes) {
                DSP_CUDA(cudaStreamWaitEvent(hp.s_out, hp.ev_exec[s], 0));
                DSP_CUDA(cudaMemcpyAsync(ch.dst, hp.out[s].p, ch.out_bytes, cudaMemcpyDeviceToHost, hp.s_out));
                DSP_CUDA(cudaEventRecord(hp.ev_out[s], hp.s_out));
                draining[s] = true;
            }
        }
        return tail ? tail() : DSPB200_OK;
    };
    return settle(hp.s_out, settle(hp.s_exec, settle(hp.s_in, queue())));
}

int state_prologue_dev(const void* x, int64_t nx, int64_t ncols, const void* si_in, void* si_out, void* out, int64_t ns,
                       size_t esz, cudaStream_t st) {
    DSP_REQUIRE(nx >= 0 && ncols >= 0, "negative size");
    const size_t sbytes = (size_t)(ns * ncols) * esz, xbytes = (size_t)(nx * ncols) * esz;
    DSP_REQUIRE(!ranges_overlap(si_in, sbytes, si_out, sbytes), "si_in and si_out overlap");
    DSP_REQUIRE(!ranges_overlap(x, xbytes, out, xbytes), "x and out overlap (filtering in place needs the host form)");
    DSP_REQUIRE(!ranges_overlap(x, xbytes, si_out, sbytes) && !ranges_overlap(si_in, sbytes, out, xbytes) &&
                    !ranges_overlap(out, xbytes, si_out, sbytes),
                "a state buffer overlaps x or out");
    if (ncols == 0) return DSPB200_OK;
    if (nx == 0) {                                                       // the state passes through unchanged
        if (si_out && sbytes) {
            if (si_in) DSP_CUDA(cudaMemcpyAsync(si_out, si_in, sbytes, cudaMemcpyDeviceToDevice, st));
            else DSP_CUDA(cudaMemsetAsync(si_out, 0, sbytes, st));
        }
        return DSPB200_OK;
    }
    DSP_REQUIRE(x && out, "NULL argument");
    return DSPB200_OK;
}

// ---- plan cache / scratch arena of the plan-less entry points
static std::recursive_mutex g_conv_mutex;
ConvenienceLock::ConvenienceLock() { g_conv_mutex.lock(); }
ConvenienceLock::~ConvenienceLock() { g_conv_mutex.unlock(); }

struct PlanEntry {
    int device, rank, type;
    long long n[3], idist, odist, batch;
    bool embed;
    cufftHandle handle;
    uint64_t stamp;
};
static std::vector<PlanEntry> g_plans;
static uint64_t g_plan_clock = 0;

int plan_cache_get(int* handle, int rank, const long long* n, bool embed, long long idist, long long odist, int type, long long batch) {
    int dev = 0;
    DSP_CUDA(cudaGetDevice(&dev));
    long long nn[3] = {1, 1, 1};
    for (int d = 0; d < rank; ++d) nn[d] = n[d];
    for (auto& e : g_plans) {
        if (e.device == dev && e.rank == rank && e.type == type && e.embed == embed && e.idist == idist && e.odist == odist &&
            e.batch == batch && e.n[0] == nn[0] && e.n[1] == nn[1] && e.n[2] == nn[2]) {
            e.stamp = ++g_plan_clock;
            *handle = (int)e.handle;
            return DSPB200_OK;
        }
    }
    cufftHandle h = 0;
    size_t ws = 0;
    cufftResult r = cufftCreate(&h);
    if (r == CUFFT_SUCCESS)
        r = cufftMakePlanMany64(h, rank, nn, embed ? nn : nullptr, 1, embed ? idist : 0, embed ? nn : nullptr, 1, embed ? odist : 0,
                                (cufftType)type, batch, &ws);
    if (r != CUFFT_SUCCESS) {
        if (h) cufftDestroy(h);
        set_error("cuFFT error %d creating a cached plan", (int)r);
        return DSPB200_ECUFFT;
    }
    if (g_plans.size() >= 32) {                       // evict the least recently used plan
        size_t lru = 0;
        for (size_t i = 1; i < g_plans.size(); ++i) if (g_plans[i].stamp < g_plans[lru].stamp) lru = i;
        cufftDestroy(g_plans[lru].handle);
        g_plans.erase(g_plans.begin() + (long)lru);
    }
    g_plans.push_back(PlanEntry{dev, rank, type, {nn[0], nn[1], nn[2]}, idist, odist, batch, embed, h, ++g_plan_clock});
    *handle = (int)h;
    return DSPB200_OK;
}

static DevBuf g_scratch[8];
DevBuf& scratch_buf(int slot) { return g_scratch[slot & 7]; }
void scratch_trim(size_t keep_bytes) {
    for (auto& b : g_scratch) if (b.cap > keep_bytes) b.release();
}

}  // namespace dspb200

using namespace dspb200;

extern "C" {

int dspb200_version(void) { return DSPB200_VERSION; }
const char* dspb200_last_error(void) { return g_err; }
int64_t dspb200_launch_count(void) { return g_launches.load(); }

int dspb200_device_count(int* count) {
    DSP_REQUIRE(count != nullptr, "count is NULL");
    *count = 0;
    DSP_CUDA(cudaGetDeviceCount(count));
    return DSPB200_OK;
}

int dspb200_set_device(int device) {
    DSP_CUDA(cudaSetDevice(device));
    return DSPB200_OK;
}

int dspb200_device_info(int* sm_count, int* cc_major, int* cc_minor, size_t* total_mem, size_t* l2_bytes) {
    int dev = 0;
    DSP_CUDA(cudaGetDevice(&dev));
    cudaDeviceProp p;
    DSP_CUDA(cudaGetDeviceProperties(&p, dev));
    if (sm_count) *sm_count = p.multiProcessorCount;
    if (cc_major) *cc_major = p.major;
    if (cc_minor) *cc_minor = p.minor;
    if (total_mem) *total_mem = p.totalGlobalMem;
    if (l2_bytes) *l2_bytes = (size_t)p.l2CacheSize;
    return DSPB200_OK;
}

int dspb200_malloc(void** dptr, size_t bytes) {
    DSP_REQUIRE(dptr != nullptr, "dptr is NULL");
    *dptr = nullptr;
    if (bytes == 0) return DSPB200_OK;
    DSP_CUDA(cudaMalloc(dptr, bytes));
    return DSPB200_OK;
}
int dspb200_free(void* dptr) {
    if (dptr) DSP_CUDA(cudaFree(dptr));
    return DSPB200_OK;
}
int dspb200_host_alloc(void** hptr, size_t bytes) {
    DSP_REQUIRE(hptr != nullptr, "hptr is NULL");
    *hptr = nullptr;
    if (bytes == 0) return DSPB200_OK;
    DSP_CUDA(cudaHostAlloc(hptr, bytes, cudaHostAllocDefault));
    return DSPB200_OK;
}
int dspb200_host_free(void* hptr) {
    if (hptr) DSP_CUDA(cudaFreeHost(hptr));
    return DSPB200_OK;
}
int dspb200_memcpy_h2d(void* dst, const void* src, size_t bytes, void* stream) {
    if (bytes == 0) return DSPB200_OK;
    DSP_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    return DSPB200_OK;
}
int dspb200_memcpy_d2h(void* dst, const void* src, size_t bytes, void* stream) {
    if (bytes == 0) return DSPB200_OK;
    DSP_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    return DSPB200_OK;
}
int dspb200_memcpy2d_d2d(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t height, void* stream) {
    if (width == 0 || height == 0) return DSPB200_OK;
    DSP_REQUIRE(dst && src && dpitch >= width && spitch >= width, "NULL argument or a pitch below the row width");
    return memcpy2d_dd(dst, dpitch, src, spitch, width, height, (cudaStream_t)stream);
}
int dspb200_stream_sync(void* stream) {
    DSP_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return DSPB200_OK;
}

}  // extern "C"
