// dspb200 -- time-domain FIR: filt(b, 1, x) / tdfilt (src/dspbase.jl:26-66, 95-154; src/Filters/filt.jl:431-443).
//
// The reference runs a transposed direct-form loop whose state update is si[j] = muladd(x_i, b[j+1], si[j+1])
// (:95-105, and the unrolled NTuple form :118-141), which unrolls to
//     y[i] = fma(x[i], b[1], fma(x[i-1], b[2], ... fma(x[i-nb+2], b[nb-1], x[i-nb+1]*b[nb])))
// i.e. one fused multiply-add per tap, oldest tap first.  fir_tile_kernel (fir_tile.cuh: 8 outputs per thread, 8 taps per
// chunk, 128-bit loads) evaluates exactly that chain per output, so Float32/Float64 results match the reference bit for bit
// on FMA hardware.  It stages the x tile (+ tap-chunk halo) and the tap chunk in shared memory, padded so that the
// sliding-window reads are bank-conflict free.
//
// The stateful form (DF2TFilter / filt(b, 1, x, si), src/Filters/filt.jl:157-181, src/deprecated.jl:80-101) is the same
// kernel with STATE = true: in transposed direct form the FIR state is the partial chain of the next nb - 1 outputs, so
// the call evaluates outputs 0 .. nx + nb - 2 of the column, seeds outputs i < nb - 1 with si_in[i] and stores outputs
// nx + j as si_out[j].  Filtering in chunks is therefore bit-identical to filtering in one call.
#include "common.cuh"
#include "fir_tile.cuh"
#include <new>

namespace dspb200 {

template <typename T, bool CPLX> struct fir_elt { using type = T; };
template <typename T> struct fir_elt<T, true> { using type = cx<T>; };

// ---------------------------------------------------------------------------------------------- register-tiled kernel
// fir_tile.cuh: a thread owns G consecutive outputs, 8 taps per chunk, two 8-sample register runs that swap roles.
// STATE (DF2TFilter, filt(b, a, x, si)): a column has nx + nb - 1 outputs; outputs i < nb - 1 start their chain from
// si_in[i], outputs i >= nx are the final state si_out[i - nx] (fir_tile.cuh, fir_state_init / fir_state_store).
// si_in / si_out hold nb - 1 elements per column and may be NULL (zero state / state not wanted).  The STATE instances ask
// for one resident CTA per SM at least: without that bound ptxas keeps the ComplexF32 256-thread instance at 64 registers
// and spills the state pointers.
template <typename E, int NT, bool STATE>
__global__ void __launch_bounds__(NT, STATE ? 1 : 0)
fir_tile_kernel(const E* __restrict__ x, int64_t nx, int64_t tiles_per_col, const E* __restrict__ b, int nb,
                E* __restrict__ out, const E* __restrict__ si_in, E* __restrict__ si_out) {
    using Gm = fir_geom<E, NT>;
    constexpr int G = Gm::G;
    __shared__ __align__(16) E xs[Gm::XS];
    __shared__ __align__(16) E bs[Gm::KC];
    const int tid = threadIdx.x;
    const int64_t col = blockIdx.x / tiles_per_col;
    const int64_t tile = blockIdx.x % tiles_per_col;
    const int64_t i0 = tile * Gm::TILE;
    const E* xc = x + col * nx;
    E* oc = out + col * nx;
    E acc[G];
    if constexpr (STATE) {
        fir_state_init<E, G>(acc, i0 + (int64_t)G * tid, si_in ? si_in + col * (nb - 1) : nullptr, nb);
    } else {
#pragma unroll
        for (int o = 0; o < G; ++o) acc[o] = fir_zero((E*)nullptr);
    }
    const int nb8 = (nb + 7) & ~7;                                      // taps nb .. nb8-1 are padding (skipped)
    for (int k_hi = nb8 - 1; k_hi >= 0; k_hi -= Gm::KC) {
        const int kc = k_hi + 1 < Gm::KC ? k_hi + 1 : Gm::KC;           // padded taps k_hi, k_hi-1, .., k_hi-kc+1 (a multiple of 8)
        __syncthreads();
        fir_stage<E, NT>(tid, xs, bs, xc, nx, i0 - k_hi, Gm::TILE + kc + 8, b, nb, k_hi, kc);
        __syncthreads();
        fir_round<E, NT>(tid, acc, xs, bs, nb, k_hi, kc);
    }
    const int64_t i = i0 + (int64_t)G * tid;
    if (i + G <= nx && (reinterpret_cast<uintptr_t>(oc + i) & 15) == 0) {
#pragma unroll
        for (int v = 0; v < G; v += Gm::VEC) *reinterpret_cast<uint4*>(oc + i + v) = *reinterpret_cast<const uint4*>(&acc[v]);
    } else if constexpr (STATE) {
        fir_state_store<E, G>(acc, i, nx, nb, oc, si_out ? si_out + col * (nb - 1) : nullptr);
    } else {
#pragma unroll
        for (int o = 0; o < G; ++o)
            if (i + o < nx) oc[i + o] = acc[o];
    }
}

// 128-thread tiles when the 256-thread grid would not cover every SM eight times over, so short inputs still spread
// over the whole GPU.  nout = outputs per column (nx, or nx + nb - 1 with STATE).
template <typename E, bool STATE>
static int fir_launch(const E* x, int64_t nx, int64_t nout, int64_t ncols, const E* b, int nb, E* out, const E* si_in, E* si_out,
                      cudaStream_t st) {
    const bool small = cdiv(nout, fir_geom<E, 256>::TILE) * ncols < (int64_t)8 * device_sm_count();
    const int64_t tiles = cdiv(nout, small ? fir_geom<E, 128>::TILE : fir_geom<E, 256>::TILE), blocks = tiles * ncols;
    DSP_REQUIRE(blocks < (int64_t)0x7fffffff, "too many tiles for one launch");
    if (small) fir_tile_kernel<E, 128, STATE><<<(unsigned)blocks, 128, 0, st>>>(x, nx, tiles, b, nb, out, si_in, si_out);
    else fir_tile_kernel<E, 256, STATE><<<(unsigned)blocks, 256, 0, st>>>(x, nx, tiles, b, nb, out, si_in, si_out);
    DSP_LAUNCH_OK();
    return DSPB200_OK;
}

template <bool STATE>
static int fir_dispatch(int dtype, const void* x, int64_t nx, int64_t nout, int64_t ncols, const void* b, int nb, void* out,
                        const void* si_in, void* si_out, cudaStream_t st) {
#define FIR_CALL(E_) fir_launch<E_, STATE>((const E_*)x, nx, nout, ncols, (const E_*)b, nb, (E_*)out, (const E_*)si_in, (E_*)si_out, st)
    switch (dtype) {
        case DSPB200_F32: return FIR_CALL(float);
        case DSPB200_F64: return FIR_CALL(double);
        case DSPB200_C32: return FIR_CALL(cx<float>);
        default: return FIR_CALL(cx<double>);
    }
#undef FIR_CALL
}

struct FirPlanImpl {
    int dtype = 0;
    int64_t nb = 0;
    int device = 0;
    void* d_b = nullptr;
    DevBuf in, out, si_in, si_out;
    cudaStream_t s_exec = nullptr;
};

// makes the plan's device current and creates its stream on first use
static int ensure_streams(FirPlanImpl* p) {
    DSP_CUDA(cudaSetDevice(p->device));
    return ensure_stream(&p->s_exec);
}

}  // namespace dspb200

using namespace dspb200;

struct dspb200_fir_plan {
    FirPlanImpl impl;
};

extern "C" {

int dspb200_fir_plan_create(dspb200_fir_plan** plan, int dtype, const void* b_host, int64_t nb) {
    DSP_RANGE("dspb200_fir_plan_create");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    *plan = nullptr;
    DSP_REQUIRE(dtype_valid(dtype), "invalid dtype %d", dtype);
    DSP_REQUIRE(b_host != nullptr && nb >= 1, "filter vector b must be non-empty");   // ArgumentError src/dspbase.jl:28
    DSP_REQUIRE(nb < (int64_t(1) << 30), "filter too long");
    dspb200_fir_plan* h = new (std::nothrow) dspb200_fir_plan();
    DSP_REQUIRE(h != nullptr, "out of host memory");
    FirPlanImpl* p = &h->impl;
    p->dtype = dtype; p->nb = nb;
    const cudaError_t e = cudaGetDevice(&p->device);
    const int rc = e != cudaSuccess ? cuda_fail(e, "cudaGetDevice", __FILE__, __LINE__) : upload(&p->d_b, b_host, (size_t)nb * dtype_size(dtype));
    if (rc != DSPB200_OK) { dspb200_fir_plan_destroy(h); return rc; }
    *plan = h;
    return DSPB200_OK;
}

int dspb200_fir_exec_dev(dspb200_fir_plan* plan, const void* x, int64_t nx, int64_t ncols, void* out, void* stream) {
    DSP_RANGE("dspb200_fir_exec_dev");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    DSP_REQUIRE(nx >= 0 && ncols >= 0, "negative size");
    if (nx == 0 || ncols == 0) return DSPB200_OK;
    DSP_REQUIRE(x && out, "NULL argument");
    FirPlanImpl* p = &plan->impl;
    return fir_dispatch<false>(p->dtype, x, nx, nx, ncols, p->d_b, (int)p->nb, out, nullptr, nullptr, (cudaStream_t)stream);
}

int dspb200_fir_exec_state_dev(dspb200_fir_plan* plan, const void* x, int64_t nx, int64_t ncols, const void* si_in, void* si_out,
                               void* out, void* stream) {
    DSP_RANGE("dspb200_fir_exec_state_dev");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    FirPlanImpl* p = &plan->impl;
    const int64_t ns = p->nb - 1;
    cudaStream_t st = (cudaStream_t)stream;
    DSP_TRY(state_prologue_dev(x, nx, ncols, si_in, si_out, out, ns, dtype_size(p->dtype), st));
    if (nx == 0 || ncols == 0) return DSPB200_OK;
    if (ns == 0)                                                         // nb == 1: no state, out = x * b[1] (src/Filters/filt.jl:161-162)
        return fir_dispatch<false>(p->dtype, x, nx, nx, ncols, p->d_b, 1, out, nullptr, nullptr, st);
    return fir_dispatch<true>(p->dtype, x, nx, nx + ns, ncols, p->d_b, (int)p->nb, out, si_in, si_out, st);
}

int dspb200_fir_exec_state(dspb200_fir_plan* plan, const void* x, int64_t nx, int64_t ncols, const void* si_in, void* si_out,
                           void* out) {
    DSP_RANGE("dspb200_fir_exec_state");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    FirPlanImpl* p = &plan->impl;
    return exec_state_host(p, p->s_exec, x, nx, ncols, si_in, si_out, out, p->nb - 1, dtype_size(p->dtype), p->in, p->out, p->si_in,
                           p->si_out, [&](const void* d_x, const void* d_si_in, void* d_si_out, void* d_out) {
                               return dspb200_fir_exec_state_dev(plan, d_x, nx, ncols, d_si_in, d_si_out, d_out, p->s_exec);
                           });
}

int dspb200_fir_exec(dspb200_fir_plan* plan, const void* x, int64_t nx, int64_t ncols, void* out) {
    DSP_RANGE("dspb200_fir_exec");
    DSP_REQUIRE(plan != nullptr, "plan is NULL");
    DSP_REQUIRE(nx >= 0 && ncols >= 0, "negative size");
    if (nx == 0 || ncols == 0) return DSPB200_OK;
    DSP_REQUIRE(x && out, "NULL argument");
    FirPlanImpl* p = &plan->impl;
    DSP_TRY(ensure_streams(p));
    const size_t bytes = (size_t)(nx * ncols) * dtype_size(p->dtype);
    return run_staged(p->s_exec, {{x, bytes, &p->in}}, {{out, bytes, &p->out}},
                      [&] { return dspb200_fir_exec_dev(plan, p->in.p, nx, ncols, p->out.p, p->s_exec); });
}

int dspb200_fir_plan_destroy(dspb200_fir_plan* plan) {
    if (!plan) return DSPB200_OK;
    FirPlanImpl* p = &plan->impl;
    if (p->d_b) cudaFree(p->d_b);
    p->in.release(); p->out.release(); p->si_in.release(); p->si_out.release();
    if (p->s_exec) cudaStreamDestroy(p->s_exec);
    delete plan;
    return DSPB200_OK;
}

}  // extern "C"
