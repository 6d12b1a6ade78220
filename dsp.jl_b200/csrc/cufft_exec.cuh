// dspb200 -- cuFFT calls: error plumbing, plan types, batched 1-D plans and one dispatch for every transform.
#pragma once
#include "common.cuh"
#include <cufft.h>

namespace dspb200 {

int cufft_fail(cufftResult r, const char* what);
#define DSP_CUFFT(call)                                                    \
    do {                                                                   \
        cufftResult r__ = (call);                                          \
        if (r__ != CUFFT_SUCCESS) return ::dspb200::cufft_fail(r__, #call); \
    } while (0)

// The transform of complex (cplx) or real data in Float64 (f64) or Float32, direction CUFFT_FORWARD or CUFFT_INVERSE: complex
// data C2C / Z2Z either way, real data R2C / D2Z forward and C2R / Z2D inverse.
inline cufftType fft_type(bool cplx, bool f64, int dir) {
    if (cplx) return f64 ? CUFFT_Z2Z : CUFFT_C2C;
    if (dir == CUFFT_FORWARD) return f64 ? CUFFT_D2Z : CUFFT_R2C;
    return f64 ? CUFFT_Z2D : CUFFT_C2R;
}

// *h = a new plan of `batch` packed n-point 1-D transforms of that kind (0 when it fails)
int fft_plan_1d(cufftHandle* h, bool cplx, bool f64, int dir, int64_t n, int64_t batch);

// Queues plan h's transform of that kind from `in` to `out` on st and counts it as one launch.
int fft_exec(cufftHandle h, bool cplx, bool f64, int dir, const void* in, void* out, cudaStream_t st);

}  // namespace dspb200
