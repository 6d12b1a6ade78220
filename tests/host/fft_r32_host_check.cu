// Host-side emulation of the 32 · 32 · 16 plan of the 16384-point Float32 overlap-save kernels (fft_r32 in fft_core.cuh;
// no GPU needed): the forward transform and the overlap-save pipeline  first | radix-32 | [last, x H, swap, first] |
// radix-32 | last  run for all "threads" sequentially, exactly as os_unit_r32 sequences them between barriers, and are
// compared with a double-precision FFT; every shared-memory access of the plan is audited for bank conflicts, and the
// layout's padding must be the smallest conflict-free one.
// Build (host compiler only): g++ -std=c++17 -O2 -x c++ -I/usr/local/cuda/include fft_r32_host_check.cu
// (run by tests/test_host_fft_r32.py)
#ifndef __CUDACC__
static inline void __syncthreads() {}
#endif
#include "../../dsp.jl_b200/csrc/fft_core.cuh"
#include <algorithm>
#include <complex>
#include <vector>
#include <cstdio>
#include <cmath>
#include <cstdlib>

using namespace dspb200;
namespace dspb200 { void set_error(const char*, ...) {} int cuda_fail(cudaError_t, const char*, const char*, int) { return -2; } void count_launch(int) {} int device_sm_count() { return 132; } }

typedef std::complex<double> cd;

static void ref_fft(std::vector<cd>& a, bool inv) {   // iterative radix-2, double
    const size_t n = a.size();
    for (size_t i = 1, j = 0; i < n; ++i) {
        size_t bit = n >> 1;
        for (; j & bit; bit >>= 1) j ^= bit;
        j ^= bit;
        if (i < j) std::swap(a[i], a[j]);
    }
    for (size_t len = 2; len <= n; len <<= 1) {
        const double ang = 2 * M_PI / (double)len * (inv ? 1 : -1);
        for (size_t i = 0; i < n; i += len)
            for (size_t k = 0; k < len / 2; ++k) {
                cd w = std::polar(1.0, ang * (double)k);
                cd u = a[i + k], v = a[i + k + len / 2] * w;
                a[i + k] = u + v; a[i + k + len / 2] = u - v;
            }
    }
}

// The 32 · 32 · 16 plan of the 16384-point Float32 overlap-save kernels (fft_r32), sequenced as os_unit runs it: a thread
// owns first-pass residue class tid, middle butterfly tid and last-pass butterflies tid, tid + 512.
struct EmuR32 {
    using T = float;
    static constexpr int N = fft_r32::N, NT = fft_r32::NT, Q = fft_r32::Q;
    std::vector<cx<T>> sm, tab;
    FftR32Ctx<T> ctx;
    EmuR32() : sm(fft_r32::PADDED_LEN), tab(fft_r32::TABLE_LEN) {
        fft_r32_fill_tables<T>(tab.data());
        ctx = FftR32Ctx<T>{sm.data(), tab.data(), tab.data() + fft_r32::T32_LEN};
    }
    void first(const std::vector<cx<T>>& x) {
        for (int tid = 0; tid < NT; ++tid) {
            cx<T> v[32];
            for (int m = 0; m < 32; ++m) v[m] = x[tid + Q * m];
            fft_r32_first_bfly<T>(v);
            fft_r32_store_block<T>(ctx.sm, tid, v);
        }
    }
    void middle() { for (int tid = 0; tid < NT; ++tid) fft_r32_middle<T>(ctx, tid); }
    void last(std::vector<cx<T>>& X) {
        for (int t = 0; t < fft_r32::QL; ++t) {
            cx<T> v[16];
            fft_r32_last_load<T>(ctx, t, v);
            fft_r32_last_bfly<T>(ctx, t, v);
            for (int s = 0; s < 16; ++s) X[t + 1024 * s] = v[s];
        }
    }
    void forward(const std::vector<cx<T>>& x, std::vector<cx<T>>& X) { first(x); middle(); last(X); }
    void convolve(const std::vector<cx<T>>& x, const std::vector<cx<T>>& H, std::vector<cx<T>>& y) {
        first(x);
        middle();
        std::vector<cx<T>> regs((size_t)NT * 32);
        for (int tid = 0; tid < NT; ++tid) {            // phase A (registers), then the barrier, then phase B
            cx<T> v[2][16], z[32];
            for (int it = 0; it < 2; ++it) {
                fft_r32_last_load<T>(ctx, tid + it * NT, v[it]);
                fft_r32_last_bfly<T>(ctx, tid + it * NT, v[it]);
            }
            for (int m = 0; m < 32; ++m) z[m] = cswap(cmul(v[m & 1][m >> 1], H[tid + Q * m]));
            fft_r32_first_bfly<T>(z);
            for (int m = 0; m < 32; ++m) regs[(size_t)tid * 32 + m] = z[m];
        }
        for (int tid = 0; tid < NT; ++tid) {
            cx<T> z[32];
            for (int m = 0; m < 32; ++m) z[m] = regs[(size_t)tid * 32 + m];
            fft_r32_store_block<T>(ctx.sm, tid, z);
        }
        middle();
        last(y);
        for (auto& v : y) v = cswap(v);
    }
};

// Bank audit of every shared-memory access of the 32 · 32 · 16 plan for a padding C: the worst number of wavefronts a
// half warp (8-byte accesses) or a quarter warp (16-byte accesses) needs.  128 bytes = 16 complex Float32 per wavefront.
static int r32_wavefronts(int C) {
    auto addr = [&](int p) { return p + C * (p >> 10); };
    auto groups = [](const long long* byte, int lanes, int width) {    // distinct `width`-byte accesses per bank set
        int cnt[32] = {0};
        int worst = 0;
        for (int l = 0; l < lanes; ++l)
            for (int b = 0; b < width / 4; ++b) worst = std::max(worst, ++cnt[(byte[l] / 4 + b) % 32]);
        return worst;
    };
    int worst = 1;
    long long byte[16];
    // first-pass / bracket stores: 16-byte pairs of residue classes c .. c+7
    for (int c0 = 0; c0 < fft_r32::Q; c0 += 8)
        for (int r = 0; r < 32; r += 2) {
            for (int l = 0; l < 8; ++l) byte[l] = 8LL * addr(32 * fft_r32_block_of(c0 + l) + r);
            worst = std::max(worst, groups(byte, 8, 16));
        }
    // radix-32 pass: butterflies tid .. tid+15, operand r
    for (int t0 = 0; t0 < fft_r32::Q; t0 += 16)
        for (int r = 0; r < 32; ++r) {
            for (int l = 0; l < 16; ++l) { const int b = t0 + l; byte[l] = 8LL * addr((b >> 5) * 1024 + (b & 31) + 32 * r); }
            worst = std::max(worst, groups(byte, 16, 8));
        }
    // last pass: butterflies t .. t+15, operand s
    for (int t0 = 0; t0 < fft_r32::QL; t0 += 16)
        for (int s = 0; s < 16; ++s) {
            for (int l = 0; l < 16; ++l) byte[l] = 8LL * addr(t0 + l + 1024 * s);
            worst = std::max(worst, groups(byte, 16, 8));
        }
    return worst;
}

static int check_r32(double tol) {
    // the layout constant is the smallest conflict-free padding (even: 16-byte aligned runs)
    int cmin = -1;
    for (int C = 0; C <= 16 && cmin < 0; C += 2) if (r32_wavefronts(C) == 1) cmin = C;
    EmuR32* e = new EmuR32();
    constexpr int N = fft_r32::N;
    using T = float;
    std::vector<cx<T>> x(N), X(N), h(N), H(N), y(N);
    std::vector<cd> xr(N), hr(N);
    srand(1234 + N);
    for (int j = 0; j < N; ++j) {
        double a = rand() / (double)RAND_MAX - 0.5, b = rand() / (double)RAND_MAX - 0.5;
        x[j] = mkc<T>((T)a, (T)b);
        xr[j] = cd((double)x[j].x, (double)x[j].y);
        a = rand() / (double)RAND_MAX - 0.5; b = rand() / (double)RAND_MAX - 0.5;
        h[j] = (j < N / 4 + 1) ? mkc<T>((T)a, (T)b) : mkc<T>(T(0), T(0));
        hr[j] = cd((double)h[j].x, (double)h[j].y);
    }
    e->forward(x, X);
    std::vector<cd> Xr = xr;
    ref_fft(Xr, false);
    double num = 0, den = 0;
    for (int k = 0; k < N; ++k) {
        num += std::norm(cd((double)X[k].x, (double)X[k].y) - Xr[k]);
        den += std::norm(Xr[k]);
    }
    const double ef = std::sqrt(num / den);
    // H = FFT(h) / N from the double-precision FFT, rounded once, then the 32 · 32 · 16 pipeline
    std::vector<cd> Hr = hr, Yr(N);
    ref_fft(Hr, false);
    for (int k = 0; k < N; ++k) H[k] = mkc<T>((T)(Hr[k].real() / N), (T)(Hr[k].imag() / N));
    e->convolve(x, H, y);
    for (int k = 0; k < N; ++k) Yr[k] = Xr[k] * Hr[k];
    ref_fft(Yr, true);
    num = den = 0;
    for (int j = 0; j < N; ++j) {
        num += std::norm(cd((double)y[j].x, (double)y[j].y) - Yr[j] / (double)N);
        den += std::norm(Yr[j] / (double)N);
    }
    const double ec = std::sqrt(num / den);
    const int wf = r32_wavefronts(fft_r32::C10);
    const bool ok = ef < tol && ec < 2 * tol && wf == 1 && cmin == fft_r32::C10;
    printf("N=%5d f32 32x32x16  forward relerr %.3e  conv relerr %.3e  wavefronts/access %d (C10 %d, smallest %d)  %s\n", N, ef,
           ec, wf, fft_r32::C10, cmin, ok ? "ok" : "FAIL");
    delete e;
    return ok ? 0 : 1;
}

int main() {
    const int bad = check_r32(5e-7);
    printf(bad ? "FAILED\n" : "ALL OK\n");
    return bad;
}
