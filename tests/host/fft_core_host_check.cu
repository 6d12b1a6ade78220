// Host-side emulation of the shared-memory FFT core (no GPU needed): every pass of the forward transform and of the
// overlap-save pipeline (first | middle | [last, x H, swap, first] | middle | last) is run for all "threads"
// sequentially, exactly as the kernels sequence them between barriers, and compared with a double-precision FFT;
// the padded layout is audited for bank conflicts of the scattered first-pass stores.
// Build (host compiler only): g++ -std=c++17 -O2 -x c++ -I/usr/local/cuda/include fft_core_host_check.cu
// (run by tests/test_host_fft.py)
#ifndef __CUDACC__
static inline void __syncthreads() {}
#endif
#include "../../dsp.jl_b200/csrc/fft_core.cuh"
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

template <typename T, int N> struct Emu {
    using P = fft_plan_traits<N>;
    static constexpr int NT = fft_threads<N>::value;
    static constexpr int Q = P::Q;
    static constexpr int ITERS = (Q + NT - 1) / NT;
    std::vector<cx<T>> sm, t16, t256, tl;
    FftCtx<T> ctx;
    Emu() : sm(padded_len<T>(N)), t16(fft_tw16_len(N)), t256(fft_tw256_len(N)), tl(fft_tl_len<N>() + 1) {
        fft_fill_tables<T>(t16.data(), t256.data(), N);
        fft_fill_tl<T>(tl.data(), N);
        if ((long long)fft_tl_len<N>() != fft_tl_len_rt(N)) { printf("tl length mismatch N=%d\n", N); exit(2); }
        ctx.sm = sm.data(); ctx.t16 = t16.data(); ctx.t256 = t256.data(); ctx.tl = tl.data();
    }
    // the passes between the first and the last one, every "thread" in turn, as fft_middle sequences them
    void middle() {
        if constexpr (P::NMID >= 1) for (int tid = 0; tid < NT; ++tid) fft_pass16<T, N, NT, 16>(ctx, tid);
        if constexpr (P::NMID == 2) for (int tid = 0; tid < NT; ++tid) fft_pass16<T, N, NT, 256>(ctx, tid);
    }
    // forward: x natural -> X natural
    void forward(const std::vector<cx<T>>& x, std::vector<cx<T>>& X) {
        auto ld0 = [&](int j, int, int) { return x[j]; };
        for (int tid = 0; tid < NT; ++tid) fft_first_pass<T, N, NT, false>(ctx, tid, ld0);
        middle();
        for (int tid = 0; tid < NT; ++tid)
            for (int it = 0; it < ITERS; ++it) {
                const int tp = tid + it * NT;
                if (tp >= Q) break;
                cx<T> v[16];
                fft_last_pass<T, N>(ctx, tp, v);
                for (int r = 0; r < 16; ++r) X[tp + r * Q] = v[r];
            }
    }
    // overlap-save pipeline: y = N * ifft(fft(x) .* h) through the fused bracket [last, x H, swap, first]
    void convolve(const std::vector<cx<T>>& x, const std::vector<cx<T>>& H, std::vector<cx<T>>& y) {
        auto ld0 = [&](int j, int, int) { return x[j]; };
        for (int tid = 0; tid < NT; ++tid) fft_first_pass<T, N, NT, false>(ctx, tid, ld0);
        middle();
        std::vector<cx<T>> regs((size_t)Q * 16);
        for (int tp = 0; tp < Q; ++tp) {                 // phase A (registers), then the barrier, then phase B
            cx<T> v[16];
            fft_last_pass<T, N>(ctx, tp, v);
            for (int r = 0; r < 16; ++r) v[r] = cswap(cmul(v[r], H[tp + r * Q]));
            fft_bfly16_plain<T>(v);
            for (int r = 0; r < 16; ++r) regs[(size_t)tp * 16 + r] = v[r];
        }
        for (int tp = 0; tp < Q; ++tp) {
            cx<T> v[16];
            for (int r = 0; r < 16; ++r) v[r] = regs[(size_t)tp * 16 + r];
            fft_store_block<T, N>(ctx.sm, tp, v);
        }
        middle();
        for (int tp = 0; tp < Q; ++tp) {
            cx<T> v[16];
            fft_last_pass<T, N>(ctx, tp, v);
            for (int r = 0; r < 16; ++r) y[tp + r * Q] = cswap(v[r]);
        }
    }
};

// bank-conflict audit of the scattered first-pass stores: lanes c .. c+7 of a quarter warp write 16-byte chunks
template <typename T, int N> static int scatter_wavefronts() {
    constexpr int Q = fft_plan_traits<N>::Q;
    int worst = 1;
    for (int c0 = 0; c0 + 8 <= Q; c0 += 8) {
        int cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int l = 0; l < 8; ++l) {
            const long long byte = (long long)padaddr<T, N>(16 * fft_block_of<N>(c0 + l)) * (long long)sizeof(cx<T>);
            cnt[(byte / 16) % 8]++;
        }
        for (int g = 0; g < 8; ++g) if (cnt[g] > worst) worst = cnt[g];
    }
    return worst;
}

template <typename T, int N> static int check(double tol) {
    Emu<T, N>* e = new Emu<T, N>();
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
    // circular convolution through the fused pipeline against the double-precision one
    e->forward(h, H);
    for (int k = 0; k < N; ++k) H[k] = cscale(H[k], T(1) / T(N));
    e->convolve(x, H, y);
    std::vector<cd> Hr = hr, Yr(N);
    ref_fft(Hr, false);
    for (int k = 0; k < N; ++k) Yr[k] = Xr[k] * Hr[k];
    ref_fft(Yr, true);
    num = den = 0;
    for (int j = 0; j < N; ++j) {
        num += std::norm(cd((double)y[j].x, (double)y[j].y) - Yr[j] / (double)N);
        den += std::norm(Yr[j] / (double)N);
    }
    const double ec = std::sqrt(num / den);
    const int wf = scatter_wavefronts<T, N>();
    const bool ok = ef < tol && ec < 2 * tol && wf == 1;
    printf("N=%5d %s  forward relerr %.3e  conv relerr %.3e  scatter-store wavefronts/quarter-warp %d  %s\n", N,
           sizeof(T) == 4 ? "f32" : "f64", ef, ec, wf, ok ? "ok" : "FAIL");
    delete e;
    return ok ? 0 : 1;
}

int main() {
    int bad = 0;
    bad += check<float, 32>(5e-7);
    bad += check<float, 64>(5e-7);
    bad += check<float, 128>(5e-7);
    bad += check<float, 256>(5e-7);
    bad += check<float, 512>(5e-7);
    bad += check<float, 1024>(5e-7);
    bad += check<float, 2048>(5e-7);
    bad += check<float, 4096>(5e-7);
    bad += check<float, 8192>(5e-7);
    bad += check<float, 16384>(5e-7);
    bad += check<double, 256>(1e-15);
    bad += check<double, 1024>(1e-15);
    bad += check<double, 2048>(1e-15);
    bad += check<double, 4096>(1e-15);
    bad += check<double, 8192>(1e-15);
    printf(bad ? "FAILED\n" : "ALL OK\n");
    return bad;
}
