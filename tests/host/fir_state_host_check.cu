// Host-side emulation of the STATE instances of fir_tile_kernel (dsp.jl_b200/csrc/fir.cu, fir_tile.cuh; no GPU needed):
// the state seeding, staging, multiply-add rounds and routed stores are run for every "thread" of every CTA in turn, as
// the kernel sequences them between its barriers, over nx + nb - 1 outputs per column of a two-column signal.  The
// outputs AND the final state are compared BIT FOR BIT with the literal transposed direct-form loop of the reference
// with the state carried in and out (src/dspbase.jl:95-105).  Shared memory is poisoned with NaNs before every round.
// The newest tap's term enters the literal loop as muladd(x, b[nb], 0): for real eltypes that is the reference's product
// b[nb] * x (up to the sign of a zero); for complex eltypes it is the fused form the stateless kernel uses as well.
// A chunked pass (state handed from call to call) must equal the single pass exactly.
// Build (host compiler only): g++ -std=c++17 -O2 -march=native -x c++ -I/usr/local/cuda/include fir_state_host_check.cu
// (run by tests/test_df2t_fir.py)
#include "../../dsp.jl_b200/csrc/fir_tile.cuh"
#include <vector>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <limits>

using namespace dspb200;
namespace dspb200 { void set_error(const char*, ...) {} int cuda_fail(cudaError_t, const char*, const char*, int) { return -2; } void count_launch(int) {} int device_sm_count() { return 132; } }

static unsigned long long rng_state = 0x9E3779B97F4A7C15ULL;
static double rnd() {                                     // xorshift, uniform in (-1, 1)
    rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17;
    return (double)(rng_state >> 11) / (double)(1ULL << 53) * 2.0 - 1.0;
}
template <typename T> static void fill(T& v) { v = (T)rnd(); }
template <typename T> static void fill(cx<T>& v) { v.x = (T)rnd(); v.y = (T)rnd(); }
template <typename T> static void poison(T& v) { v = std::numeric_limits<T>::quiet_NaN(); }
template <typename T> static void poison(cx<T>& v) { v.x = v.y = std::numeric_limits<T>::quiet_NaN(); }

// the reference loop on one column: y[0 .. nx), state si (nb - 1 values) updated in place
template <typename E> static void df2t_literal(const E* b, int nb, const E* x, long long nx, E* si, E* y) {
    const int ns = nb - 1;
    const E zero = fir_zero((E*)nullptr);
    for (long long i = 0; i < nx; ++i) {
        const E xi = x[i];
        y[i] = fir_fma(xi, b[0], si[0]);
        for (int j = 0; j < ns - 1; ++j) si[j] = fir_fma(xi, b[j + 1], si[j + 1]);
        si[ns - 1] = fir_fma(xi, b[ns], zero);
    }
}

// one launch of fir_tile_kernel<E, NT, true> over ncols columns (x, out: nx per column; si_in, si_out: nb - 1 per column)
template <typename E, int NT>
static void kernel_state(const E* x, long long nx, int ncols, const E* b, int nb, E* out, const E* si_in, E* si_out) {
    using Gm = fir_geom<E, NT>;
    constexpr int G = Gm::G;
    E* xs = (E*)aligned_alloc(16, ((sizeof(E) * Gm::XS + 15) / 16) * 16);
    E* bs = (E*)aligned_alloc(16, sizeof(E) * Gm::KC);
    std::vector<E> acc((size_t)NT * G);
    const long long tiles = (nx + nb - 1 + Gm::TILE - 1) / Gm::TILE;
    const int nb8 = (nb + 7) & ~7;
    for (int col = 0; col < ncols; ++col)
        for (long long tile = 0; tile < tiles; ++tile) {
            const long long i0 = tile * Gm::TILE;
            const E* xc = x + (size_t)col * nx;
            E* oc = out + (size_t)col * nx;
            for (int tid = 0; tid < NT; ++tid) {
                E (&a)[G] = *reinterpret_cast<E (*)[G]>(&acc[(size_t)tid * G]);
                fir_state_init<E, G>(a, i0 + (long long)G * tid, si_in ? si_in + (size_t)col * (nb - 1) : nullptr, nb);
            }
            for (int k_hi = nb8 - 1; k_hi >= 0; k_hi -= Gm::KC) {
                const int kc = k_hi + 1 < Gm::KC ? k_hi + 1 : Gm::KC;
                for (int j = 0; j < Gm::XS; ++j) poison(xs[j]);
                for (int j = 0; j < Gm::KC; ++j) poison(bs[j]);
                for (int tid = 0; tid < NT; ++tid)
                    fir_stage<E, NT>(tid, xs, bs, xc, nx, i0 - k_hi, Gm::TILE + kc + 8, b, nb, k_hi, kc);
                for (int tid = 0; tid < NT; ++tid) {
                    E (&a)[G] = *reinterpret_cast<E (*)[G]>(&acc[(size_t)tid * G]);
                    fir_round<E, NT>(tid, a, xs, bs, nb, k_hi, kc);
                }
            }
            for (int tid = 0; tid < NT; ++tid) {
                const E (&a)[G] = *reinterpret_cast<const E (*)[G]>(&acc[(size_t)tid * G]);
                const long long i = i0 + (long long)G * tid;
                if (i + G <= nx) {                                   // the kernel's 128-bit store path
                    for (int o = 0; o < G; ++o) oc[i + o] = a[o];
                } else {
                    fir_state_store<E, G>(a, i, nx, nb, oc, si_out ? si_out + (size_t)col * (nb - 1) : nullptr);
                }
            }
        }
    free(xs); free(bs);
}

template <typename E> static int diff(const std::vector<E>& a, const std::vector<E>& b, const char* what, int nb, long long nx, int NT) {
    int bad = 0;
    for (size_t i = 0; i < a.size(); ++i)
        if (memcmp(&a[i], &b[i], sizeof(E)) != 0 && ++bad <= 3)
            printf("  %s mismatch: sizeof(E)=%d NT=%d nb=%d nx=%lld at %zu\n", what, (int)sizeof(E), NT, nb, nx, i);
    return bad;
}

template <typename E, int NT> static int run_case(int nb, long long nx, bool zero_state) {
    const int ncols = 2, ns = nb - 1;
    std::vector<E> x((size_t)nx * ncols), b(nb), si0((size_t)ns * ncols), ref((size_t)nx * ncols), sref(si0.size());
    for (auto& v : x) fill(v);
    for (auto& v : b) fill(v);
    for (auto& v : si0) { if (zero_state) v = fir_zero((E*)nullptr); else fill(v); }
    sref = si0;
    for (int c = 0; c < ncols; ++c) df2t_literal(b.data(), nb, &x[(size_t)c * nx], nx, &sref[(size_t)c * ns], &ref[(size_t)c * nx]);
    std::vector<E> y(x.size()), so(si0.size());
    for (auto& v : y) poison(v);
    for (auto& v : so) poison(v);
    kernel_state<E, NT>(x.data(), nx, ncols, b.data(), nb, y.data(), zero_state ? nullptr : si0.data(), so.data());
    return diff(y, ref, "output", nb, nx, NT) + diff(so, sref, "state", nb, nx, NT);
}

// one column in irregular chunks, the state of each call fed to the next: equal to the single pass
template <typename E, int NT> static int run_chunked(int nb, const std::vector<long long>& chunks) {
    const int ns = nb - 1;
    long long n = 0;
    for (long long c : chunks) n += c;
    std::vector<E> x(n), b(nb), si0(ns), ref(n), sref;
    for (auto& v : x) fill(v);
    for (auto& v : b) fill(v);
    for (auto& v : si0) fill(v);
    sref = si0;
    df2t_literal(b.data(), nb, x.data(), n, sref.data(), ref.data());
    std::vector<E> y(n), sa = si0, sb(ns);
    long long pos = 0;
    for (long long c : chunks) {
        kernel_state<E, NT>(x.data() + pos, c, 1, b.data(), nb, y.data() + pos, sa.data(), sb.data());
        sa.swap(sb);
        pos += c;
    }
    return diff(y, ref, "chunked output", nb, n, NT) + diff(sa, sref, "chunked state", nb, n, NT);
}

template <typename E, int NT> static int run_all(const char* name) {
    using Gm = fir_geom<E, NT>;
    static const int nbs[] = {2, 3, 7, 8, 9, 16, 17, 66, 67, 257, 511, 512, 513, 520, 1030};
    int bad = 0, cases = 0;
    for (int nb : nbs) {
        const long long nxs[] = {0, 1, nb - 2, nb - 1, nb, Gm::TILE - 1, 2 * Gm::TILE + 17};
        for (long long nx : nxs) {
            if ((long long)nb * (nx + nb) > 2000000) continue;     // keeps the whole check to a few seconds
            bad += run_case<E, NT>(nb, nx, false);
            ++cases;
        }
        bad += run_case<E, NT>(nb, Gm::TILE + 5, true);            // si_in == NULL: the zero state
        bad += run_chunked<E, NT>(nb, {0, 1, (long long)nb - 2, (long long)nb - 1, (long long)nb, 3, Gm::TILE + 9, 0, 2});
        cases += 2;
    }
    bad += run_case<E, NT>(1500, Gm::TILE + 40, false);            // three staging rounds
    printf("%s NT=%d: %d cases, %d mismatches\n", name, NT, cases + 1, bad);
    return bad;
}

int main() {
    int bad = 0;
    bad += run_all<float, 256>("Float32");
    bad += run_all<float, 128>("Float32");
    bad += run_all<double, 256>("Float64");
    bad += run_all<double, 128>("Float64");
    bad += run_all<cx<float>, 256>("ComplexF32");
    bad += run_all<cx<float>, 128>("ComplexF32");
    bad += run_all<cx<double>, 256>("ComplexF64");
    bad += run_all<cx<double>, 128>("ComplexF64");
    printf(bad ? "FAIL\n" : "OK\n");
    return bad ? 1 : 0;
}
