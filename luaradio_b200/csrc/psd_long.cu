// PSD of long frames, 8192 <= N <= 2^20 points (power of two): window -> DFT -> |X_k|^2 / scale [-> 10 log10], as the
// psd kernels of aux_blocks.cu compute it for N <= 4096.  tests/psd_long_ref.py models the decomposition in float32.
//
// Every transform is a Stockham autosort FFT held in shared memory: radix-16 passes, then one pass of the remaining
// radix (2, 4 or 8).  Each thread keeps 32 points in registers per pass; the window is applied at the load from HBM
// and |X|^2 / scale (in double, rounded once) at the store.
//   * N <= 16384: one CTA per frame, the whole frame in shared memory (132 KiB at N = 16384); one HBM pass.
//   * N >= 32768: four-step form N = N1 N2 through an HBM scratch buffer.  The column kernel transforms TILE / N1
//     adjacent columns x[n1 N2 + n2] over n1 and stores Y[k1][n2] W_N^(n2 k1); the row kernel transforms TILE / N2
//     adjacent rows over n2 and stores X[k1 + N1 k2], TILE / N2 consecutive k1 per k2.  A call runs in batches of
//     PSD_LONG_BATCH / N frames so that the scratch buffer stays at 256 MiB.
#include "blocks.h"

#include <cmath>
#include <vector>

namespace lrb {

namespace {

constexpr int PL_P = 32;                 // points per thread and pass
constexpr int PL_TILE = 8192;            // points per CTA of the two-pass form
enum { PL_SINGLE = 0, PL_COL = 1, PL_ROW = 2 };

__host__ __device__ constexpr int pl_npass(int L) { int n = 0; while (L >= 16) { L /= 16; ++n; } return n + (L > 1 ? 1 : 0); }
__host__ __device__ constexpr int pl_radix(int L, int p) { for (int i = 0; i < p; ++i) L /= 16; return L >= 16 ? 16 : L; }
__host__ __device__ constexpr int pl_span(int L, int p) { int s = 1; for (int i = 0; i < p; ++i) s *= pl_radix(L, i); return s; }
__host__ __device__ constexpr int pl_brev(int q, int R) { int r = 0; for (int b = 1; b < R; b <<= 1) { r = (r << 1) | (q & 1); q >>= 1; } return r; }
constexpr size_t pl_smem(int points) { return sizeof(float2) * (size_t)(points + points / 32); }

// one float2 of padding per 32: the radix-16 scatter of the first passes would otherwise hit one bank
__device__ __forceinline__ int pl_pad(int i) { return i + (i >> 5); }

// W_16^e, e < 8 (e is a compile-time constant after unrolling)
__device__ __forceinline__ float2 pl_w16(int e) {
    const float c1 = 0.92387953251128674f, s1 = 0.38268343236508978f, h = 0.70710678118654752f;
    switch (e) {
        case 1: return make_float2(c1, -s1);
        case 2: return make_float2(h, -h);
        case 3: return make_float2(s1, -c1);
        case 4: return make_float2(0.f, -1.f);
        case 5: return make_float2(-s1, -c1);
        case 6: return make_float2(-h, -h);
        default: return make_float2(-c1, -s1);
    }
}

// R-point DFT, radix-2 decimation in frequency: natural order in, bit-reversed order out.  One template level per
// stage (half-span H), so that every loop has a compile-time trip count and u stays in registers.
template <int R, int H = R / 2>
__device__ __forceinline__ void pl_dft(float2 (&u)[R]) {
#pragma unroll
    for (int b = 0; b < R; b += 2 * H) {
#pragma unroll
        for (int i = 0; i < H; ++i) {
            const float2 a = u[b + i], c = u[b + i + H];
            u[b + i] = fadd2(a, c);
            float2 d = fsub2(a, c);
            const int e = i * (8 / H);                            // W_(2H)^i = W_16^(i 8 / H)
            if (e == 4) d = make_float2(d.y, -d.x);
            else if (e != 0) d = cmul(d, pl_w16(e));
            u[b + i + H] = d;
        }
    }
    if constexpr (H > 1) pl_dft<R, H / 2>(u);
}

struct PlArgs {
    const void* in;           // SINGLE / COL: the frames (complex64 or float32); ROW: the scratch buffer
    void* out;                // SINGLE / ROW: the PSD (float32); COL: the scratch buffer
    const float* window;
    const float2* tw;         // W_L^m, m < L
    const float2* lo;         // COL: W_N^m, m < 1024
    const float2* hi;         // COL: W_N^(1024 m), m < N / 1024
    int N1, N2;               // COL / ROW: column length and row length (N1 N2 = N)
    int complex_in, logarithmic;
    double inv_scale;
};

// item t of a pass: (sequence c, butterfly j).  Consecutive threads take consecutive sequences (COL: adjacent columns,
// ROW: the k1 of one k2 at the store), except at the row kernel's load, where they walk along the row in HBM.
template <int L, int C, bool JFAST, int R>
__device__ __forceinline__ void pl_item(int t, int& c, int& j) {
    if (JFAST) { j = t % (L / R); c = t / (L / R); }
    else { c = t % C; j = t / C; }
}

template <int L, int C, int MODE>
__device__ __forceinline__ float2 pl_load_global(const PlArgs& a, long long f, int g, int c, int idx) {
    const long long N = (long long)a.N1 * a.N2;
    if (MODE == PL_ROW) return __ldcs(reinterpret_cast<const float2*>(a.in) + f * N + (long long)(g * C + c) * L + idx);
    const int n = MODE == PL_SINGLE ? idx : idx * a.N2 + g * C + c;
    const float w = __ldg(a.window + n);
    if (a.complex_in) {
        const float2 v = __ldcs(reinterpret_cast<const float2*>(a.in) + f * N + n);
        return make_float2(v.x * w, v.y * w);
    }
    return make_float2(__ldcs(reinterpret_cast<const float*>(a.in) + f * N + n) * w, 0.f);
}

template <int L, int C, int MODE>
__device__ __forceinline__ void pl_store_global(const PlArgs& a, long long f, int g, int c, int idx, float2 v) {
    const long long N = (long long)a.N1 * a.N2;
    if (MODE == PL_COL) {
        const int n2 = g * C + c, m = n2 * idx;                   // idx = k1; m < N
        v = cmul(cmul(v, __ldg(a.lo + (m & 1023))), __ldg(a.hi + (m >> 10)));
        __stcg(reinterpret_cast<float2*>(a.out) + f * N + (long long)idx * a.N2 + n2, v);
        return;
    }
    double p = ((double)v.x * v.x + (double)v.y * v.y) * a.inv_scale;
    if (a.logarithmic) p = 10.0 * log10(p);
    const long long k = MODE == PL_SINGLE ? idx : (long long)(g * C + c) + (long long)a.N1 * idx;
    __stcs(reinterpret_cast<float*>(a.out) + f * N + k, (float)p);
}

// pass PASS of the Stockham transform: twiddle, R-point DFT, scatter to shared memory (or the epilogue after the last
// pass), then gather the next pass's inputs
template <int L, int C, int MODE, int PASS>
__device__ __forceinline__ void pl_pass(const PlArgs& a, long long f, int g, float2 (&v)[PL_P], float2* sm) {
    constexpr int R = pl_radix(L, PASS), NS = pl_span(L, PASS), T = L * C / PL_P, IT = PL_P / R;
    constexpr bool LAST = PASS + 1 == pl_npass(L), JF = MODE == PL_ROW && PASS == 0;
#pragma unroll
    for (int it = 0; it < IT; ++it) {
        int c, j;
        pl_item<L, C, JF, R>(threadIdx.x + it * T, c, j);
        float2 u[R];
#pragma unroll
        for (int r = 0; r < R; ++r) u[r] = v[it * R + r];
        if (NS > 1) {
            const int k = j & (NS - 1);
#pragma unroll
            for (int r = 1; r < R; ++r) u[r] = cmul(u[r], __ldg(a.tw + k * r * (L / (NS * R))));
        }
        pl_dft<R>(u);
        const int base = (j / NS) * NS * R + (j & (NS - 1));
#pragma unroll
        for (int q = 0; q < R; ++q) {
            if (LAST) pl_store_global<L, C, MODE>(a, f, g, c, base + q * NS, u[pl_brev(q, R)]);
            else sm[pl_pad((base + q * NS) * C + c)] = u[pl_brev(q, R)];
        }
    }
    if constexpr (!LAST) {
        constexpr int R2 = pl_radix(L, PASS + 1), IT2 = PL_P / R2;
        __syncthreads();
#pragma unroll
        for (int it = 0; it < IT2; ++it) {
            int c, j;
            pl_item<L, C, false, R2>(threadIdx.x + it * T, c, j);
#pragma unroll
            for (int r = 0; r < R2; ++r) v[it * R2 + r] = sm[pl_pad((j + r * (L / R2)) * C + c)];
        }
        __syncthreads();                                          // in place: every gather is done before the next scatter
        pl_pass<L, C, MODE, PASS + 1>(a, f, g, v, sm);
    }
}

// SINGLE: one frame per CTA (C = 1); COL / ROW: tile blockIdx.x % tiles of frame blockIdx.x / tiles
template <int L, int C, int MODE>
__global__ void __launch_bounds__(L * C / PL_P, L * C / PL_P <= 256 ? 2 : 1)
psd_long_kernel(PlArgs a) {
    extern __shared__ __align__(16) float2 plsm[];
    constexpr int R0 = pl_radix(L, 0), T = L * C / PL_P;
    const int tiles = MODE == PL_SINGLE ? 1 : MODE == PL_COL ? a.N2 / C : a.N1 / C;
    const long long f = blockIdx.x / tiles;
    const int g = blockIdx.x % tiles;
    float2 v[PL_P];
#pragma unroll
    for (int it = 0; it < PL_P / R0; ++it) {
        int c, j;
        pl_item<L, C, MODE == PL_ROW, R0>(threadIdx.x + it * T, c, j);
#pragma unroll
        for (int r = 0; r < R0; ++r) v[it * R0 + r] = pl_load_global<L, C, MODE>(a, f, g, c, j + r * (L / R0));
    }
    pl_pass<L, C, MODE, 0>(a, f, g, v, plsm);
}

template <int L, int C, int MODE>
int pl_opt_in() {
    LRB_CHECK(cudaFuncSetAttribute(psd_long_kernel<L, C, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl_smem(L * C)));
    return 0;
}

template <int L, int C, int MODE>
void pl_launch(const PlArgs& a, long long ctas, cudaStream_t s) {
    psd_long_kernel<L, C, MODE><<<(unsigned)ctas, L * C / PL_P, pl_smem(L * C), s>>>(a);
}

void pl_table(std::vector<float2>& t, int L, long long N, long long stride) {
    for (long long m = 0; m < L; ++m) {
        const double ph = 2 * M_PI * (double)((m * stride) % N) / (double)N;
        t.push_back(make_float2((float)std::cos(ph), (float)(-std::sin(ph))));
    }
}

// N = N1 N2 with N2 = 2^ceil(log2(N) / 2)
void pl_split(int N, int* N1, int* N2) {
    int m = 0;
    while ((1 << m) < N) ++m;
    *N2 = 1 << ((m + 1) / 2);
    *N1 = N / *N2;
}

}  // namespace

int PsdLong::init(int N_) {
    N = N_;
    std::vector<float2> t;
    if (N <= PSD_LONG_SINGLE_MAX) {
        pl_table(t, N, N, 1);
        if (N == 8192 ? pl_opt_in<8192, 1, PL_SINGLE>() : pl_opt_in<16384, 1, PL_SINGLE>()) return -1;
    } else {
        int N1, N2;
        pl_split(N, &N1, &N2);
        pl_table(t, N1, N1, 1);                                   // W_N1^m
        pl_table(t, N2, N2, 1);                                   // W_N2^m
        pl_table(t, 1024, N, 1);                                  // W_N^m, m < 1024
        pl_table(t, N / 1024, N, 1024);                           // W_N^(1024 m)
        int rc = 0;
        switch (N1) {
            case 128: rc |= pl_opt_in<128, PL_TILE / 128, PL_COL>(); break;
            case 256: rc |= pl_opt_in<256, PL_TILE / 256, PL_COL>(); break;
            case 512: rc |= pl_opt_in<512, PL_TILE / 512, PL_COL>(); break;
            default: rc |= pl_opt_in<1024, PL_TILE / 1024, PL_COL>(); break;
        }
        switch (N2) {
            case 256: rc |= pl_opt_in<256, PL_TILE / 256, PL_ROW>(); break;
            case 512: rc |= pl_opt_in<512, PL_TILE / 512, PL_ROW>(); break;
            default: rc |= pl_opt_in<1024, PL_TILE / 1024, PL_ROW>(); break;
        }
        if (rc) return -1;
    }
    return d_tw.upload(t.data(), sizeof(float2) * t.size());
}

int PsdLong::run(const void* x, const float* window, float* y, long long frames, bool cplx, double inv_scale,
                 bool logarithmic, cudaStream_t s) {
    PlArgs a{};
    a.window = window;
    a.complex_in = cplx ? 1 : 0;
    a.logarithmic = logarithmic ? 1 : 0;
    a.inv_scale = inv_scale;
    const float2* tw = d_tw.as<const float2>();
    if (N <= PSD_LONG_SINGLE_MAX) {
        a.in = x; a.out = y; a.tw = tw; a.N1 = 1; a.N2 = N;
        if (N == 8192) pl_launch<8192, 1, PL_SINGLE>(a, frames, s);
        else pl_launch<16384, 1, PL_SINGLE>(a, frames, s);
        count_launch();
        LRB_CHECK(cudaGetLastError());
        return 0;
    }
    int N1, N2;
    pl_split(N, &N1, &N2);
    const long long batch = PSD_LONG_BATCH / N;
    const size_t need = sizeof(float2) * (size_t)N * (size_t)(frames < batch ? frames : batch);
    if (need > d_scratch.capacity()) {
        LRB_CHECK(cudaStreamSynchronize(s));                      // the old buffer may still be read by queued work
        if (d_scratch.reserve(need) != 0) return -1;
    }
    float2* scratch = d_scratch.as<float2>();
    const size_t esize = cplx ? sizeof(float2) : sizeof(float);
    a.N1 = N1; a.N2 = N2;
    for (long long f0 = 0; f0 < frames; f0 += batch) {
        const long long nb = frames - f0 < batch ? frames - f0 : batch;
        PlArgs c = a;
        c.in = static_cast<const char*>(x) + (size_t)f0 * N * esize;
        c.out = scratch;
        c.tw = tw;
        c.lo = tw + N1 + N2;
        c.hi = c.lo + 1024;
        const long long col_ctas = nb * (N2 / (PL_TILE / N1));
        switch (N1) {
            case 128: pl_launch<128, PL_TILE / 128, PL_COL>(c, col_ctas, s); break;
            case 256: pl_launch<256, PL_TILE / 256, PL_COL>(c, col_ctas, s); break;
            case 512: pl_launch<512, PL_TILE / 512, PL_COL>(c, col_ctas, s); break;
            default: pl_launch<1024, PL_TILE / 1024, PL_COL>(c, col_ctas, s); break;
        }
        PlArgs r = a;
        r.in = scratch;
        r.out = y + (size_t)f0 * N;
        r.tw = tw + N1;
        const long long row_ctas = nb * (N1 / (PL_TILE / N2));
        switch (N2) {
            case 256: pl_launch<256, PL_TILE / 256, PL_ROW>(r, row_ctas, s); break;
            case 512: pl_launch<512, PL_TILE / 512, PL_ROW>(r, row_ctas, s); break;
            default: pl_launch<1024, PL_TILE / 1024, PL_ROW>(r, row_ctas, s); break;
        }
        count_launch(2);
        LRB_CHECK(cudaGetLastError());
    }
    return 0;
}

}  // namespace lrb
