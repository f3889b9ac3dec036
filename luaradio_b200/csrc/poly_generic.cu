// Generic-shape polyphase decimating FIR: any tap count (up to the parameter-bank budget), decimation factor from a
// templated list, complex or real input, real or complex taps.  The catch-all `fir_generic_kernel` computes one output
// per thread with one L1 load per MAC; this kernel is the register-tiled form for every DecimatorBlock / decimating
// FIRFilterBlock shape that has no hand-unrolled instantiation in tuner.cu (composites/decimator.lua:34-41 with any
// factor, firfilter.lua:111-163 followed by downsampler.lua:40-56).
//
// Only kept outputs are computed.  A CTA stages (TO + Qn - 1) * D input samples in natural order in shared memory
// (Qn = ceil(M / D) tap blocks; thread stride padded to an odd number of elements: conflict-free), each thread owns R
// consecutive outputs and walks the window blocks jb = 0 .. R + Qn - 2: the D samples of block jb are loaded once and feed
// every output r with tap block q = jb - r.  The tap index is warp-uniform, so the taps come from the kernel-parameter
// constant bank through the uniform datapath (no shared-memory or L1 traffic for taps); the loop over jb is a run-time
// loop, the r x p nest is unrolled.
#include "common.cuh"

#include <cstring>

namespace lrb {

namespace {

constexpr int PG_THREADS = 128;
constexpr int PG_R = 8;
constexpr int PG_TO = PG_THREADS * PG_R;
constexpr int PG_MAXT = 960;                 // taps incl. zero padding to a whole number of blocks (floats; complex taps use 2)

struct GenParams {
    float hr[PG_MAXT];           // reversed taps, zero padded at the front to Qn*D (complex taps: interleaved re, im)
    long long first;             // input index of output 0
    long long n, n_out;
    int Qn, Hm1;
};

template <typename T> struct Elem;
template <> struct Elem<float2> {
    static __device__ __forceinline__ float2 zero() { return make_float2(0.f, 0.f); }
    static __device__ __forceinline__ void mac(float2& a, float2 v, float h) { a = ffma2(v, make_float2(h, h), a); }
    static __device__ __forceinline__ void macc(float2& a, float2 v, float hx, float hy) {
        a = ffma2(v, make_float2(hx, hx), a);
        a = ffma2(make_float2(-v.y, v.x), make_float2(hy, hy), a);
    }
};
template <> struct Elem<float> {
    static __device__ __forceinline__ float zero() { return 0.f; }
    static __device__ __forceinline__ void mac(float& a, float v, float h) { a = fmaf(v, h, a); }
    static __device__ __forceinline__ void macc(float&, float, float, float) {}
};

template <int D>
struct PgLayout {
    static constexpr int RD = PG_R * D;
    static constexpr int PADE = (RD % 2 == 0) ? 1 : 0;       // odd thread stride
    __host__ __device__ static constexpr int pad(int e) { return e + PADE * (e / RD); }
    __host__ static size_t smem_elems(int Qn) { return (size_t)pad((PG_TO + Qn) * D) + 2; }
};

template <typename T, int D, bool CTAPS>
__global__ void __launch_bounds__(PG_THREADS)
poly_generic_kernel(const T* __restrict__ x, const T* __restrict__ hist, T* __restrict__ y, const __grid_constant__ GenParams P) {
    using L = PgLayout<D>;
    using E = Elem<T>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T* S = reinterpret_cast<T*>(smem_raw);
    const int tid = threadIdx.x;
    const int Qn = P.Qn;
    const long long tile = blockIdx.x;
    const long long B = P.first + tile * (long long)(PG_TO * D) - (long long)(Qn * D - 1);   // input index of element 0
    const int span = (PG_TO + Qn - 1) * D;
    // ---- stage (guarded: history before the call, zeros after its end)
    const bool interior = B >= 0 && B + span <= P.n;
    if (interior) {
        for (int e = tid; e < span; e += PG_THREADS) S[L::pad(e)] = __ldg(x + B + e);
    } else {
        for (int e = tid; e < span; e += PG_THREADS) {
            const long long i = B + e;
            T v = E::zero();
            if (i >= 0) { if (i < P.n) v = __ldg(x + i); }
            else if (P.Hm1 + i >= 0) v = __ldg(hist + (P.Hm1 + i));
            S[L::pad(e)] = v;
        }
    }
    __syncthreads();
    // ---- compute
    T acc[PG_R];
#pragma unroll
    for (int r = 0; r < PG_R; ++r) acc[r] = E::zero();
    const T* tb = S + tid * (L::RD + L::PADE);
    const int nblk = PG_R + Qn - 1;
#pragma unroll 1
    for (int jb = 0; jb < nblk; ++jb) {
        T xs[D];
        // block jb of this thread: elements (tid*R + jb)*D + p -> padded: the thread base absorbs tid's padding, and a
        // block never straddles a padding slot (blocks are D long, slots sit every R*D)
        const T* bp = tb + jb * D + L::PADE * (jb / PG_R);
#pragma unroll
        for (int p = 0; p < D; ++p) xs[p] = bp[p];
#pragma unroll
        for (int r = 0; r < PG_R; ++r) {
            const int q = jb - r;                          // warp-uniform
            if (q >= 0 && q < Qn) {
#pragma unroll
                for (int p = 0; p < D; ++p) {
                    if constexpr (CTAPS) E::macc(acc[r], xs[p], P.hr[2 * (q * D + p)], P.hr[2 * (q * D + p) + 1]);
                    else E::mac(acc[r], xs[p], P.hr[q * D + p]);
                }
            }
        }
    }
    // ---- store
    const long long m0 = tile * PG_TO + (long long)tid * PG_R;
#pragma unroll
    for (int r = 0; r < PG_R; ++r)
        if (m0 + r < P.n_out) y[m0 + r] = acc[r];
}

template <typename T, int D, bool CTAPS>
int launch_pg(const GenParams& P, const void* x, const void* hist, void* y, cudaStream_t s) {
    using L = PgLayout<D>;
    const size_t smem = L::smem_elems(P.Qn) * sizeof(T);
    auto k = poly_generic_kernel<T, D, CTAPS>;
    static size_t configured_dev[LRB_MAX_DEVICES] = {0};
    size_t& configured = configured_dev[ctx().device & (LRB_MAX_DEVICES - 1)];
    if (smem > configured) {
        LRB_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = smem;
    }
    const long long tiles = (P.n_out + PG_TO - 1) / PG_TO;
    if (tiles > 2147483647LL) { set_error("fir: too many tiles for one launch"); return -1; }
    k<<<(unsigned)tiles, PG_THREADS, smem, s>>>((const T*)x, (const T*)hist, (T*)y, P);
    count_launch();
    LRB_CHECK(cudaGetLastError());
    return 0;
}

template <int D>
int launch_pg_d(FirKind kind, const GenParams& P, const void* x, const void* hist, void* y, cudaStream_t s) {
    if (kind == FIR_RRRF) return launch_pg<float, D, false>(P, x, hist, y, s);
    return kind == FIR_CCCF ? launch_pg<float2, D, true>(P, x, hist, y, s) : launch_pg<float2, D, false>(P, x, hist, y, s);
}

}  // namespace

// Is (kind, M, D) covered?  D from the instantiated list, the padded taps within the parameter budget, and the tile
// (1024 + Qn) * D samples within 200 KB of shared memory.
bool poly_generic_supports(FirKind kind, int M, int D) {
    if (kind == FIR_HILBERT) return false;
    switch (D) { case 2: case 3: case 4: case 5: case 6: case 7: case 8: case 10: case 12: case 16: case 20: case 25: break; default: return false; }
    const int Qn = (M + D - 1) / D;
    const int taps = Qn * D * (kind == FIR_CCCF ? 2 : 1);
    if (taps > PG_MAXT) return false;
    const size_t elem = kind == FIR_RRRF ? 4 : 8;
    return (size_t)(PG_TO + Qn + PG_TO / PG_R + 4) * D * elem <= (size_t)200 * 1024;
}

// taps: natural order (float, or interleaved complex for FIR_CCCF); (kind, M, D) covered.  0, or -1 with the error set.
int launch_poly_generic(FirKind kind, const void* x, const void* hist, const void* taps_host, int M, int D,
                        long long first, long long n, long long n_out, void* y, cudaStream_t s) {
    if (n_out <= 0) return 0;
    GenParams P;
    std::memset(&P, 0, sizeof(P));
    const int Qn = (M + D - 1) / D, z = Qn * D - M;
    const float* t = (const float*)taps_host;
    for (int i = z; i < Qn * D; ++i) {
        const int k = M - 1 - (i - z);                       // hr'[i] = h[M-1-(i-z)]
        if (kind == FIR_CCCF) { P.hr[2 * i] = t[2 * k]; P.hr[2 * i + 1] = t[2 * k + 1]; }
        else P.hr[i] = t[k];
    }
    P.first = first; P.n = n; P.n_out = n_out; P.Qn = Qn; P.Hm1 = M - 1;
    switch (D) {
        case 2: return launch_pg_d<2>(kind, P, x, hist, y, s);
        case 3: return launch_pg_d<3>(kind, P, x, hist, y, s);
        case 4: return launch_pg_d<4>(kind, P, x, hist, y, s);
        case 5: return launch_pg_d<5>(kind, P, x, hist, y, s);
        case 6: return launch_pg_d<6>(kind, P, x, hist, y, s);
        case 7: return launch_pg_d<7>(kind, P, x, hist, y, s);
        case 8: return launch_pg_d<8>(kind, P, x, hist, y, s);
        case 10: return launch_pg_d<10>(kind, P, x, hist, y, s);
        case 12: return launch_pg_d<12>(kind, P, x, hist, y, s);
        case 16: return launch_pg_d<16>(kind, P, x, hist, y, s);
        case 20: return launch_pg_d<20>(kind, P, x, hist, y, s);
        case 25: return launch_pg_d<25>(kind, P, x, hist, y, s);
    }
    set_error("fir: no generic polyphase kernel for D = %d", D);
    return -1;
}

}  // namespace lrb
