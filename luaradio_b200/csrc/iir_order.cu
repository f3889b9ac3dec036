// IIRFilterBlock with 11..64 feed-forward or feedback taps (iirfilter.lua:113-179) as a state-space scan in double.
//
//     y[n] = (sum_{j<nb} b[j] x[n-j] - sum_{1<=j<na} a[j] y[n-j]) / a[0]
//
// Split into the FIR part u = (b / a0) * x and the all-pole part of order q = na - 1.  The state is the last q
// outputs s = (y[-1], .., y[-q]); with zero input one sample maps s -> M s (M the companion matrix of a / a0), V samples
// -> M^V s, and the output i samples after a state s is the homogeneous response hom[.][i] . s (row 0 of M^(i+1)).
//   thread: V samples of u and of the recurrence from a zero state (yl), end state z_t = (yl[V-1], .., yl[V-q]);
//   CTA:    warp 0 chains the thread states serially, lanes over the rows of M^V: e_(t+1) = z_t + M^V e_t;
//           e_P is the tile's aggregate (the end state of the tile from a zero state);
//   grid:   decoupled look-back over per-tile (aggregate | inclusive prefix) q-vector records, the predecessor d tiles
//           back weighted with M^(T (d-1)) (host table): always the aggregates of the IO_LBW - 1 nearest predecessors
//           and the prefix of the one IO_LBW back (or of tile 0), so the sums do not depend on timing and the outputs
//           are bit-identical from run to run;
//   CTA:    warp 0 chains again from the tile's carry: s_t, the exact state in front of each thread;
//   thread: y[i] = yl[i] + hom[.][i] . s_t, rounded to float32 once.
// State, carries and accumulation are double: the powers of M for poles near the unit circle grow far above 1
// before they decay.  No warm-up and no truncation: exact up to rounding for any pole radius.  One launch per call.
// Algorithmic traffic 8 B/sample real, 16 B/sample complex, plus one q-vector record pair per 2048-sample tile.
#include "common.cuh"
#include "blocks.h"

#include <cmath>
#include <vector>

namespace lrb {

namespace {

constexpr int IO_THREADS = 64;                         // two warps: warp 0 runs the chains and the look-back
constexpr int IO_V = 32;                               // samples per thread
constexpr int IO_TILE = IO_THREADS * IO_V;
constexpr int IO_LBW = 8;                              // aggregates folded in before a tile waits for a prefix
constexpr int IO_XOFF = IIR_ORDER_MAX_TAPS - 1;        // staged inputs start this far before the tile

struct IoParams {
    double b[IIR_ORDER_MAX_TAPS];                      // b[j] / a0
    double c[IIR_ORDER_MAX_TAPS];                      // c[j] = -a[j] / a0 for 1 <= j <= q; 0 elsewhere
    int nb, q;
};

template <typename T> struct Wide;
template <> struct Wide<float> { using type = double; };
template <> struct Wide<float2> { using type = double2; };

__device__ __forceinline__ double dzero(double) { return 0.0; }
__device__ __forceinline__ double2 dzero(double2) { return make_double2(0.0, 0.0); }
__device__ __forceinline__ double dfma(double s, double v, double a) { return fma(s, v, a); }
__device__ __forceinline__ double2 dfma(double s, double2 v, double2 a) { return make_double2(fma(s, v.x, a.x), fma(s, v.y, a.y)); }
__device__ __forceinline__ double widen(float v) { return (double)v; }
__device__ __forceinline__ double2 widen(float2 v) { return make_double2((double)v.x, (double)v.y); }
__device__ __forceinline__ float narrow(double v) { return __double2float_rn(v); }
__device__ __forceinline__ float2 narrow(double2 v) { return make_float2(__double2float_rn(v.x), __double2float_rn(v.y)); }
__device__ __forceinline__ float fzero(float) { return 0.f; }
__device__ __forceinline__ float2 fzero(float2) { return make_float2(0.f, 0.f); }
__device__ __forceinline__ double shfl(double v, int l) { return __shfl_sync(0xffffffffu, v, l); }
__device__ __forceinline__ double2 shfl(double2 v, int l) {
    return make_double2(__shfl_sync(0xffffffffu, v.x, l), __shfl_sync(0xffffffffu, v.y, l));
}
__device__ __forceinline__ double ldcg(const double* p) { return __ldcg(p); }
__device__ __forceinline__ double2 ldcg(const double2* p) { return __ldcg(p); }

// staged input e lives at xs[e + e / 32]: thread t reads e = t V + i, so a warp's 32 reads hit 32 banks
__device__ __forceinline__ int xpad(int e) { return e + (e >> 5); }
constexpr int xs_len() { return IO_TILE + IO_XOFF + (IO_TILE + IO_XOFF) / 32 + 1; }

// Rows r0 = lane and r1 = lane + 32 of  acc + W v,  W column-major q x q in global memory, v distributed like acc.
template <typename D, int QM>
__device__ __forceinline__ void matvec_rows(const double* __restrict__ W, int q, int lane, D v0, D v1, D& acc0, D& acc1) {
    const int r0 = lane, r1 = lane + 32;
    for (int cc = 0; cc < q && cc < 32; ++cc) {
        const D vc = shfl(v0, cc);
        if (r0 < q) acc0 = dfma(__ldg(W + cc * q + r0), vc, acc0);
        if (QM > 32 && r1 < q) acc1 = dfma(__ldg(W + cc * q + r1), vc, acc1);
    }
    if (QM > 32) {
        for (int cc = 32; cc < q; ++cc) {
            const D vc = shfl(v1, cc - 32);
            if (r0 < q) acc0 = dfma(__ldg(W + cc * q + r0), vc, acc0);
            if (r1 < q) acc1 = dfma(__ldg(W + cc * q + r1), vc, acc1);
        }
    }
}

// One record per tile and kind: q elements at rec + tile * q.  flags[tile] = epoch * 4 + 1 (aggregate) / + 2 (prefix).
template <typename T, int QM>
__global__ void __launch_bounds__(IO_THREADS)
iir_order_kernel(const T* __restrict__ x, long long n, T* __restrict__ y, const IoParams P,
                 const double* __restrict__ mats, const double* __restrict__ hom,
                 const T* __restrict__ xhist_in, T* __restrict__ xhist_out,
                 const typename Wide<T>::type* __restrict__ ys_in, typename Wide<T>::type* __restrict__ ys_out,
                 unsigned long long* ticket, unsigned long long ticket_base, volatile int* flags,
                 typename Wide<T>::type* agg, typename Wide<T>::type* pfx, unsigned epoch) {
    using D = typename Wide<T>::type;
    extern __shared__ __align__(16) unsigned char io_smem[];
    D* sv = reinterpret_cast<D*>(io_smem);                          // [IO_THREADS][QM + 1]: z_t, then s_t
    T* xs = reinterpret_cast<T*>(sv + IO_THREADS * (QM + 1));       // staged inputs, then staged outputs
    __shared__ int s_tile;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int q = P.q, nb = P.nb, nh = nb - 1;
    if (tid == 0) s_tile = (int)(atomicAdd(ticket, 1ULL) - ticket_base);
    __syncthreads();
    const int tile = s_tile;
    const long long base = (long long)tile * IO_TILE;
    const bool last_tile = base + IO_TILE >= n;

    // ---- stage x[base - IO_XOFF, base + TILE): the carried history before the stream, zeros past its end
    for (int e = tid; e < IO_TILE + IO_XOFF; e += IO_THREADS) {
        const long long g = base - IO_XOFF + e;
        T v = fzero(T());
        if (g >= n) v = fzero(T());
        else if (g >= 0) v = x[g];
        else if (g >= -nh) v = xhist_in[nh + g];
        xs[xpad(e)] = v;
    }
    __syncthreads();

    // ---- u and the recurrence from a zero state over this thread's V samples
    D yl[IO_V];
    const int e0 = IO_XOFF + tid * IO_V;
#pragma unroll
    for (int i = 0; i < IO_V; ++i) {
        D acc = dzero(D());
        for (int j = 0; j < nb; ++j) acc = dfma(P.b[j], widen(xs[xpad(e0 + i - j)]), acc);
#pragma unroll
        for (int j = 1; j <= i && j < IIR_ORDER_MAX_TAPS && j <= QM; ++j) acc = dfma(P.c[j], yl[i - j], acc);
        yl[i] = acc;
    }
    D* my = sv + tid * (QM + 1);
#pragma unroll
    for (int k = 0; k < QM; ++k)
        if (k < q) my[k] = k < IO_V ? yl[IO_V - 1 - k] : dzero(D());
    __syncthreads();

    const int r0 = lane, r1 = lane + 32;
    if (warp == 0 && q > 0) {
        const double* MV = mats;                                    // M^V
        // ---- chain 1: the tile's aggregate
        D e0v = dzero(D()), e1v = dzero(D());
        for (int t = 0; t < IO_THREADS; ++t) {
            const D* zt = sv + t * (QM + 1);
            D n0 = r0 < q ? zt[r0] : dzero(D()), n1 = (QM > 32 && r1 < q) ? zt[r1] : dzero(D());
            matvec_rows<D, QM>(MV, q, lane, e0v, e1v, n0, n1);
            e0v = n0;
            e1v = n1;
        }
        // ---- look-back
        D c0 = dzero(D()), c1 = dzero(D());
        if (tile == 0) {
            if (r0 < q) c0 = ys_in[r0];
            if (QM > 32 && r1 < q) c1 = ys_in[r1];
        } else {
            if (r0 < q) agg[(long long)tile * q + r0] = e0v;
            if (QM > 32 && r1 < q) agg[(long long)tile * q + r1] = e1v;
            __threadfence();
            __syncwarp();
            if (lane == 0) flags[tile] = (int)(epoch * 4u + 1u);
            // A fixed walk: the aggregates of the nearer predecessors and the prefix of tile max(tile - LBW, 0),
            // whatever else is already visible, so the carry (and every output) is the same from run to run.
            const int dlast = tile < IO_LBW ? tile : IO_LBW;
            for (int d = 1; d <= dlast; ++d) {
                const int j = tile - d;
                const bool want_pfx = d == dlast;                   // tile 0 publishes only a prefix
                int f = 0;
                if (lane == 0) {
                    do { f = flags[j]; } while ((unsigned)f >> 2 != epoch || (want_pfx && (f & 3) != 2));
                }
                f = __shfl_sync(0xffffffffu, f, 0);                 // one flag value for the whole warp
                __threadfence();
                const D* v = (want_pfx ? pfx : agg) + (long long)j * q;
                const D v0 = r0 < q ? ldcg(v + r0) : dzero(D());
                const D v1 = (QM > 32 && r1 < q) ? ldcg(v + r1) : dzero(D());
                matvec_rows<D, QM>(mats + (size_t)d * q * q, q, lane, v0, v1, c0, c1);    // M^(T (d-1))
            }
        }
        // ---- inclusive prefix = aggregate + M^T carry
        {
            D p0 = e0v, p1 = e1v;
            matvec_rows<D, QM>(mats + (size_t)2 * q * q, q, lane, c0, c1, p0, p1);
            if (!last_tile) {
                if (r0 < q) pfx[(long long)tile * q + r0] = p0;
                if (QM > 32 && r1 < q) pfx[(long long)tile * q + r1] = p1;
                __threadfence();
                __syncwarp();
                if (lane == 0) flags[tile] = (int)(epoch * 4u + 2u);
            }
        }
        // ---- chain 2: the exact state in front of each thread
        for (int t = 0; t < IO_THREADS; ++t) {
            D* zt = sv + t * (QM + 1);
            D n0 = r0 < q ? zt[r0] : dzero(D()), n1 = (QM > 32 && r1 < q) ? zt[r1] : dzero(D());
            if (r0 < q) zt[r0] = c0;
            if (QM > 32 && r1 < q) zt[r1] = c1;
            matvec_rows<D, QM>(MV, q, lane, c0, c1, n0, n1);
            c0 = n0;
            c1 = n1;
        }
    }
    __syncthreads();

    // ---- the homogeneous response of the thread's incoming state
    for (int k = 0; k < q; ++k) {
        const D sk = my[k];
        const double* hk = hom + k * IO_V;
#pragma unroll
        for (int i = 0; i < IO_V; ++i) yl[i] = dfma(__ldg(hk + i), sk, yl[i]);
    }

    // ---- carried state for the next call: the last q outputs (most recent first) and the last nb - 1 inputs
    const long long g0 = base + (long long)tid * IO_V;
#pragma unroll
    for (int i = 0; i < IO_V; ++i) {
        const long long g = g0 + i;
        if (g < n && g >= n - q) ys_out[n - 1 - g] = yl[i];
    }
    if (tile == 0) {
        for (int k = (int)(n < (long long)q ? n : q) + tid; k < q; k += IO_THREADS) ys_out[k] = ys_in[k - n];
        for (int k = tid; k < nh; k += IO_THREADS) {
            const long long i = n - nh + k;
            xhist_out[k] = i >= 0 ? x[i] : xhist_in[nh + i];
        }
    }

    // ---- outputs, rounded once, stored through shared memory (coalesced at any alignment)
#pragma unroll
    for (int i = 0; i < IO_V; ++i) xs[xpad(tid * IO_V + i)] = narrow(yl[i]);
    __syncthreads();
    const int cnt = last_tile ? (int)(n - base) : IO_TILE;
    for (int e = tid; e < cnt; e += IO_THREADS) y[base + e] = xs[xpad(e)];
}

template <typename T, int QM>
size_t io_smem_bytes() {
    return sizeof(typename Wide<T>::type) * IO_THREADS * (QM + 1) + sizeof(T) * xs_len();
}

// the homogeneous response of unit state e_c over L samples: g[c * L + m] = y[m] with y[-1-c] = 1, zero input.  Run in
// long double and rounded once, so each table entry is within one double rounding of the exact power of M.
std::vector<double> homogeneous(const double* cdiv, int q, int L) {
    std::vector<double> g((size_t)q * L, 0.0);
    std::vector<long double> yv((size_t)(q + L));
    for (int c = 0; c < q; ++c) {
        std::fill(yv.begin(), yv.end(), 0.0L);
        yv[(size_t)(q - 1 - c)] = 1.0L;                             // yv[q + m] = y[m]
        for (int m = 0; m < L; ++m) {
            long double acc = 0.0L;
            for (int j = 1; j <= q; ++j) acc += (long double)cdiv[j] * yv[(size_t)(q + m - j)];
            yv[(size_t)(q + m)] = acc;
            g[(size_t)c * L + m] = (double)acc;
        }
    }
    return g;
}

template <typename T, int QM>
void launch_shape(int tiles, cudaStream_t s, const void* x, long long n, void* y, const IoParams& P, const double* mats,
                  const double* hom, const void* xh_in, void* xh_out, const void* ys_in, void* ys_out,
                  unsigned long long* ticket, unsigned long long tb, int* flags, void* agg, void* pfx, unsigned epoch) {
    using D = typename Wide<T>::type;
    const size_t sm = io_smem_bytes<T, QM>();
    static bool attr = false;                                       // per instantiation, once per process
    if (!attr) {
        cudaFuncSetAttribute(iir_order_kernel<T, QM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
        attr = true;
    }
    iir_order_kernel<T, QM><<<tiles, IO_THREADS, sm, s>>>((const T*)x, n, (T*)y, P, mats, hom, (const T*)xh_in, (T*)xh_out,
                                                          (const D*)ys_in, (D*)ys_out, ticket, tb, flags, (D*)agg, (D*)pfx, epoch);
}

}  // namespace

// ---------------------------------------------------------------------------------------------
IirOrderBlock::IirOrderBlock(bool cplx, const float* b_, unsigned nb_, const float* a_, unsigned na_, bool dev)
    : Block(std::string(cplx ? "iir_crcf" : "iir_rrrf") + "(scan," + std::to_string((int)na_ - 1) + ")",
            cplx ? 8 : 4, cplx ? 8 : 4, dev) {
    complex_data = cplx;
    nb = (int)nb_;
    q = (int)na_ - 1;
    const double a0 = a_[0];
    b.assign((size_t)nb, 0.0);
    cdiv.assign((size_t)q + 1, 0.0);
    for (int j = 0; j < nb; ++j) b[(size_t)j] = (double)b_[j] / a0;
    for (int j = 1; j <= q; ++j) cdiv[(size_t)j] = -(double)a_[j] / a0;
    // decay length of 1/A(z): last index where the impulse response is >= 1e-10 of its peak (IirGeneralBlock's measure)
    const int limit = 1 << 16;
    std::vector<double> h((size_t)limit);
    double peak = 0.0;
    long long last = 0;
    for (int i = 0; i < limit; ++i) {
        double v = (i == 0) ? 1.0 : 0.0;
        for (int j = 1; j <= q && j <= i; ++j) v += cdiv[(size_t)j] * h[(size_t)(i - j)];
        h[(size_t)i] = v;
        if (!std::isfinite(v)) { last = limit; break; }
        if (std::fabs(v) > peak) peak = std::fabs(v);
        if (std::fabs(v) >= 1e-10 * peak) last = i;
    }
    decay = (last + q + nb >= limit - 1) ? -1 : last + q + nb;
}

int IirOrderBlock::init() {
    const size_t de = complex_data ? 2 * sizeof(double) : sizeof(double);
    if (carry(d_xhist, (size_t)(nb > 1 ? nb - 1 : 1) * in_size, cur) != 0 || carry(d_ystate, (size_t)(q > 0 ? q : 1) * de, cur) != 0)
        return -1;
    if (d_ticket.alloc_zeroed(sizeof(unsigned long long)) != 0 || d_flags.alloc_zeroed(sizeof(int) * IIR_ORDER_MAX_TILES) != 0)
        return -1;
    if (q == 0) return 0;
    // M^k from the homogeneous responses: (M^k)[r][c] = g_c[k-1-r] for k > r, else [c == r - k]
    const int L = IO_TILE * (IO_LBW - 1) + 1;
    const std::vector<double> g = homogeneous(cdiv.data(), q, L > IO_V ? L : IO_V);
    const int Lg = L > IO_V ? L : IO_V;
    auto power = [&](long long k, double* W) {                     // column-major
        for (int c = 0; c < q; ++c)
            for (int r = 0; r < q; ++r)
                W[(size_t)c * q + r] = (k > r) ? g[(size_t)c * Lg + (size_t)(k - 1 - r)] : (c == r - k ? 1.0 : 0.0);
    };
    const size_t qq = (size_t)q * q;
    std::vector<double> mats(qq * (1 + IO_LBW));
    power(IO_V, mats.data());
    for (int e = 0; e < IO_LBW; ++e) power((long long)IO_TILE * e, mats.data() + qq * (1 + e));
    std::vector<double> hom((size_t)q * IO_V);
    for (int c = 0; c < q; ++c)
        for (int i = 0; i < IO_V; ++i) hom[(size_t)c * IO_V + i] = g[(size_t)c * Lg + i];
    if (d_mats.upload(mats.data(), sizeof(double) * mats.size()) != 0 || d_hom.upload(hom.data(), sizeof(double) * hom.size()) != 0)
        return -1;
    return 0;
}

int IirOrderBlock::run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) {
    *n_out = n;
    if (n == 0) return 0;
    const long long maxn = (long long)IIR_ORDER_MAX_TILES * IO_TILE;
    const size_t de = complex_data ? 2 * sizeof(double) : sizeof(double);
    IoParams P;
    for (int j = 0; j < IIR_ORDER_MAX_TAPS; ++j) {
        P.b[j] = j < nb ? b[(size_t)j] : 0.0;
        P.c[j] = (j >= 1 && j <= q) ? cdiv[(size_t)j] : 0.0;
    }
    P.nb = nb;
    P.q = q;
    size_t done = 0;
    while (done < n) {
        const long long nc = (long long)(n - done) < maxn ? (long long)(n - done) : maxn;
        const int tiles = (int)((nc + IO_TILE - 1) / IO_TILE);
        const size_t rec = (size_t)tiles * (size_t)(q > 0 ? q : 1) * de;
        if (d_agg.reserve(rec) != 0 || d_pfx.reserve(rec) != 0) return -1;
        epoch = (epoch + 1) & 0x3fffffffu;
        if (epoch == 0) {                                           // wrapped: clear stale flags
            LRB_CHECK(cudaMemsetAsync(d_flags.get(), 0, sizeof(int) * IIR_ORDER_MAX_TILES, s));
            epoch = 1;
        }
        const char* xin = (const char*)dx + done * in_size;
        char* yout = (char*)dy + done * out_size;
#define LRB_IO(TT, QQ)                                                                                                  \
        launch_shape<TT, QQ>(tiles, s, xin, nc, yout, P, d_mats.as<double>(), d_hom.as<double>(), d_xhist[cur].get(),   \
                             d_xhist[cur ^ 1].get(), d_ystate[cur].get(), d_ystate[cur ^ 1].get(),                       \
                             d_ticket.as<unsigned long long>(), ticket_base, d_flags.as<int>(), d_agg.get(), d_pfx.get(), epoch)
        if (complex_data) { if (q <= 16) LRB_IO(float2, 16); else if (q <= 32) LRB_IO(float2, 32); else LRB_IO(float2, 64); }
        else { if (q <= 16) LRB_IO(float, 16); else if (q <= 32) LRB_IO(float, 32); else LRB_IO(float, 64); }
#undef LRB_IO
        count_launch();
        LRB_CHECK(cudaGetLastError());
        ticket_base += (unsigned long long)tiles;
        cur ^= 1;
        consumed += (uint64_t)nc;
        done += (size_t)nc;
    }
    return 0;
}

}  // namespace lrb
