// Level control: AGCBlock and PowerSquelchBlock as one-pass block-parallel scans.
//
// Reference recurrences (radio/blocks/signal/agc.lua:72-115, powersquelch.lua:43-75), in Lua numbers (double):
//     P[n] = (1-pa) P[n-1] + pa |x[n]|^2                                  power estimator (both blocks)
//     AGC:       P[n] >= theta:  g[n] = (1-ga) g[n-1] + ga (T (1/P[n])),  y[n] = float(sqrt(g[n]) x[n])
//                otherwise:      g[n] = g[n-1],                            y[n] = x[n]
//     squelch:   y[n] = P[n] >= theta ? x[n] : 0
//
// Stage A: the power estimator is an affine recurrence with the constant slope a = 1-pa, scanned like iir.cu's single
// pole (thread-sequential -> warp Kogge-Stone with slopes a^(V 2^k) -> CTA Horner over warps -> decoupled look-back over
// tiles), all in double.  Each thread then re-runs its own V samples from the exact carry in the reference's operation
// order, which gives P[n] and the gate.
// Stage B (AGC only): the gain map of an open sample is g -> b g + u[n] (b = 1-ga, u[n] = ga (T (1/P[n]))), of a closed
// one the identity; a span with m open samples composes to g -> b^m g + B.  The (m, B) pairs are scanned the same way
// (b^m from a host table; for spans longer than a tile from the binary powers b^(2^k)), published per tile, looked back
// a second time, and each thread re-runs its gain recurrence from the exact carry.  A tile whose gate is closed on every
// sample publishes the identity map and skips the second look-back: it costs the copy.
// x is read once and y written once: 8 B/sample real, 16 B/sample complex, plus a few records per 2048-sample tile.
#include "../../include/lrb200.h"
#include "common.cuh"
#include "blocks.h"

#include <cmath>
#include <new>
#include <vector>

namespace lrb {

namespace {

constexpr int LV_THREADS = 256;
constexpr int LV_LOGW = 3;                         // log2(warps per CTA)
constexpr int LV_V = 8;                            // samples per thread
constexpr int LV_TILE = LV_THREADS * LV_V;
static_assert((32 << LV_LOGW) == LV_THREADS, "LV_LOGW must be log2(warps per CTA)");

struct LevelParams {
    double a, pa;                  // power estimator: a = 1 - pa
    double b, ga;                  // gain filter: b = 1 - ga
    double T, theta;               // linear target and threshold
    double ca[5 + LV_LOGW + 1];    // ca[k] = a^(V 2^k); ca[5 + LOGW] = a^TILE
    double b2[32];                 // b2[k] = b^(2^k)
};

constexpr int LV_WIN = 4;                          // look-back: 32-tile windows fetched per round trip

// One look-back record per tile and stage: {value (2 words), open count m, flag = epoch * 4 + 1 (aggregate) / + 2 (inclusive
// prefix)}, written and read as ONE 16-byte access, so a reader that sees the flag sees the value: one memory round trip
// per window instead of flag, fence and value load.
struct LevelRecords {
    unsigned long long* ticket;
    uint4* rec_a;                  // power estimator: value = aggregate / prefix power
    uint4* rec_b;                  // gain (AGC): value = offset B / prefix gain, m = open samples of the aggregate
};

__device__ __forceinline__ uint4 ld_rec(const uint4* p) {
    uint4 r;
    asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void st_rec(uint4* p, double v, unsigned m, unsigned flag) {
    asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};"
                 :: "l"(p), "r"((unsigned)__double2loint(v)), "r"((unsigned)__double2hiint(v)), "r"(m), "r"(flag) : "memory");
}
__device__ __forceinline__ double rec_value(uint4 r) { return __hiloint2double((int)r.y, (int)r.x); }

__device__ __forceinline__ double esq(float v) { return __dmul_rn((double)v, (double)v); }
__device__ __forceinline__ double esq(float2 v) {     // complexfloat32.lua:174: re*re + im*im in double
    return __dadd_rn(__dmul_rn((double)v.x, (double)v.x), __dmul_rn((double)v.y, (double)v.y));
}
__device__ __forceinline__ float zero_of(float) { return 0.f; }
__device__ __forceinline__ float2 zero_of(float2) { return make_float2(0.f, 0.f); }
__device__ __forceinline__ float scale_of(float v, double s) { return __double2float_rn(__dmul_rn(s, (double)v)); }
__device__ __forceinline__ float2 scale_of(float2 v, double s) {
    return make_float2(__double2float_rn(__dmul_rn(s, (double)v.x)), __double2float_rn(__dmul_rn(s, (double)v.y)));
}

// x[b .. b+8) / y[b .. b+8) as 128-bit accesses (tile and thread bases are multiples of 8 samples)
__device__ __forceinline__ void load8(const float* p, float (&v)[LV_V]) {
    const float4 u = __ldcs(reinterpret_cast<const float4*>(p)), w = __ldcs(reinterpret_cast<const float4*>(p) + 1);
    v[0] = u.x; v[1] = u.y; v[2] = u.z; v[3] = u.w; v[4] = w.x; v[5] = w.y; v[6] = w.z; v[7] = w.w;
}
__device__ __forceinline__ void load8(const float2* p, float2 (&v)[LV_V]) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float4 u = __ldcs(reinterpret_cast<const float4*>(p) + k);
        v[2 * k] = make_float2(u.x, u.y);
        v[2 * k + 1] = make_float2(u.z, u.w);
    }
}
__device__ __forceinline__ void store8(float* p, const float (&v)[LV_V]) {
    __stcs(reinterpret_cast<float4*>(p), make_float4(v[0], v[1], v[2], v[3]));
    __stcs(reinterpret_cast<float4*>(p) + 1, make_float4(v[4], v[5], v[6], v[7]));
}
__device__ __forceinline__ void store8(float2* p, const float2 (&v)[LV_V]) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
        __stcs(reinterpret_cast<float4*>(p) + k, make_float4(v[2 * k].x, v[2 * k].y, v[2 * k + 1].x, v[2 * k + 1].y));
}

// b^m for any m >= 0 from the binary powers
__device__ __forceinline__ double pow_b(const LevelParams& P, unsigned m) {
    double r = 1.0;
    for (int k = 0; m; ++k, m >>= 1)
        if (m & 1u) r *= P.b2[k];
    return r;
}

// (LV_THREADS, 2): a 128-register budget.  Under the default budget of 64 ptxas spilled the gate mask around the
// slow-path subroutine calls of __drcp_rn / __dsqrt_rn.
template <typename T, bool AGC>
__global__ void __launch_bounds__(LV_THREADS, 2)
level_kernel(const T* __restrict__ x, long long n, T* __restrict__ y, LevelParams P, const double* __restrict__ pw,
             const double2* __restrict__ st_in, double2* __restrict__ st_out, LevelRecords R,
             unsigned long long ticket_base, unsigned epoch) {
    __shared__ int s_tile;
    __shared__ double s_warp[LV_THREADS / 32];
    __shared__ int s_wm[LV_THREADS / 32];
    __shared__ double s_agg, s_carry;
    __shared__ int s_aggm;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_tile = (int)(atomicAdd(R.ticket, 1ULL) - ticket_base);
    __syncthreads();
    const int tile = s_tile;
    const long long base = (long long)tile * LV_TILE + (long long)tid * LV_V;
    const bool last_tile = (long long)(tile + 1) * LV_TILE >= n;

    // ---- load, |x|^2 and the thread's zero-state power
    T xv[LV_V];
    const bool full = base + LV_V <= n;
    const bool vec = full && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
    if (vec) {
        load8(x + base, xv);
    } else {
#pragma unroll
        for (int i = 0; i < LV_V; ++i) xv[i] = base + i < n ? x[base + i] : zero_of(T());
    }
    double p = 0.0;
#pragma unroll
    for (int i = 0; i < LV_V; ++i) p = fma(P.a, p, P.pa * esq(xv[i]));

    // ---- stage A: warp scan, CTA carry, decoupled look-back
    double Bw = p;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        const double o = __shfl_up_sync(0xffffffffu, Bw, 1 << k);
        if (lane >= (1 << k)) Bw = fma(P.ca[k], o, Bw);
    }
    if (lane == 31) s_warp[warp] = Bw;
    double prevB = __shfl_up_sync(0xffffffffu, Bw, 1);
    if (lane == 0) prevB = 0.0;
    __syncthreads();
    double carryW = 0.0;                               // power at the end of warp-1, zero state from the tile start
    for (int w = 0; w < warp; ++w) carryW = fma(P.ca[5], carryW, s_warp[w]);
    double f_lane = 1.0;                               // a^(V lane)
#pragma unroll
    for (int k = 0; k < 5; ++k) if (lane & (1 << k)) f_lane *= P.ca[k];
    const double excl = fma(f_lane, carryW, prevB);
    if (tid == LV_THREADS - 1) s_agg = fma(f_lane * P.ca[0], carryW, Bw);
    __syncthreads();
    if (warp == 0) {
        const double cT = P.ca[5 + LV_LOGW];
        double carry_in = 0.0;
        if (tile == 0) {
            carry_in = st_in->x;
        } else {
            if (lane == 0) st_rec(R.rec_a + tile, s_agg, 0u, epoch * 4u + 1u);
            double wl = 1.0, pwr = cT;                 // wl = cT^lane, pwr -> cT^32
#pragma unroll
            for (int k = 0; k < 5; ++k) { if (lane & (1 << k)) wl *= pwr; pwr *= pwr; }
            double mult = 1.0;
            int jbase = tile - 1;
            bool done = false;
            while (!done) {
                // lane L of window k holds tile jbase - 32 k - L.  The nearest window is fetched (and waited for) first; the
                // older ones are fetched together after it, so that they show the prefixes published in the meantime.
                uint4 r[LV_WIN];
#pragma unroll
                for (int k = 0; k < LV_WIN; ++k) {
                    if (done) break;
                    if (k <= 1) {
                        double wk = mult;
#pragma unroll
                        for (int q = 0; q < LV_WIN; ++q) {
                            const int j = jbase - 32 * (q - k) - lane;
                            if (q == k || (k == 1 && q > 1)) {
                                r[q] = make_uint4(0u, 0u, 0u, 0u);
                                if (j >= 0 && wl * wk != 0.0) r[q] = ld_rec(R.rec_a + j);
                            }
                            if (q >= k) wk *= pwr;
                        }
                    }
                    const int j = jbase - lane;
                    const double wgt = wl * mult;
                    const bool dead = wgt == 0.0;      // a predecessor whose weight underflows cannot change the carry
                    if (j >= 0 && !dead)
                        while (r[k].w >> 2 != epoch) r[k] = ld_rec(R.rec_a + j);
                    const unsigned pmask = __ballot_sync(0xffffffffu, j >= 0 && (dead || (r[k].w & 3) == 2));
                    const int lastl = pmask ? (__ffs(pmask) - 1) : 31;
                    double c = (j >= 0 && !dead && lane <= lastl) ? wgt * rec_value(r[k]) : 0.0;
#pragma unroll
                    for (int off = 16; off >= 1; off >>= 1) c += __shfl_xor_sync(0xffffffffu, c, off);
                    carry_in += c;
                    done = pmask != 0;                 // tile 0 always publishes a prefix
                    mult *= pwr;
                    jbase -= 32;
                }
            }
        }
        if (lane == 0) {
            st_rec(R.rec_a + tile, fma(cT, carry_in, s_agg), 0u, epoch * 4u + 2u);
            s_carry = carry_in;
        }
    }
    __syncthreads();
    double f_thread = f_lane;                          // a^(V tid)
#pragma unroll
    for (int k = 0; k < LV_LOGW; ++k) if (warp & (1 << k)) f_thread *= P.ca[5 + k];
    double pw_cur = fma(f_thread, s_carry, excl);      // power just before this thread's first sample

    // ---- the thread's own samples in the reference's operation order: P[n] and the gate
    unsigned openm = 0;
    double u[LV_V];
    int m = 0;
    double Bg = 0.0;
    double p_last = 0.0;
#pragma unroll
    for (int i = 0; i < LV_V; ++i) {
        pw_cur = __dadd_rn(__dmul_rn(P.a, pw_cur), __dmul_rn(P.pa, esq(xv[i])));
        if (base + i == n - 1) p_last = pw_cur;
        const bool op = base + i < n && pw_cur >= P.theta;
        openm |= (unsigned)op << i;
        u[i] = 0.0;
        if constexpr (AGC) {
            if (op) {
                u[i] = __dmul_rn(P.ga, __dmul_rn(P.T, __drcp_rn(pw_cur)));
                Bg = fma(P.b, Bg, u[i]);
                ++m;
            }
        }
    }

    T yv[LV_V];
    if constexpr (!AGC) {
#pragma unroll
        for (int i = 0; i < LV_V; ++i) yv[i] = (openm >> i & 1u) ? xv[i] : zero_of(T());
        if (base <= n - 1 && n - 1 < base + LV_V) *st_out = make_double2(p_last, 0.0);
    } else {
        // ---- stage B: scan of the (open count, offset) gain maps
        const bool any_open = __syncthreads_or(openm != 0);
        double g_cur = 0.0;
        if (!any_open && !last_tile) {
            // closed tile: publish the identity map (or, as tile 0, the carried gain) and pass the samples through
            if (tid == 0) {
                if (tile == 0) st_rec(R.rec_b, st_in->y, 0u, epoch * 4u + 2u);
                else st_rec(R.rec_b + tile, 0.0, 0u, epoch * 4u + 1u);
            }
        } else {
            int Mw = m;
            double Bv = Bg;
#pragma unroll
            for (int k = 0; k < 5; ++k) {
                const int om = __shfl_up_sync(0xffffffffu, Mw, 1 << k);
                const double ob = __shfl_up_sync(0xffffffffu, Bv, 1 << k);
                if (lane >= (1 << k)) { Bv = fma(__ldg(pw + Mw), ob, Bv); Mw += om; }
            }
            if (lane == 31) { s_wm[warp] = Mw; s_warp[warp] = Bv; }
            int pm = __shfl_up_sync(0xffffffffu, Mw, 1);
            double pb = __shfl_up_sync(0xffffffffu, Bv, 1);
            if (lane == 0) { pm = 0; pb = 0.0; }
            __syncthreads();
            int cm = 0;                                // maps of the warps before this one, composed
            double cb = 0.0;
            for (int w = 0; w < warp; ++w) { cb = fma(__ldg(pw + s_wm[w]), cb, s_warp[w]); cm += s_wm[w]; }
            const int ex_m = cm + pm;                  // this thread's exclusive map from the tile start
            const double ex_b = fma(__ldg(pw + pm), cb, pb);
            if (tid == LV_THREADS - 1) { s_aggm = cm + Mw; s_agg = fma(__ldg(pw + Mw), cb, Bv); }
            __syncthreads();
            if (warp == 0) {
                double carry_in;
                if (tile == 0) {
                    carry_in = st_in->y;
                } else {
                    if (lane == 0) st_rec(R.rec_b + tile, s_agg, (unsigned)s_aggm, epoch * 4u + 1u);
                    unsigned acc_m = 0;                // composition of the tiles already walked (newer than the window)
                    double acc_b = 0.0;
                    int jbase = tile - 1;
                    bool done = false;
                    while (!done) {
                      uint4 r[LV_WIN];                 // fetched as in stage A: the nearest window first
#pragma unroll
                      for (int k = 0; k < LV_WIN; ++k) {
                        if (done) break;
                        if (k <= 1) {
#pragma unroll
                            for (int q = k; q < (k == 0 ? 1 : LV_WIN); ++q) {
                                const int j = jbase - 32 * (q - k) - lane;
                                r[q] = j >= 0 ? ld_rec(R.rec_b + j) : make_uint4(0u, 0u, 0u, 0u);
                            }
                        }
                        const int j = jbase - lane;
                        if (j >= 0)
                            while (r[k].w >> 2 != epoch) r[k] = ld_rec(R.rec_b + j);
                        const bool pfx = j >= 0 && (r[k].w & 3) == 2;
                        unsigned wm = pfx ? 0u : r[k].z;   // a prefix is the absolute gain: (0, g)
                        double wb = j >= 0 ? rec_value(r[k]) : 0.0;
                        const unsigned pmask = __ballot_sync(0xffffffffu, pfx);
                        const int lastl = pmask ? (__ffs(pmask) - 1) : 31;
                        if (j < 0 || lane > lastl) { wm = 0; wb = 0.0; }
                        // ordered reduction, lane 0 = newest: lane L absorbs the older lanes L+d ..
#pragma unroll
                        for (int d = 1; d < 32; d <<= 1) {
                            const unsigned om = __shfl_down_sync(0xffffffffu, wm, d);
                            const double ob = __shfl_down_sync(0xffffffffu, wb, d);
                            if (lane + d < 32) { wb = fma(pow_b(P, wm), ob, wb); wm += om; }
                        }
                        wm = __shfl_sync(0xffffffffu, wm, 0);
                        wb = __shfl_sync(0xffffffffu, wb, 0);
                        const double sl = pow_b(P, acc_m);
                        acc_b = fma(sl, wb, acc_b);
                        acc_m += wm;
                        done = pmask != 0 || sl == 0.0;  // a prefix, or everything older is scaled to zero
                        jbase -= 32;
                      }
                    }
                    carry_in = acc_b;
                }
                if (lane == 0) {
                    st_rec(R.rec_b + tile, fma(__ldg(pw + s_aggm), carry_in, s_agg), 0u, epoch * 4u + 2u);
                    s_carry = carry_in;
                }
            }
            __syncthreads();
            g_cur = fma(__ldg(pw + ex_m), s_carry, ex_b);   // gain just before this thread's first sample
        }
#pragma unroll
        for (int i = 0; i < LV_V; ++i) {
            if (openm >> i & 1u) {
                g_cur = __dadd_rn(__dmul_rn(P.b, g_cur), u[i]);
                yv[i] = scale_of(xv[i], __dsqrt_rn(g_cur));
            } else {
                yv[i] = xv[i];
            }
            if (base + i == n - 1) *st_out = make_double2(p_last, g_cur);
        }
    }

    if (vec) {
        store8(y + base, yv);
    } else {
#pragma unroll
        for (int i = 0; i < LV_V; ++i) if (base + i < n) y[base + i] = yv[i];
    }
}

}  // namespace

// ---------------------------------------------------------------------------------------------
LevelBlock::LevelBlock(bool agc_, double power_alpha, double gain_alpha, double target, double threshold, bool cplx, bool dev)
    : Block(agc_ ? (cplx ? "agc_cc" : "agc_rr") : (cplx ? "powersquelch_cc" : "powersquelch_rr"), cplx ? 8 : 4, cplx ? 8 : 4, dev) {
    agc = agc_;
    complex_data = cplx;
    pa = power_alpha;
    ga = gain_alpha;
    T = target;
    theta = threshold;
}

int LevelBlock::init() {
    if (carry(d_state, 2 * sizeof(double), cur) != 0 || d_ticket.alloc_zeroed(sizeof(unsigned long long)) != 0 ||
        d_rec.alloc_zeroed(rec_bytes()) != 0)
        return -1;
    if (agc) {
        // b^k for the in-tile compositions (k <= one tile's samples)
        std::vector<double> pw((size_t)LV_TILE + 1);
        const double b = 1 - ga;
        pw[0] = 1.0;
        for (int k = 1; k <= LV_TILE; ++k) pw[(size_t)k] = pw[(size_t)k - 1] * b;
        if (d_pw.upload(pw.data(), sizeof(double) * pw.size()) != 0) return -1;
    }
    return 0;
}

long long LevelBlock::memory_in() const {
    if (agc) return -1;                    // a closed gate holds the gain for ever
    // the power estimator's pole decays to 1e-12 (as IirBlock::memory_in)
    const long long w = decay_samples(1 - pa);
    return w < 0 ? -1 : w + 1;
}

int LevelBlock::run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) {
    *n_out = n;
    LevelParams P;
    P.pa = pa;
    P.a = 1 - pa;
    P.ga = ga;
    P.b = 1 - ga;
    P.T = T;
    P.theta = theta;
    double p = 1.0;
    for (int i = 0; i < LV_V; ++i) p *= P.a;
    for (int k = 0; k < 5 + LV_LOGW + 1; ++k) { P.ca[k] = p; p = p * p; }
    double q = P.b;
    for (int k = 0; k < 32; ++k) { P.b2[k] = q; q = q * q; }
    LevelRecords R;
    R.ticket = d_ticket.as<unsigned long long>();
    R.rec_a = d_rec.as<uint4>();
    R.rec_b = agc ? d_rec.as<uint4>() + LEVEL_MAX_TILES : nullptr;
    const long long maxn = (long long)LEVEL_MAX_TILES * LV_TILE;
    size_t done = 0;
    while (done < n) {
        const long long nc = (long long)(n - done) < maxn ? (long long)(n - done) : maxn;
        epoch = (epoch + 1) & 0x3fffffffu;
        if (epoch == 0) {                  // wrapped: clear stale flags
            LRB_CHECK(cudaMemsetAsync(d_rec.get(), 0, rec_bytes(), s));
            epoch = 1;
        }
        const int tiles = (int)((nc + LV_TILE - 1) / LV_TILE);
        const char* xin = (const char*)dx + done * in_size;
        char* yout = (char*)dy + done * out_size;
        const double2* si = d_state[cur].as<const double2>();
        double2* so = d_state[cur ^ 1].as<double2>();
#define LRB_LEVEL(TT, AA)                                                                                           \
        level_kernel<TT, AA><<<tiles, LV_THREADS, 0, s>>>((const TT*)xin, nc, (TT*)yout, P, d_pw.as<double>(), si, so, R, ticket_base, epoch)
        if (complex_data) { if (agc) LRB_LEVEL(float2, true); else LRB_LEVEL(float2, false); }
        else { if (agc) LRB_LEVEL(float, true); else LRB_LEVEL(float, false); }
#undef LRB_LEVEL
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
