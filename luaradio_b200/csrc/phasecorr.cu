// BinaryPhaseCorrectorBlock as a reduce / scan / apply over 2048-sample tiles.
//
// Reference recurrence (radio/blocks/signal/binaryphasecorrector.lua:36-77), in Lua numbers (double) unless noted:
//     at every global sample index k*I (measurement k):
//         phi  = atan2f(im, re), folded into (-pi/2, pi/2] with math.pi
//         avg  = (avg + phi/N) - last/N          last = float32(phi) of measurement k-N, 0 while the window fills
//     y[i] = x[i] * ComplexFloat32(cos(-avg), sin(-avg))      (avg after the last measurement at or before i)
// The average is a prefix sum of the per-measurement terms +phi/N, -last/N.  Its association may differ from the
// reference's; every term is the reference's own double.
//
// Three launches per call of up to 256 Mi samples, no per-sample or per-measurement scratch:
//   pc_reduce_kernel  one warp per tile sums the terms of the tile's measurements.  It reads only the measurement samples
//                     (one 32 B sector each) and the sample N*I earlier, or the carried window for the call's first N.
//                     CTAs past the tiles write the next call's window (slot k mod N = float32 phi of the newest
//                     measurement k of this call with that slot, else the carried value) into the other ping-pong buffer.
//   pc_scan_kernel    one CTA scans the tile sums, seeded with the carried average: each tile's starting average, and
//                     the carried average for the next call.
//   pc_apply_kernel   each thread owns 8 samples: it sums its own terms, a CTA scan gives its starting average, and it
//                     re-walks its samples in the reference's order, forming one phasor per measurement (double sincos,
//                     rounded to float32) and the product in double, rounded once (complexfloat32.lua:79-81).
// x is read twice in the worst case (I = 1), once plus one sector per I samples otherwise; y is written once.
#include "../../include/lrb200.h"
#include "common.cuh"
#include "blocks.h"

namespace lrb {

namespace {

constexpr int PC_THREADS = 256;
constexpr int PC_V = 8;                            // samples per thread in the apply pass (16: 110 registers, 2 CTAs per SM)
constexpr int PC_TILE = PC_THREADS * PC_V;
constexpr int PC_SCAN_THREADS = 1024;
constexpr int PC_REDUCE_TILES = PC_THREADS / 32;   // tiles per reduce CTA, one per warp

struct PcParams {
    const float2* x;
    float2* y;
    long long n;
    unsigned N, I;
    long long r0;                  // local index of the call's first measurement
    long long K;                   // measurements in the call
    unsigned k0n;                  // window slot of the call's first measurement: its global number mod N
    const double* st_in;           // carried state: {average, window[N] as float32}
    double* st_out;
    double* tsum;                  // per-tile sums of the terms
    double* tpfx;                  // per-tile starting averages
    int tiles;
};

__device__ __forceinline__ const float* window_of(const double* st) { return reinterpret_cast<const float*>(st + 1); }

// binaryphasecorrector.lua:47-51: ComplexFloat32:arg() is atan2f; the fold runs in double with math.pi
__device__ __forceinline__ double fold(float a) {
    constexpr double pi = 3.141592653589793;
    double phi = (double)a;
    phi = phi < -pi / 2 ? __dadd_rn(phi, pi) : phi;
    phi = phi > pi / 2 ? __dsub_rn(phi, pi) : phi;
    return phi;
}
__device__ __forceinline__ float arg_of(float2 v) { return atan2f(v.y, v.x); }

// first measurement j (local) at or after local sample index p
__device__ __forceinline__ long long first_meas(const PcParams& P, long long p) {
    return p <= P.r0 ? 0 : (p - P.r0 + P.I - 1) / P.I;
}

// the window value measurement j replaces: float32 phi of measurement j - N, from x or from the carried window
__device__ __forceinline__ float last_of(const PcParams& P, long long j) {
    if (j >= (long long)P.N) return __double2float_rn(fold(arg_of(__ldg(P.x + P.r0 + (j - P.N) * (long long)P.I))));
    unsigned s = P.k0n + (unsigned)j;
    if (s >= P.N) s -= P.N;
    return window_of(P.st_in)[s];
}

__device__ __forceinline__ double add_terms(double a, double phi, float last, unsigned N) {
    return __dsub_rn(__dadd_rn(a, __ddiv_rn(phi, (double)N)), __ddiv_rn((double)last, (double)N));
}

// exclusive prefix of v over the CTA in thread order; *total = the CTA's sum
template <int THREADS>
__device__ __forceinline__ double cta_exclusive(double v, double* s_warp, double* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double inc = v;
#pragma unroll
    for (int k = 1; k < 32; k <<= 1) {
        const double o = __shfl_up_sync(0xffffffffu, inc, k);
        if (lane >= k) inc += o;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    double before = 0.0, all = 0.0;
    for (int w = 0; w < THREADS / 32; ++w) {
        if (w < warp) before += s_warp[w];
        all += s_warp[w];
    }
    *total = all;
    return before + (inc - v);
}

__global__ void __launch_bounds__(PC_THREADS) pc_reduce_kernel(PcParams P) {
    const int tid = threadIdx.x;
    const int rblocks = (P.tiles + PC_REDUCE_TILES - 1) / PC_REDUCE_TILES;
    if ((int)blockIdx.x >= rblocks) {
        // the next call's window
        const unsigned s = (blockIdx.x - (unsigned)rblocks) * PC_THREADS + tid;
        if (s >= P.N) return;
        const unsigned jl = s >= P.k0n ? s - P.k0n : s + P.N - P.k0n;    // first local j with slot s
        float v = window_of(P.st_in)[s];
        if ((long long)jl < P.K) {
            const long long j = jl + (P.K - 1 - jl) / P.N * P.N;         // the newest one
            v = __double2float_rn(fold(arg_of(__ldg(P.x + P.r0 + j * (long long)P.I))));
        }
        reinterpret_cast<float*>(P.st_out + 1)[s] = v;
        return;
    }
    // one warp per tile: a tile holds TILE / I measurements, 128 for I = 32 -- too few to keep a whole CTA busy
    const int lane = tid & 31, tile = blockIdx.x * PC_REDUCE_TILES + (tid >> 5);
    if (tile >= P.tiles) return;
    const long long t0 = (long long)tile * PC_TILE;
    const long long t1 = t0 + PC_TILE < P.n ? t0 + PC_TILE : P.n;
    const long long j1 = first_meas(P, t1);
    double acc = 0.0;
    for (long long j = first_meas(P, t0) + lane; j < j1; j += 32)
        acc = add_terms(acc, fold(arg_of(__ldg(P.x + P.r0 + j * (long long)P.I))), last_of(P, j), P.N);
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) P.tsum[tile] = acc;
}

__global__ void __launch_bounds__(PC_SCAN_THREADS) pc_scan_kernel(PcParams P) {
    __shared__ double s_warp[PC_SCAN_THREADS / 32];
    const int per = (P.tiles + PC_SCAN_THREADS - 1) / PC_SCAN_THREADS;
    const int b = threadIdx.x * per, e = b + per < P.tiles ? b + per : P.tiles;
    // each thread's span is read 8 values at a time, the loads issued before the sums: one memory latency per 8 tiles
    constexpr int U = 8;
    double v = 0.0;
    for (int t0 = b; t0 < e; t0 += U) {
        double w[U];
#pragma unroll
        for (int k = 0; k < U; ++k) w[k] = t0 + k < e ? P.tsum[t0 + k] : 0.0;
#pragma unroll
        for (int k = 0; k < U; ++k) v += w[k];
    }
    double total;
    const double avg = P.st_in[0];
    double run = cta_exclusive<PC_SCAN_THREADS>(v, s_warp, &total);
    for (int t0 = b; t0 < e; t0 += U) {
        double w[U];
#pragma unroll
        for (int k = 0; k < U; ++k) w[k] = t0 + k < e ? P.tsum[t0 + k] : 0.0;
#pragma unroll
        for (int k = 0; k < U; ++k) {
            if (t0 + k < e) P.tpfx[t0 + k] = avg + run;
            run += w[k];
        }
    }
    if (threadIdx.x == 0) P.st_out[0] = avg + total;
}

__global__ void __launch_bounds__(PC_THREADS, 3) pc_apply_kernel(PcParams P) {
    __shared__ double s_warp[PC_THREADS / 32];
    const int tid = threadIdx.x;
    const long long base = (long long)blockIdx.x * PC_TILE + (long long)tid * PC_V;

    float2 xv[PC_V];
    const bool vec = base + PC_V <= P.n && ((reinterpret_cast<uintptr_t>(P.x) | reinterpret_cast<uintptr_t>(P.y)) & 15) == 0;
    if (vec) {
#pragma unroll
        for (int k = 0; k < PC_V / 2; ++k) {
            const float4 u = __ldcs(reinterpret_cast<const float4*>(P.x + base) + k);
            xv[2 * k] = make_float2(u.x, u.y);
            xv[2 * k + 1] = make_float2(u.z, u.w);
        }
    } else {
#pragma unroll
        for (int i = 0; i < PC_V; ++i) xv[i] = base + i < P.n ? P.x[base + i] : make_float2(0.f, 0.f);
    }

    // the thread's measurements: their angles, the window values they replace, and the sum of their terms
    long long j = first_meas(P, base);
    long long pm = j < P.K ? P.r0 + j * (long long)P.I : P.n;             // next measurement's local index
    unsigned mmask = 0;
    float at[PC_V], lst[PC_V];
    double acc = 0.0;
#pragma unroll
    for (int i = 0; i < PC_V; ++i) {
        at[i] = 0.f;
        lst[i] = 0.f;
        if (base + i == pm && pm < P.n) {
            at[i] = arg_of(xv[i]);
            lst[i] = last_of(P, j);
            acc = add_terms(acc, fold(at[i]), lst[i], P.N);
            mmask |= 1u << i;
            pm += P.I;
            ++j;
        }
    }
    double total;
    double avg = P.tpfx[blockIdx.x] + cta_exclusive<PC_THREADS>(acc, s_warp, &total);

    double pr = 1.0, pi = 0.0;                     // the float32 phasor, held as doubles: converted once per measurement
#pragma unroll
    for (int i = 0; i < PC_V; ++i) {
        const bool m = (mmask >> i) & 1u;
        if (m) avg = add_terms(avg, fold(at[i]), lst[i], P.N);
        if (i == 0 || m) {
            double sn, cs;
            sincos(-avg, &sn, &cs);
            pr = (double)__double2float_rn(cs);
            pi = (double)__double2float_rn(sn);
        }
        // complexfloat32.lua:79-81: float32 operands, products and sums in double, one rounding per component
        const double xr = xv[i].x, xi = xv[i].y;
        xv[i] = make_float2(__double2float_rn(__dsub_rn(__dmul_rn(xr, pr), __dmul_rn(xi, pi))),
                            __double2float_rn(__dadd_rn(__dmul_rn(xr, pi), __dmul_rn(xi, pr))));
    }

    if (vec) {
#pragma unroll
        for (int k = 0; k < PC_V / 2; ++k)
            __stcs(reinterpret_cast<float4*>(P.y + base) + k, make_float4(xv[2 * k].x, xv[2 * k].y, xv[2 * k + 1].x, xv[2 * k + 1].y));
    } else {
#pragma unroll
        for (int i = 0; i < PC_V; ++i) if (base + i < P.n) P.y[base + i] = xv[i];
    }
}

}  // namespace

// ---------------------------------------------------------------------------------------------
PhaseCorrectorBlock::PhaseCorrectorBlock(unsigned num_samples, unsigned sample_interval, bool dev) : Block("phasecorr", 8, 8, dev) {
    N = num_samples;
    I = sample_interval;
}

int PhaseCorrectorBlock::init() {
    if (carry(d_state, sizeof(double) + sizeof(float) * (size_t)N, cur) != 0) return -1;
    return d_tiles.reserve(2 * sizeof(double) * PC_MAX_TILES);
}

long long PhaseCorrectorBlock::memory_in() const {
    // a cold start N*I samples back has filled the window for every later output (DESIGN.md §5)
    const unsigned long long m = (unsigned long long)N * I;
    return m > (unsigned long long)LLONG_MAX ? -1 : (long long)m;
}

int PhaseCorrectorBlock::run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) {
    *n_out = n;
    const long long maxn = (long long)PC_MAX_TILES * PC_TILE;
    size_t done = 0;
    while (done < n) {
        const long long nc = (long long)(n - done) < maxn ? (long long)(n - done) : maxn;
        PcParams P;
        P.x = (const float2*)dx + done;
        P.y = (float2*)dy + done;
        P.n = nc;
        P.N = N;
        P.I = I;
        P.r0 = (long long)((I - consumed % I) % I);
        P.K = nc > P.r0 ? (nc - P.r0 - 1) / I + 1 : 0;
        P.k0n = (unsigned)(((consumed + I - 1) / I) % N);
        P.st_in = d_state[cur].as<const double>();
        P.st_out = d_state[cur ^ 1].as<double>();
        P.tsum = d_tiles.as<double>();
        P.tpfx = d_tiles.as<double>() + PC_MAX_TILES;
        P.tiles = (int)((nc + PC_TILE - 1) / PC_TILE);
        const unsigned wblocks = (N + PC_THREADS - 1) / PC_THREADS;
        const unsigned rblocks = (unsigned)((P.tiles + PC_REDUCE_TILES - 1) / PC_REDUCE_TILES);
        pc_reduce_kernel<<<rblocks + wblocks, PC_THREADS, 0, s>>>(P);
        pc_scan_kernel<<<1, PC_SCAN_THREADS, 0, s>>>(P);
        pc_apply_kernel<<<P.tiles, PC_THREADS, 0, s>>>(P);
        count_launch(3);
        LRB_CHECK(cudaGetLastError());
        cur ^= 1;
        consumed += (uint64_t)nc;
        done += (size_t)nc;
    }
    return 0;
}

}  // namespace lrb
