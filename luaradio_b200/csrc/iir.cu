// Single-pole IIR (SinglepoleLowpass/Highpass, FMDeemphasis) as a one-pass block-parallel scan.
//
// Reference recurrence (radio/blocks/signal/iirfilter.lua:113-179, liquid iirfilt :79-109):
//     y[n] = (sum_{j<nb} b[j] x[n-j] - a[1] y[n-1]) / a[0]
// With u[n] = sum_j (b[j]/a0) x[n-j] and c = -a1/a0 this is the affine recurrence y[n] = c*y[n-1] + u[n].
// Affine maps compose associatively, and every map here has the same slope c, so the composition over
// a span of k samples has slope c^k (a host-precomputed constant) and only the offsets need scanning:
//   thread: V sequential steps -> warp: Kogge-Stone with slopes c^(V*2^k) -> CTA: Horner over warps ->
//   grid:   decoupled look-back over per-tile (aggregate | inclusive prefix) records.
// The input is read once and the output written once (8 B/sample real, 16 B/sample complex).
#include "common.cuh"
#include <cmath>

namespace lrb {

namespace {

constexpr int IIR_THREADS = 512;
constexpr int IIR_LOGW = 4;                 // log2(warps per CTA)
constexpr int IIR_V = 8;
constexpr int IIR_TILE = IIR_THREADS * IIR_V;
static_assert((32 << IIR_LOGW) == IIR_THREADS, "IIR_LOGW must be log2(warps per CTA)");
constexpr int IIR_MAX_NB = 9;

struct IirParams {
    float b[IIR_MAX_NB];
    int nb;
    float c;
    float cp[5 + IIR_LOGW + 1];   // cp[k] = c^(V * 2^k); cp[5 + LOGW] = c^TILE
};

__device__ __forceinline__ float zero_of(float) { return 0.f; }
__device__ __forceinline__ float2 zero_of(float2) { return make_float2(0.f, 0.f); }
__device__ __forceinline__ float fmas(float c, float v, float a) { return fmaf(c, v, a); }
__device__ __forceinline__ float2 fmas(float c, float2 v, float2 a) { return ffma2(v, make_float2(c, c), a); }
__device__ __forceinline__ float shfl_up_t(float v, int d) { return __shfl_up_sync(0xffffffffu, v, d); }
__device__ __forceinline__ float2 shfl_up_t(float2 v, int d) {
    return make_float2(__shfl_up_sync(0xffffffffu, v.x, d), __shfl_up_sync(0xffffffffu, v.y, d));
}
__device__ __forceinline__ float shfl_xor_t(float v, int d) { return __shfl_xor_sync(0xffffffffu, v, d); }
__device__ __forceinline__ float2 shfl_xor_t(float2 v, int d) {
    return make_float2(__shfl_xor_sync(0xffffffffu, v.x, d), __shfl_xor_sync(0xffffffffu, v.y, d));
}
__device__ __forceinline__ float add_t(float a, float b) { return a + b; }
__device__ __forceinline__ float2 add_t(float2 a, float2 b) { return fadd2(a, b); }
__device__ __forceinline__ float ld_cg(const float* p) { return __ldcg(p); }
__device__ __forceinline__ float2 ld_cg(const float2* p) { return __ldcg(p); }

// LOCAL = true: the pole's memory is shorter than IIR_WARM samples (|c|^IIR_WARM < 1e-12, e.g. FM de-emphasis
// at 220.5 kHz: 0.9413^512 = 4e-14), so a tile needs nothing from its predecessors beyond float32 resolution:
// every CTA restarts IIR_WARM samples early from a zero state and discards that lead-in.  No tickets, flags or
// fences -- a plain streaming kernel.  LOCAL = false: exact decoupled look-back for slow poles.
constexpr int IIR_WARM = 512;
constexpr int IIR_PAY = IIR_THREADS * IIR_V - IIR_WARM;   // payload samples per CTA after the first

// x[b-1 .. b+8) for a real single-pole design (NBT = 2, V = 8): the 8 own samples as two 128-bit loads (32-byte aligned
// per thread; the two instructions of a warp touch the same sectors, so L1 moves 2 KB per KB used instead of the
// 9 KB of nine scalar loads) plus the one sample before.
__device__ __forceinline__ void load9(const float* __restrict__ xb, float (&xv)[9]) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(xb + 1));
    const float4 b = __ldg(reinterpret_cast<const float4*>(xb + 5));
    xv[0] = __ldg(xb);
    xv[1] = a.x; xv[2] = a.y; xv[3] = a.z; xv[4] = a.w;
    xv[5] = b.x; xv[6] = b.y; xv[7] = b.z; xv[8] = b.w;
}
__device__ __forceinline__ void load9(const float2* __restrict__ xb, float2 (&xv)[9]) {
#pragma unroll
    for (int i = 0; i < 9; ++i) xv[i] = __ldg(xb + i);
}

// x[b .. b+8) for a pure pole (NBT = 1): two 128-bit loads
__device__ __forceinline__ void load8(const float* __restrict__ xb, float (&xv)[8]) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(xb));
    const float4 b = __ldg(reinterpret_cast<const float4*>(xb + 4));
    xv[0] = a.x; xv[1] = a.y; xv[2] = a.z; xv[3] = a.w;
    xv[4] = b.x; xv[5] = b.y; xv[6] = b.z; xv[7] = b.w;
}
__device__ __forceinline__ void load8(const float2* __restrict__ xb, float2 (&xv)[8]) {
#pragma unroll
    for (int i = 0; i < 8; ++i) xv[i] = __ldg(xb + i);
}

// NBT: compile-time number of feed-forward taps (2 for every single-pole design of the reference; IIR_MAX_NB = generic).
// With the generic 9-slot loops the kernel was instruction-bound (ncu: 74 % issue-active, ~70 instr per sample).
template <typename T, bool LOCAL, int NBT>
__global__ void __launch_bounds__(IIR_THREADS)
iir1_scan_kernel(const T* __restrict__ x, long long n, T* __restrict__ y, IirParams P,
                 const T* __restrict__ xhist_in, T* __restrict__ xhist_out,
                 const T* __restrict__ ystate_in, T* __restrict__ ystate_out,
                 long long first, int D, int* ticket, volatile int* flags, T* agg, T* pfx, unsigned epoch) {
    __shared__ int s_tile;
    __shared__ int s_off;
    __shared__ long long s_q;
    __shared__ T s_warp[IIR_THREADS / 32];
    __shared__ T s_carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int tile;
    long long span0;                                  // first sample index of this CTA's span
    long long pay0;                                   // first sample index this CTA stores
    // LOCAL: persistent CTAs, grid-stride over the tiles (`epoch` carries the tile count): 15 000 short-lived
    // 4096-sample CTAs spent most of their life in launch/drain latency
    int tile_iter = blockIdx.x;
    const bool vec_ok = (reinterpret_cast<uintptr_t>(x) & 15) == 0;   // tile/thread bases are multiples of 8 samples
    T xnext[IIR_V + NBT - 1];                         // LOCAL: next tile's inputs, fetched while this tile is scanned
    bool have_next = false;
next_tile:
    if constexpr (LOCAL) {
        tile = tile_iter;
        pay0 = tile == 0 ? 0 : (long long)IIR_TILE + (long long)(tile - 1) * IIR_PAY;
        span0 = tile == 0 ? 0 : pay0 - IIR_WARM;
    } else {
        if (tid == 0) s_tile = atomicAdd(ticket, 1);
        __syncthreads();
        tile = s_tile;
        span0 = pay0 = (long long)tile * IIR_TILE;
    }
    if (D > 1 && tid == 0) {
        // decimation phase of this span, once per tile: floor-div/mod of (span0 - first) by D
        long long d0 = span0 - first, qq = d0 / D, rr = d0 - qq * D;
        if (rr < 0) { rr += D; qq -= 1; }
        s_off = (int)rr;
        s_q = qq;
    }
    const long long base = span0 + (long long)tid * IIR_V;
    const int nh = P.nb - 1;

    // ---- u[i] = sum_j b[j] x[i-j] over this thread's V samples (zero beyond n)
    T xv[IIR_V + NBT - 1];
    if (LOCAL && have_next) {
#pragma unroll
        for (int i = 0; i < IIR_V + NBT - 1; ++i) xv[i] = xnext[i];
    } else if (base >= NBT - 1 && base + IIR_V <= n) {
        // interior thread: no bounds checks
        const T* xb = x + (base - (NBT - 1));
        if constexpr (NBT == 2 && IIR_V == 8) {
            if (vec_ok) load9(xb, xv);
            else {
#pragma unroll
                for (int i = 0; i < 9; ++i) xv[i] = __ldg(xb + i);
            }
        } else if constexpr (NBT == 1 && IIR_V == 8) {
            if (vec_ok) load8(xb, xv);
            else {
#pragma unroll
                for (int i = 0; i < 8; ++i) xv[i] = __ldg(xb + i);
            }
        } else {
#pragma unroll
            for (int i = 0; i < IIR_V + NBT - 1; ++i) xv[i] = __ldg(xb + i);
        }
    } else {
#pragma unroll
        for (int i = 0; i < IIR_V + NBT - 1; ++i) {
            long long idx = base + i - (NBT - 1);
            T v = zero_of(T());
            if (i >= NBT - 1 - nh) {
                if (idx >= 0) { if (idx < n) v = __ldg(x + idx); }
                else if (nh + idx >= 0) v = __ldg(xhist_in + (nh + idx));
            }
            xv[i] = v;
        }
    }
    T yl[IIR_V];
#pragma unroll
    for (int i = 0; i < IIR_V; ++i) {
        T u = zero_of(T());
#pragma unroll
        for (int j = 0; j < NBT; ++j)
            if (NBT < IIR_MAX_NB || j < P.nb) u = fmas(P.b[j], xv[i + NBT - 1 - j], u);
        yl[i] = (i == 0) ? u : fmas(P.c, yl[i - 1], u);
    }

    if constexpr (LOCAL) {
        // prefetch the inputs of this CTA's next tile (interior threads only; the rest reload with bounds checks)
        have_next = false;
        const int nt = tile_iter + gridDim.x;
        if (nt < (int)epoch) {
            const long long nb0 = (long long)IIR_TILE + (long long)(nt - 1) * IIR_PAY - IIR_WARM + (long long)tid * IIR_V;
            if (nb0 >= NBT - 1 && nb0 + IIR_V <= n) {
                const T* xb = x + (nb0 - (NBT - 1));
                if constexpr (NBT == 2 && IIR_V == 8) {
                    if (vec_ok) load9(xb, xnext);
                    else {
#pragma unroll
                        for (int i = 0; i < 9; ++i) xnext[i] = __ldg(xb + i);
                    }
                } else if constexpr (NBT == 1 && IIR_V == 8) {
                    if (vec_ok) load8(xb, xnext);
                    else {
#pragma unroll
                        for (int i = 0; i < 8; ++i) xnext[i] = __ldg(xb + i);
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < IIR_V + NBT - 1; ++i) xnext[i] = __ldg(xb + i);
                }
                have_next = true;
            }
        }
    }

    // ---- warp scan of the per-thread zero-state end values
    T B = yl[IIR_V - 1];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        T o = shfl_up_t(B, 1 << k);
        if (lane >= (1 << k)) B = fmas(P.cp[k], o, B);
    }
    if (lane == 31) s_warp[warp] = B;
    T prevB = shfl_up_t(B, 1);                      // inclusive value of lane-1 (zero-state from warp start)
    if (lane == 0) prevB = zero_of(T());
    __syncthreads();
    const int dec_off = (D > 1) ? s_off : 0;        // read here: thread 0 rewrites them at the top of its next pass
    const long long dec_q = (D > 1) ? s_q : 0;
    T carryW = zero_of(T());                        // value at the end of warp-1, zero-state from tile start
    for (int w = 0; w < warp; ++w) carryW = fmas(P.cp[5], carryW, s_warp[w]);
    float f_lane = 1.f;                             // c^(V*lane)
#pragma unroll
    for (int k = 0; k < 5; ++k) if (lane & (1 << k)) f_lane *= P.cp[k];
    const T excl = fmas(f_lane, carryW, prevB);     // y just before this thread's first sample, zero-state from tile start

    // ---- tile aggregate + decoupled look-back.  The whole of warp 0 walks back 32 predecessor tiles at a
    // time (warp-uniform control flow: a single spinning lane in front of __syncthreads() is NOT safe).
    __shared__ T s_agg;
    if (tid == IIR_THREADS - 1) s_agg = fmas(f_lane * P.cp[0], carryW, B);
    __syncthreads();
    if constexpr (LOCAL) {
        if (tid == 0) s_carry = (tile == 0) ? __ldg(ystate_in) : zero_of(T());
    } else if (warp == 0) {
        const float cT = P.cp[5 + IIR_LOGW];
        T carry_in;
        if (tile == 0) {
            carry_in = __ldg(ystate_in);
        } else {
            if (lane == 0) {
                agg[tile] = s_agg;
                __threadfence();
                flags[tile] = (int)(epoch * 4u + 1u);
            }
            __syncwarp();
            float wl = 1.f, pw = cT;                // wl = cT^lane, pw -> cT^32
#pragma unroll
            for (int k = 0; k < 5; ++k) { if (lane & (1 << k)) wl *= pw; pw *= pw; }
            T acc = zero_of(T());
            float mult = 1.f;
            int jbase = tile - 1;
            while (true) {
                const int j = jbase - lane;
                // a predecessor whose weight c^(distance) is below float32 resolution cannot change the result:
                // it is treated as a (zero) prefix, which cuts the serial tile-to-tile dependency for every
                // pole whose memory is shorter than a tile (FM de-emphasis: c^4096 underflows to 0).
                const bool dead = fabsf(wl * mult) < 1e-12f;
                int f = 0;
                T v = zero_of(T());
                if (j >= 0 && !dead) {
                    do { f = flags[j]; } while ((unsigned)f >> 2 != epoch);
                    __threadfence();
                    v = ((f & 3) == 2) ? ld_cg(pfx + j) : ld_cg(agg + j);
                }
                const unsigned pmask = __ballot_sync(0xffffffffu, j >= 0 && (dead || (f & 3) == 2));
                const int last = pmask ? (__ffs(pmask) - 1) : 31;    // nearest tile that ends the walk
                T contrib = (j >= 0 && lane <= last) ? fmas(wl, v, zero_of(T())) : zero_of(T());
#pragma unroll
                for (int off = 16; off >= 1; off >>= 1) contrib = add_t(contrib, shfl_xor_t(contrib, off));
                acc = fmas(mult, contrib, acc);
                if (pmask) break;                   // tile 0 always publishes a prefix, so this terminates
                mult *= pw;
                jbase -= 32;
            }
            carry_in = acc;
        }
        if (lane == 0) {
            pfx[tile] = fmas(cT, carry_in, s_agg);
            __threadfence();
            flags[tile] = (int)(epoch * 4u + 2u);
            s_carry = carry_in;
        }
    }
    __syncthreads();
    const T carry_in = s_carry;
    float f_thread = f_lane;                        // c^(V*tid)
#pragma unroll
    for (int k = 0; k < IIR_LOGW; ++k) if (warp & (1 << k)) f_thread *= P.cp[5 + k];
    const T carry_t = fmas(f_thread, carry_in, excl);

    // ---- outputs y[i] = yl[i] + c^(i+1) * carry_t, stored with tile-relative 32-bit bookkeeping.  (The first
    // versions did a 64-bit division, then several 64-bit compares, per sample: ncu showed 68 % of the executed
    // instructions after the last barrier.)  rel = index relative to span0; [lo, hi) is what this CTA stores.
    const int rel0 = tid * IIR_V;
    const int lo = (int)(pay0 - span0);
    const long long remain = n - span0;
    const int hi = remain < (long long)IIR_TILE ? (int)remain : IIR_TILE;
    T vals[IIR_V];
    {
        float cpow = P.c;
#pragma unroll
        for (int i = 0; i < IIR_V; ++i) { vals[i] = fmas(cpow, carry_t, yl[i]); cpow *= P.c; }
    }
    if (D == 1) {
        T* yo = y + span0 + rel0;
        if (rel0 >= lo && rel0 + IIR_V <= hi) {
#pragma unroll
            for (int i = 0; i < IIR_V; ++i) yo[i] = vals[i];
        } else {
#pragma unroll
            for (int i = 0; i < IIR_V; ++i) if (rel0 + i >= lo && rel0 + i < hi) yo[i] = vals[i];
        }
    } else {
        // kept samples: (span0 + rel - first) % D == 0  <=>  (rel + s_off) % D == 0, output index s_q + (rel + s_off) / D
        const unsigned e = (unsigned)(rel0 + dec_off);
        const unsigned q = e / (unsigned)D, r = e - q * (unsigned)D;
        int knext = r ? (int)((unsigned)D - r) : 0;               // first kept sample of this thread (offset in 0..)
        T* yo = y + (dec_q + (long long)q + (r ? 1 : 0));
#pragma unroll
        for (int i = 0; i < IIR_V; ++i) {
            if (i == knext) {
                if (rel0 + i >= lo && rel0 + i < hi) *yo = vals[i];
                ++yo;
                knext += D;
            }
        }
    }
    if (remain <= (long long)IIR_TILE && hi - 1 >= rel0 && hi - 1 < rel0 + IIR_V) {
        // the stream's last sample lives in this thread: carried output state
#pragma unroll
        for (int i = 0; i < IIR_V; ++i) if (rel0 + i == hi - 1) *ystate_out = vals[i];
    }
    // ---- carried input history for the next call: last nb-1 inputs of [xhist_in | x]
    if (tile == 0 && tid < nh) {
        long long i = n - nh + tid;
        xhist_out[tid] = (i >= 0) ? x[i] : xhist_in[nh + i];
    }
    if constexpr (LOCAL) {
        tile_iter += gridDim.x;
        if (tile_iter < (int)epoch) goto next_tile;   // (the three barriers of the next pass order the shared scratch)
    }
}

}  // namespace

int iir_work_alloc(IirScanWork* w, int elem_size) {
    w->max_tiles = 1 << 15;   // 128 Mi samples per launch
    if (w->ticket.reserve(sizeof(int)) != 0 || w->flags.alloc_zeroed(sizeof(int) * w->max_tiles) != 0 ||
        w->agg.reserve((size_t)elem_size * w->max_tiles) != 0 || w->pfx.reserve((size_t)elem_size * w->max_tiles) != 0)
        return -1;
    w->epoch = 0;
    return 0;
}

long long iir_max_per_launch(const IirScanWork& w) { return (long long)w.max_tiles * IIR_TILE; }

int launch_iir1(bool complex_data, const void* x, long long n, void* y, const float* b_host, int nb, float c,
                const void* xhist_in, void* xhist_out, const void* ystate_in, void* ystate_out,
                long long first, int D, IirScanWork* w, cudaStream_t s) {
    if (n <= 0) return 0;
    if (nb < 1 || nb > IIR_MAX_NB) { set_error("iir: nb must be in 1..%d", IIR_MAX_NB); return -1; }
    if (n > iir_max_per_launch(*w)) { set_error("iir: chunk too large for one launch"); return -1; }
    IirParams P;
    for (int j = 0; j < IIR_MAX_NB; ++j) P.b[j] = j < nb ? b_host[j] : 0.f;
    P.nb = nb;
    P.c = c;
    double cd = (double)c, p = 1.0;
    for (int i = 0; i < IIR_V; ++i) p *= cd;      // c^V
    for (int k = 0; k < 5 + IIR_LOGW + 1; ++k) { P.cp[k] = (float)p; p = p * p; }
    const bool local = std::pow(std::fabs(cd), (double)IIR_WARM) < 1e-12;
    if (local) {
        int tiles = n <= IIR_TILE ? 1 : 1 + (int)((n - IIR_TILE + IIR_PAY - 1) / IIR_PAY);
        int grid = ctx().sm_count * 2;
        if (grid > tiles) grid = tiles;
#define LRB_IIR_LOCAL(TT, NN)                                                                                   \
        iir1_scan_kernel<TT, true, NN><<<grid, IIR_THREADS, 0, s>>>((const TT*)x, n, (TT*)y, P, (const TT*)xhist_in, \
            (TT*)xhist_out, (const TT*)ystate_in, (TT*)ystate_out, first, D, nullptr, nullptr, nullptr, nullptr, (unsigned)tiles)
        if (complex_data) { if (nb == 2) LRB_IIR_LOCAL(float2, 2); else if (nb == 1) LRB_IIR_LOCAL(float2, 1); else LRB_IIR_LOCAL(float2, IIR_MAX_NB); }
        else { if (nb == 2) LRB_IIR_LOCAL(float, 2); else if (nb == 1) LRB_IIR_LOCAL(float, 1); else LRB_IIR_LOCAL(float, IIR_MAX_NB); }
#undef LRB_IIR_LOCAL
        count_launch();
        LRB_CHECK(cudaGetLastError());
        return 0;
    }
    w->epoch = (w->epoch + 1) & 0x3fffffffu;
    if (w->epoch == 0) {                          // wrapped: clear stale flags
        LRB_CHECK(cudaMemsetAsync(w->flags.get(), 0, sizeof(int) * w->max_tiles, s));
        w->epoch = 1;
    }
    LRB_CHECK(cudaMemsetAsync(w->ticket.get(), 0, sizeof(int), s));
    int tiles = (int)((n + IIR_TILE - 1) / IIR_TILE);
#define LRB_IIR_SCAN(TT, NN)                                                                                    \
    iir1_scan_kernel<TT, false, NN><<<tiles, IIR_THREADS, 0, s>>>((const TT*)x, n, (TT*)y, P, (const TT*)xhist_in,  \
        (TT*)xhist_out, (const TT*)ystate_in, (TT*)ystate_out, first, D, w->ticket.as<int>(), w->flags.as<int>(), w->agg.as<TT>(), w->pfx.as<TT>(), w->epoch)
    if (complex_data) { if (nb == 2) LRB_IIR_SCAN(float2, 2); else if (nb == 1) LRB_IIR_SCAN(float2, 1); else LRB_IIR_SCAN(float2, IIR_MAX_NB); }
    else { if (nb == 2) LRB_IIR_SCAN(float, 2); else if (nb == 1) LRB_IIR_SCAN(float, 1); else LRB_IIR_SCAN(float, IIR_MAX_NB); }
#undef LRB_IIR_SCAN
    count_launch();
    LRB_CHECK(cudaGetLastError());
    return 0;
}

}  // namespace lrb

// =============================================================================================
// General-order IIRFilterBlock (iirfilter.lua:113-179): direct form I,
//     y[n] = (sum_{j<nb} b[j] x[n-j] - sum_{1<=j<na} a[j] y[n-j]) / a[0]
// Time-parallel with a measured warm-up: the host simulates the impulse response of 1/A(z) in float64 and finds
// the length W after which it stays below 1e-10 of its peak; the stream is cut into chunks, every thread runs the
// sequential recurrence over its chunk starting W samples early from (true past inputs, zero past outputs), and
// only stores its own chunk.  Chunk 0 starts from the carried state, so short calls (the reference's 256-sample
// vectors, or sample-by-sample streaming) are the plain sequential recurrence, bit for bit.  A filter whose
// response never decays gets W = infinity -> one chunk.  Not on the WBFM chain (single-pole de-emphasis uses the
// scan kernel above); this is the catch-all that makes every IIRFilterBlock signature run on the GPU.
// =============================================================================================
namespace lrb {

namespace {

constexpr int IIRG_MAX = 10;

struct IirGenParams {
    float b[IIRG_MAX];     // b[j] / a0
    float a[IIRG_MAX];     // a[j] / a0 (a[0] unused)
    int nb, na;
};

template <typename T>
__global__ void __launch_bounds__(128)
iir_general_kernel(const T* __restrict__ x, long long n, T* __restrict__ y, IirGenParams P,
                   const T* __restrict__ xhist, const T* __restrict__ yhist, long long chunk, long long warm) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long start = g * chunk;
    if (start >= n) return;
    const long long end = (start + chunk < n) ? start + chunk : n;
    long long begin = start - warm;
    const bool from_state = begin <= 0;
    if (from_state) begin = 0;
    T xs[IIRG_MAX], ys[IIRG_MAX];
#pragma unroll
    for (int j = 0; j < IIRG_MAX; ++j) { xs[j] = zero_of(T()); ys[j] = zero_of(T()); }
    const int nh = P.nb - 1, ny = P.na - 1;
    // xs[j] = x[i-1-j], ys[j] = y[i-1-j] at i = begin
#pragma unroll
    for (int j = 0; j < IIRG_MAX - 1; ++j) {
        if (j < nh) {
            const long long i = begin - 1 - j;
            xs[j] = (i >= 0) ? __ldg(x + i) : ((nh + i >= 0) ? __ldg(xhist + (nh + i)) : zero_of(T()));
        }
        if (j < ny && from_state) ys[j] = __ldg(yhist + (ny - 1 - j));
    }
    for (long long i = begin; i < end; ++i) {
        const T xi = __ldg(x + i);
        T acc = fmas(P.b[0], xi, zero_of(T()));
#pragma unroll
        for (int j = 1; j < IIRG_MAX; ++j) if (j < P.nb) acc = fmas(P.b[j], xs[j - 1], acc);
#pragma unroll
        for (int j = 1; j < IIRG_MAX; ++j) if (j < P.na) acc = fmas(-P.a[j], ys[j - 1], acc);
#pragma unroll
        for (int j = IIRG_MAX - 1; j > 0; --j) { xs[j] = xs[j - 1]; ys[j] = ys[j - 1]; }
        xs[0] = xi;
        ys[0] = acc;
        if (i >= start) y[i] = acc;
    }
}

}  // namespace

int launch_iir_general(bool complex_data, const void* x, long long n, void* y, const float* b, int nb, const float* a, int na,
                       const void* xhist, const void* yhist, long long warm, cudaStream_t s) {
    if (n <= 0) return 0;
    IirGenParams P;
    for (int j = 0; j < IIRG_MAX; ++j) { P.b[j] = j < nb ? b[j] : 0.f; P.a[j] = j < na ? a[j] : 0.f; }
    P.nb = nb;
    P.na = na;
    long long chunk = n, w = warm;
    if (warm >= 0 && warm < n) {
        chunk = 4 * warm > 512 ? 4 * warm : 512;
    } else {
        w = n;                                       // no decay information: one sequential chunk
    }
    const long long nchunks = (n + chunk - 1) / chunk;
    const int threads = 128;
    const long long blocks = (nchunks + threads - 1) / threads;
    if (complex_data)
        iir_general_kernel<float2><<<(unsigned)blocks, threads, 0, s>>>((const float2*)x, n, (float2*)y, P, (const float2*)xhist, (const float2*)yhist, chunk, w);
    else
        iir_general_kernel<float><<<(unsigned)blocks, threads, 0, s>>>((const float*)x, n, (float*)y, P, (const float*)xhist, (const float*)yhist, chunk, w);
    count_launch();
    LRB_CHECK(cudaGetLastError());
    return 0;
}

}  // namespace lrb
