// PLLBlock (radio/blocks/signal/pll.lua:140-170): a NONLINEAR recurrence -- phase detector atan2f(x conj(vco)),
// second-order loop filter, frequency clamp, phase wrap -- restated operation by operation (Lua numbers are doubles; the
// VCO output, the phase-detector product and the error are rounded to float32 where the reference stores them in
// ComplexFloat32 / Float32 cells).  state = {phi_locked, phi_multiplied, freq_locked}.  Mode 0 (pll_kernel): one thread
// runs the stream in order, exact for any input, locked or not, at a few MS/s (the reference's Lua loop: 5 MS/s on its
// i5).  Mode 1 (lrb200_pll_set_mode(q, 1)) runs calls of 2 L samples or more in the verified chunk-parallel form below.
// tests/pll_ref.py models both forms and derives the thresholds and tolerances.
#include "../../include/lrb200.h"
#include "common.cuh"
#include "blocks.h"

#include <cmath>

namespace lrb {

namespace {

constexpr double PLL_TWO_PI = 6.283185307179586476925286766559;       // fl(2 pi): the wraps subtract it exactly

struct PllParams { double alpha, beta, fmin, fmax, mult; };

// The loop step on phi and freq: returns e and leaves phi updated and wrapped and freq = freq' (the clamp is the
// caller's, after phi_multiplied's step has used freq').
__device__ __forceinline__ float pll_step(float2 xv, double& phi, double& freq, const PllParams& P) {
    double s, c;
    sincos(phi, &s, &c);
    const float vr = (float)c, vi = (float)s;
    // x * conj(vco), each component computed in double and stored as float32 (complexfloat32.lua:79-81)
    const float pr = (float)((double)xv.x * (double)vr - (double)xv.y * (double)(-vi));
    const float pi = (float)((double)xv.x * (double)(-vi) + (double)xv.y * (double)vr);
    const float e = atan2f(pi, pr);
    freq = freq + P.beta * (double)e;
    phi = phi + freq + P.alpha * (double)e;
    phi = phi > PLL_TWO_PI ? phi - PLL_TWO_PI : phi;
    phi = phi < -PLL_TWO_PI ? phi + PLL_TWO_PI : phi;
    return e;
}

__device__ __forceinline__ void pll_clamp(double& freq, const PllParams& P) {
    freq = freq > P.fmax ? P.fmax : freq;
    freq = freq < P.fmin ? P.fmin : freq;
}

// phi_multiplied's step, from freq'
__device__ __forceinline__ void pll_advance(double& phim, double freq, double e, const PllParams& P) {
    phim = phim + freq * P.mult + P.alpha * e;
    phim = phim > PLL_TWO_PI ? phim - PLL_TWO_PI : phim;
    phim = phim < -PLL_TWO_PI ? phim + PLL_TWO_PI : phim;
}

__global__ void pll_kernel(const float2* __restrict__ x, long long n, float2* __restrict__ out, float* __restrict__ err,
                           double* __restrict__ state, PllParams P) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    double phi = state[0], phim = state[1], freq = state[2];
    for (long long i = 0; i < n; ++i) {
        double s, c;
        sincos(phim, &s, &c);
        out[i] = make_float2((float)c, (float)s);
        const float e = pll_step(x[i], phi, freq, P);
        err[i] = e;
        pll_advance(phim, freq, (double)e, P);
        pll_clamp(freq, P);
    }
    state[0] = phi; state[1] = phim; state[2] = freq;
}

// ---- the chunk-parallel form, verified against the carried loop state.  From a phase guess arg(x) and the centre
// frequency the second-order loop converges to the stream's own (phi_locked, freq_locked) trajectory within W = 24 /
// (zeta * loop bandwidth) samples when the loop is locked, so every chunk is first simulated by its own thread after a
// W-sample lead-in (chunk 0 starts from the carried state and is exact).  On input that gives the loop nothing to pull
// with (zeros, noise, acquisition) the lead-in does not get there, so one thread then walks the chunks in stream order
// (pll_verify_kernel) and compares each chunk's speculated start (phi0, freq0) with the true end state of the chunk
// before it; a chunk that misses it by more than (dphi, dfreq) is run again from the true state with the sequential
// recurrence, which rewrites its errors and its summary.  phi_multiplied is NOT a function of the locked state (it
// integrates multiplier * freq' + alpha * error over the whole past), so it is carried across the chunks instead: each
// chunk's advance dP is summed in the sequential kernel's own expression and wrapped to +-2 pi at every step, the bases
// are summed and wrapped once per chunk, and the output pass advances phi_multiplied from its chunk's base exactly as
// pll_kernel does.  Every partial sum stays below 4 pi, so the rounding per sample is that of the sequential kernel: no
// sum grows with the call.
struct PllChunk { double phi0, freq0, dP, phi_end, freq_end, base; };

// Samples [start, end) from (phi, freq) with the sequential recurrence: writes their errors and returns the chunk's
// start state, advance dP and end state (base 0: pll_verify_kernel sums the bases).
__device__ __forceinline__ PllChunk pll_chunk(const float2* __restrict__ x, float* __restrict__ err, long long start,
                                              long long end, double phi, double freq, const PllParams& P) {
    const double phi0 = phi, freq0 = freq;
    double dP = 0.0;
    for (long long i = start; i < end; ++i) {
        const float e = pll_step(x[i], phi, freq, P);
        err[i] = e;
        pll_advance(dP, freq, (double)e, P);
        pll_clamp(freq, P);
    }
    return PllChunk{phi0, freq0, dP, phi, freq, 0.0};
}

__global__ void __launch_bounds__(128)
pll_sim_kernel(const float2* __restrict__ x, long long n, float* __restrict__ err, long long L, long long W, int nchunks,
               const double* __restrict__ state, PllParams P, PllChunk* __restrict__ chunks) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    const long long start = (long long)c * L, end = start + L < n ? start + L : n;
    double phi, freq;
    if (c == 0) {
        phi = state[0];
        freq = state[2];
    } else {
        const long long begin = start - W;                       // L >= W, so begin >= 0
        const float2 x0 = x[begin];
        phi = (double)atan2f(x0.y, x0.x);
        freq = 0.5 * (P.fmin + P.fmax);
        for (long long i = begin; i < start; ++i) {
            pll_step(x[i], phi, freq, P);
            pll_clamp(freq, P);
        }
    }
    chunks[c] = pll_chunk(x, err, start, end, phi, freq, P);
}

// Whether a chunk's speculated start (phi0, freq0) is within (dphi, dfreq) of the true state T; the phase difference
// modulo 2 pi (phi wraps at +-2 pi, and the lead-in's atan2f guess can land on the other branch).  NaN is a miss.
__device__ __forceinline__ bool pll_accept(double tphi, double tfreq, const PllChunk& k, double dphi, double dfreq) {
    double d = tphi - k.phi0;
    d = d - PLL_TWO_PI * rint(d / PLL_TWO_PI);
    return fabs(d) <= dphi && fabs(tfreq - k.freq0) <= dfreq;
}

// Stream order, one block.  The true state T is the carried (phi, freq) for chunk 0 and chunk c - 1's end state,
// after any re-run of it, for chunk c.  A chunk whose speculated start misses T is run again from T over its own
// samples, as pll_kernel runs them; then the bases are summed as before.  The block stages PV_BATCH chunks at a time in
// shared memory and tests each against its predecessor's speculated end in parallel, which is T unless the predecessor
// was run again; thread 0 then walks them in order, repeats the test after a re-run and runs the misses, and sums the
// bases in a second pass.  reruns[0] counts the chunks after the first that were run again.
constexpr int PV_BATCH = 256;
__global__ void __launch_bounds__(PV_BATCH)
pll_verify_kernel(const float2* __restrict__ x, long long n, float* __restrict__ err, long long L, PllChunk* chunks,
                  int nchunks, double* state, PllParams P, double dphi, double dfreq, unsigned long long* reruns) {
    __shared__ PllChunk sc[PV_BATCH];
    __shared__ bool sok[PV_BATCH];
    const int t = threadIdx.x;
    double lphi = state[0], lfreq = state[2], ph = state[1];          // thread 0: the end state before the batch
    bool prev_rerun = false;
    unsigned long long r = 0;
    for (int b0 = 0; b0 < nchunks; b0 += PV_BATCH) {
        const int c = b0 + t;
        if (c < nchunks) {
            const PllChunk k = chunks[c];
            sc[t] = k;
            sok[t] = c == 0 ? pll_accept(state[0], state[2], k, dphi, dfreq)
                            : pll_accept(chunks[c - 1].phi_end, chunks[c - 1].freq_end, k, dphi, dfreq);
        }
        __syncthreads();
        if (t == 0) {
            const int m = nchunks - b0 < PV_BATCH ? nchunks - b0 : PV_BATCH;
            for (int j = 0; j < m; ++j) {
                if (sok[j] && !prev_rerun) continue;                     // T is the predecessor's speculated end
                const double tphi = j > 0 ? sc[j - 1].phi_end : lphi, tfreq = j > 0 ? sc[j - 1].freq_end : lfreq;
                prev_rerun = !(prev_rerun && pll_accept(tphi, tfreq, sc[j], dphi, dfreq));
                if (!prev_rerun) continue;
                const long long start = (long long)(b0 + j) * L, end = start + L < n ? start + L : n;
                sc[j] = pll_chunk(x, err, start, end, tphi, tfreq, P);
                if (b0 + j > 0) ++r;
            }
            for (int j = 0; j < m; ++j) {
                sc[j].base = ph;
                ph = ph + sc[j].dP;                          // |ph| <= 4 pi: one wrap brings it back, exactly
                ph = ph > PLL_TWO_PI ? ph - PLL_TWO_PI : ph;
                ph = ph < -PLL_TWO_PI ? ph + PLL_TWO_PI : ph;
            }
            lphi = sc[m - 1].phi_end;
            lfreq = sc[m - 1].freq_end;
        }
        __syncthreads();
        if (c < nchunks) chunks[c] = sc[t];
        __syncthreads();                                     // the next batch reads chunk b0 + PV_BATCH - 1
    }
    if (t == 0) {
        state[0] = lphi;
        state[1] = ph;
        state[2] = lfreq;
        reruns[0] += r;
    }
}

__global__ void __launch_bounds__(128)
pll_out_kernel(const float* __restrict__ err, long long n, float2* __restrict__ out, long long L, int nchunks,
               PllParams P, const PllChunk* __restrict__ chunks) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    const long long start = (long long)c * L, end = start + L < n ? start + L : n;
    double phim = chunks[c].base, freq = chunks[c].freq0;
    for (long long i = start; i < end; ++i) {
        double s, cc;
        sincos(phim, &s, &cc);
        out[i] = make_float2((float)cc, (float)s);
        const double e = (double)err[i];
        freq = freq + P.beta * e;
        pll_advance(phim, freq, e, P);
        pll_clamp(freq, P);
    }
}

// The acceptance thresholds of pll_verify_kernel (derivation: tests/pll_ref.py).  A start-state offset (dphi, dfreq)
// moves the error by dphi_k and the multiplied phase by dphim_k of the linearised loop
//     dfreq' = dfreq - beta dphi,  dphi' = dphi + dfreq' - alpha dphi,  dphim' = dphim + m dfreq' - alpha dphi,
// whose largest |dphi_k| and |dphim_k| from a unit phase and a unit frequency offset are the gains g[0..3].  The box is
// (s alpha, s beta), the loop filter's step on one detector error s, with s as large as keeps a chunk that starts at its
// corner within PLL_ERR_BUDGET in error and PLL_OUT_BUDGET in output of the true trajectory.  Lead-ins on locked input
// land 4x (AM synchronous, noisy pilot) to 300x inside it; lead-ins through zeros miss it by orders of magnitude.
constexpr double PLL_ERR_BUDGET = 2.5e-7;
constexpr double PLL_OUT_BUDGET = 3.84e-7;
void pll_thresholds(double alpha, double beta, double mult, double* dphi, double* dfreq) {
    double g[4];
    for (int j = 0; j < 2; ++j) {
        double p = j == 0 ? 1.0 : 0.0, f = j == 0 ? 0.0 : 1.0, pm = 0.0, ge = std::fabs(p), go = 0.0;
        for (long long k = 1;; ++k) {
            f = f - beta * p;
            pm = pm + mult * f - alpha * p;
            p = p + f - alpha * p;
            ge = std::fmax(ge, std::fabs(p));
            go = std::fmax(go, std::fabs(pm));
            if (k > 64 && std::fabs(p) < 1e-12 * ge && std::fabs(f) < 1e-12 * beta * ge) break;
        }
        g[j] = ge;
        g[2 + j] = go;
    }
    const double se = PLL_ERR_BUDGET / (g[0] * alpha + g[1] * beta), so = PLL_OUT_BUDGET / (g[2] * alpha + g[3] * beta);
    const double sc = se < so ? se : so;
    *dphi = sc * alpha;
    *dfreq = sc * beta;
}

}  // namespace

struct PllBlock : Block {
    PllParams P;
    double init_freq;
    DeviceBuffer d_state;           // phi_locked, phi_multiplied, freq_locked
    int mode = 0;                   // 0 = exact sequential, 1 = chunk-parallel, verified against the carried state
    long long warm = 0;             // lead-in of the chunk-parallel form
    double dphi = 0.0, dfreq = 0.0; // acceptance thresholds of pll_verify_kernel
    DeviceBuffer d_chunks;
    DeviceBuffer d_reruns;          // chunks run again by pll_verify_kernel since create or reset
    unsigned long long chunks_run = 0;  // chunks after the first of every parallel call since create or reset
    PllBlock(double loop_bw_hz, double fmin_hz, double fmax_hz, double multiplier, double rate, bool dev) : Block("pll", 8, 8, dev) {
        num_outputs = 2;
        // pll.lua:113-131
        double bw = 2 * M_PI * (loop_bw_hz / rate);
        P.fmin = 2 * M_PI * (fmin_hz / rate);
        P.fmax = 2 * M_PI * (fmax_hz / rate);
        const double damping = std::sqrt(2.0) / 2;
        bw = bw / (damping + 1 / (4 * damping));
        const double denom = 1 + 2 * damping * bw + bw * bw;
        P.alpha = (4 * damping * bw) / denom;
        P.beta = (4 * bw * bw) / denom;
        P.mult = multiplier;
        init_freq = (P.fmin + P.fmax) / 2.0;
        warm = (long long)std::ceil(24.0 / (damping * bw));
        pll_thresholds(P.alpha, P.beta, P.mult, &dphi, &dfreq);
    }
    size_t out_size_of(int port) const override { return port == 0 ? 8 : 4; }
    long long memory_in() const override { return -1; }        // the multiplied phase integrates the whole past
    // the state after create and reset is not zero (freq_locked = init_freq): not carry()-declared
    int set_state() {
        const double h[3] = {0.0, 0.0, init_freq};
        LRB_CHECK(cudaMemcpyAsync(d_state.get(), h, sizeof(h), cudaMemcpyHostToDevice, ctx().stream));
        LRB_CHECK(cudaMemsetAsync(d_reruns.get(), 0, sizeof(unsigned long long), ctx().stream));
        LRB_CHECK(cudaStreamSynchronize(ctx().stream));
        chunks_run = 0;
        return 0;
    }
    int init() override {
        return d_state.reserve(3 * sizeof(double)) != 0 || d_reruns.reserve(sizeof(unsigned long long)) != 0 ? -1 : set_state();
    }
    int reset() override { consumed = 0; return set_state(); }
    int chunk_counts(uint64_t* chunks, uint64_t* reruns) {
        unsigned long long r = 0;
        LRB_CHECK(cudaMemcpyAsync(&r, d_reruns.get(), sizeof(r), cudaMemcpyDeviceToHost, ctx().stream));
        LRB_CHECK(cudaStreamSynchronize(ctx().stream));
        if (chunks) *chunks = chunks_run;
        if (reruns) *reruns = r;
        return 0;
    }
    int run(const void*, size_t, void*, size_t*, cudaStream_t) override {
        set_error("pll has two outputs (out, error): use lrb200_block_execute_multi");
        return -1;
    }
    int run_multi(const void* const* dx, int nin, size_t n, void* const* dy, int nout, size_t* n_out, cudaStream_t s) override {
        if (nin != 1 || nout != 2) { set_error("pll: expected 1 input and 2 outputs"); return -1; }
        *n_out = n;
        if (n == 0) return 0;
        const long long L = warm * 4 > 16384 ? warm * 4 : 16384;
        if (mode == 1 && (long long)n >= 2 * L) {
            const int nchunks = (int)(((long long)n + L - 1) / L);
            if (sizeof(PllChunk) * (size_t)nchunks > d_chunks.capacity()) {
                LRB_CHECK(cudaStreamSynchronize(s));
                if (d_chunks.reserve(sizeof(PllChunk) * (size_t)nchunks) != 0) return -1;
            }
            const int blocks = (nchunks + 127) / 128;
            PllChunk* chunks = d_chunks.as<PllChunk>();
            double* st = d_state.as<double>();
            pll_sim_kernel<<<blocks, 128, 0, s>>>((const float2*)dx[0], (long long)n, (float*)dy[1], L, warm, nchunks, st, P, chunks);
            pll_verify_kernel<<<1, PV_BATCH, 0, s>>>((const float2*)dx[0], (long long)n, (float*)dy[1], L, chunks, nchunks, st, P,
                                                     dphi, dfreq, d_reruns.as<unsigned long long>());
            pll_out_kernel<<<blocks, 128, 0, s>>>((const float*)dy[1], (long long)n, (float2*)dy[0], L, nchunks, P, chunks);
            count_launch(3);
            LRB_CHECK(cudaGetLastError());
            chunks_run += (unsigned long long)(nchunks - 1);
            consumed += n;
            return 0;
        }
        pll_kernel<<<1, 32, 0, s>>>((const float2*)dx[0], (long long)n, (float2*)dy[0], (float*)dy[1], d_state.as<double>(), P);
        count_launch();
        LRB_CHECK(cudaGetLastError());
        consumed += n;
        return 0;
    }
};

}  // namespace lrb

using namespace lrb;

extern "C" {

lrb200_block_t* lrb200_pll_create(double loop_bandwidth, double frequency_min, double frequency_max, double multiplier,
                                  double rate, unsigned flags) {
    if (ctx().device < 0 && lrb200_init(0) != 0) return nullptr;
    if (!(rate > 0.0) || !(loop_bandwidth > 0.0) || !std::isfinite(multiplier)) { set_error("pll: rate and loop bandwidth must be positive"); return nullptr; }
    if (!(frequency_min <= frequency_max)) { set_error("pll: frequency_min must not exceed frequency_max"); return nullptr; }
    return create_block<PllBlock>(flags, loop_bandwidth, frequency_min, frequency_max, multiplier, rate);
}

int lrb200_pll_set_mode(lrb200_block_t* q, int mode) {
    PllBlock* p = q && q->impl ? dynamic_cast<PllBlock*>(q->impl) : nullptr;
    if (!p) { set_error("not a PLL handle"); return -1; }
    if (mode != 0 && mode != 1) { set_error("pll: mode must be 0 (exact, sequential) or 1 (chunk-parallel, verified)"); return -1; }
    p->mode = mode;
    return 0;
}

int lrb200_pll_chunk_counts(lrb200_block_t* q, uint64_t* chunks, uint64_t* reruns) {
    PllBlock* p = q && q->impl ? dynamic_cast<PllBlock*>(q->impl) : nullptr;
    if (!p) { set_error("not a PLL handle"); return -1; }
    return p->chunk_counts(chunks, reruns);
}

}  // extern "C"
