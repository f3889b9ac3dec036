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
#include <cstddef>

namespace lrb {

namespace {

constexpr double PLL_TWO_PI = 6.283185307179586476925286766559;       // fl(2 pi): the wraps subtract it exactly

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


// ---- time-chunk sharding of a device DAG (graph.cu, Dag::shard_begin / shard_end).  A shard's PLL input holds, before
// the handoff point lh, a lead-in the left rank's samples fill; the loop is speculated from lh as pll_sim_kernel
// speculates a chunk, and its state at lh, at the next rank's handoff point and the wrapped sum of the multiplied
// phase's advances between them go to the shard's PllShardRecord.

// d_shard's (phi, sum of dP, freq) lands on a record's end state in one 24-byte copy
static_assert(offsetof(PllShardRecord, end_freq) - offsetof(PllShardRecord, end_phi) == 2 * sizeof(double), "end state");

// the lead-in of pll_sim_kernel over x[lh - W, lh): st = (phi, 0, freq) and the record's speculated start
__global__ void pll_lead_kernel(const float2* __restrict__ x, long long lh, long long W, PllParams P, double* st,
                                PllShardRecord* rec) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    const float2 x0 = x[lh - W];
    double phi = (double)atan2f(x0.y, x0.x), freq = 0.5 * (P.fmin + P.fmax);
    for (long long i = lh - W; i < lh; ++i) {
        pll_step(x[i], phi, freq, P);
        pll_clamp(freq, P);
    }
    st[0] = phi; st[1] = 0.0; st[2] = freq;
    rec->spec_phi = phi; rec->spec_freq = freq;
}

// one chunk of n samples in the sequential form from st, with its summary: what pll_verify_kernel makes of a re-run
// chunk (st's phim is the chunk's base and advances by its dP, wrapped once)
__global__ void pll_seq_kernel(const float2* __restrict__ x, long long n, float* __restrict__ err, double* st, PllParams P,
                               PllChunk* chunk) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    PllChunk k = pll_chunk(x, err, 0, n, st[0], st[2], P);
    k.base = st[1];
    double ph = st[1] + k.dP;
    ph = ph > PLL_TWO_PI ? ph - PLL_TWO_PI : ph;
    ph = ph < -PLL_TWO_PI ? ph + PLL_TWO_PI : ph;
    st[0] = k.phi_end; st[1] = ph; st[2] = k.freq_end;
    *chunk = k;
}

// the bases of nchunks consecutive chunks from base0, summed as pll_verify_kernel sums them
__global__ void pll_rebase_kernel(PllChunk* chunks, int nchunks, double base0) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    double ph = base0;
    for (int c = 0; c < nchunks; ++c) {
        chunks[c].base = ph;
        ph = ph + chunks[c].dP;
        ph = ph > PLL_TWO_PI ? ph - PLL_TWO_PI : ph;
        ph = ph < -PLL_TWO_PI ? ph + PLL_TWO_PI : ph;
    }
}

// after a chunk-parallel call: the loop state (phi, phim, freq) at sample `split` <= n, replayed from the start state of
// the chunk that holds it -- the state its errors were computed from -- and its base
__global__ void pll_probe_kernel(const float2* __restrict__ x, long long L, const PllChunk* __restrict__ chunks, int nchunks,
                                 long long split, PllParams P, double* out) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    int c = (int)(split / L);
    c = c < nchunks - 1 ? c : nchunks - 1;
    double phi = chunks[c].phi0, freq = chunks[c].freq0, phim = chunks[c].base;
    for (long long i = (long long)c * L; i < split; ++i) {
        const float e = pll_step(x[i], phi, freq, P);
        pll_advance(phim, freq, (double)e, P);
        pll_clamp(freq, P);
    }
    out[0] = phi; out[1] = phim; out[2] = freq;
}

}  // namespace

PllBlock::PllBlock(double loop_bw_hz, double fmin_hz, double fmax_hz, double multiplier, double rate, bool dev) : Block("pll", 8, 8, dev) {
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

int PllBlock::set_state() {
    const double h[3] = {0.0, 0.0, init_freq};
    LRB_CHECK(cudaMemcpyAsync(d_state.get(), h, sizeof(h), cudaMemcpyHostToDevice, ctx().stream));
    LRB_CHECK(cudaMemsetAsync(d_reruns.get(), 0, sizeof(unsigned long long), ctx().stream));
    LRB_CHECK(cudaStreamSynchronize(ctx().stream));
    chunks_run = 0;
    return 0;
}

int PllBlock::init() {
    return d_state.reserve(3 * sizeof(double)) != 0 || d_reruns.reserve(sizeof(unsigned long long)) != 0 ||
                   d_shard.reserve(3 * sizeof(double)) != 0
               ? -1
               : set_state();
}

int PllBlock::chunk_counts(uint64_t* chunks, uint64_t* reruns) {
    unsigned long long r = 0;
    LRB_CHECK(cudaMemcpyAsync(&r, d_reruns.get(), sizeof(r), cudaMemcpyDeviceToHost, ctx().stream));
    LRB_CHECK(cudaStreamSynchronize(ctx().stream));
    if (chunks) *chunks = chunks_run;
    if (reruns) *reruns = r;
    return 0;
}

int PllBlock::run(const void*, size_t, void*, size_t*, cudaStream_t) {
    set_error("pll has two outputs (out, error): use lrb200_block_execute_multi");
    return -1;
}

int PllBlock::reserve_chunks(int nchunks, cudaStream_t s) {
    if (sizeof(PllChunk) * (size_t)nchunks > d_chunks.capacity()) {
        LRB_CHECK(cudaStreamSynchronize(s));
        if (d_chunks.reserve(sizeof(PllChunk) * (size_t)nchunks) != 0) return -1;
    }
    return 0;
}

int PllBlock::run_multi(const void* const* dx, int nin, size_t n, void* const* dy, int nout, size_t* n_out, cudaStream_t s) {
    if (nin != 1 || nout != 2) { set_error("pll: expected 1 input and 2 outputs"); return -1; }
    *n_out = n;
    if (n == 0) return 0;
    const long long L = chunk_len();
    if (parallel(n)) {
        const int nchunks = (int)(((long long)n + L - 1) / L);
        if (reserve_chunks(nchunks, s) != 0) return -1;
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

// ---- time-chunk sharding of a device DAG --------------------------------------------------------------------------------
bool PllBlock::accepts(double tphi, double tfreq, double phi0, double freq0) const {
    double d = tphi - phi0;                            // pll_accept, on the host
    d = d - PLL_TWO_PI * std::rint(d / PLL_TWO_PI);
    return std::fabs(d) <= dphi && std::fabs(tfreq - freq0) <= dfreq;
}

double PllBlock::fold_advances(const PllShardRecord* lefts, unsigned num_left, size_t stride, size_t j) {
    double base = 0.0;
    for (unsigned r = 0; r < num_left; ++r) {
        base = base + lefts[stride * r + j].end_dP;
        base = base > PLL_TWO_PI ? base - PLL_TWO_PI : base;
        base = base < -PLL_TWO_PI ? base + PLL_TWO_PI : base;
    }
    return base;
}

int PllBlock::run_probe(const void* x, size_t n, void* const* dy, long long split, PllShardRecord* rec, cudaStream_t s) {
    if (split < 0 || split > (long long)n) { set_error("pll: probe at %lld outside a call of %zu samples", split, n); return -1; }
    size_t no = 0;
    if (parallel(n)) {
        if (run_multi(&x, 1, n, dy, 2, &no, s) != 0) return -1;
        const long long L = chunk_len();
        pll_probe_kernel<<<1, 32, 0, s>>>((const float2*)x, L, d_chunks.as<PllChunk>(), (int)(((long long)n + L - 1) / L), split, P,
                                          &rec->end_phi);
        count_launch();
        LRB_CHECK(cudaGetLastError());
        return 0;
    }
    // the sequential form carries its whole state from call to call: two calls split at `split` are the one call bit for bit
    double* st = d_state.as<double>();
    if (split > 0) {
        pll_kernel<<<1, 32, 0, s>>>((const float2*)x, split, (float2*)dy[0], (float*)dy[1], st, P);
        count_launch();
    }
    LRB_CHECK(cudaMemcpyAsync(&rec->end_phi, st, 3 * sizeof(double), cudaMemcpyDeviceToDevice, s));
    if ((long long)n > split) {
        pll_kernel<<<1, 32, 0, s>>>((const float2*)x + split, (long long)n - split, (float2*)dy[0] + split, (float*)dy[1] + split, st, P);
        count_launch();
    }
    LRB_CHECK(cudaGetLastError());
    consumed += n;
    return 0;
}

// the loop over x[off, off + len) from d_shard in the form a call of len samples runs (rerun: the chunks were simulated
// before, and are verified again against a new d_shard)
int PllBlock::shard_range(const ShardRange& r, const void* x, float* err, bool rerun, cudaStream_t s) {
    if (r.len == 0) return 0;
    const float2* xr = (const float2*)x + r.off;
    PllChunk* chunks = d_chunks.as<PllChunk>() + r.cb;
    double* st = d_shard.as<double>();
    if (r.nch == 1) {
        pll_seq_kernel<<<1, 32, 0, s>>>(xr, r.len, err + r.off, st, P, chunks);
        count_launch();
    } else {
        if (!rerun) {
            pll_sim_kernel<<<(r.nch + 127) / 128, 128, 0, s>>>(xr, r.len, err + r.off, r.L, warm, r.nch, st, P, chunks);
            chunks_run += (unsigned long long)(r.nch - 1);
            count_launch();
        }
        pll_verify_kernel<<<1, PV_BATCH, 0, s>>>(xr, r.len, err + r.off, r.L, chunks, r.nch, st, P, dphi, dfreq,
                                                 d_reruns.as<unsigned long long>());
        count_launch();
    }
    LRB_CHECK(cudaGetLastError());
    return 0;
}

int PllBlock::shard_loop(const void* x, size_t n, float* err, long long lh, long long le, PllShardRecord* rec, cudaStream_t s) {
    if (lh < warm || le < lh || le > (long long)n) {
        set_error("pll: handoff points %lld, %lld of a %zu-sample shard leave no %lld-sample lead-in", lh, le, n, warm);
        return -1;
    }
    const long long L = chunk_len();
    const long long off[3] = {lh, le, (long long)n};
    int cb = 0;
    for (int k = 0; k < 2; ++k) {
        ShardRange& r = rng[k];
        r.off = off[k];
        r.len = off[k + 1] - off[k];
        r.L = parallel((size_t)r.len) ? L : (r.len > 0 ? r.len : 1);
        r.nch = r.len == 0 ? 0 : (int)((r.len + r.L - 1) / r.L);
        r.cb = cb;
        cb += r.nch;
    }
    if (reserve_chunks(cb > 0 ? cb : 1, s) != 0) return -1;
    if (lh > 0) LRB_CHECK(cudaMemsetAsync(err, 0, (size_t)lh * sizeof(float), s));
    pll_lead_kernel<<<1, 32, 0, s>>>((const float2*)x, lh, warm, P, d_shard.as<double>(), rec);
    count_launch();
    if (shard_range(rng[0], x, err, false, s) != 0) return -1;
    LRB_CHECK(cudaMemcpyAsync(&rec->end_phi, d_shard.get(), 3 * sizeof(double), cudaMemcpyDeviceToDevice, s));
    if (shard_range(rng[1], x, err, false, s) != 0) return -1;
    consumed += n;
    return 0;
}

int PllBlock::shard_rerun(const void* x, float* err, double tphi, double tfreq, PllShardRecord* rec, cudaStream_t s) {
    const double h[3] = {tphi, 0.0, tfreq};
    LRB_CHECK(cudaMemcpyAsync(d_shard.get(), h, sizeof(h), cudaMemcpyHostToDevice, s));
    if (shard_range(rng[0], x, err, true, s) != 0) return -1;
    LRB_CHECK(cudaMemcpyAsync(&rec->end_phi, d_shard.get(), 3 * sizeof(double), cudaMemcpyDeviceToDevice, s));
    return shard_range(rng[1], x, err, true, s);
}

int PllBlock::shard_out(const float* err, float2* out, double base, cudaStream_t s) {
    const int nch = rng[0].nch + rng[1].nch;
    if (rng[0].off > 0) LRB_CHECK(cudaMemsetAsync(out, 0, (size_t)rng[0].off * sizeof(float2), s));
    if (nch == 0) return 0;
    PllChunk* chunks = d_chunks.as<PllChunk>();
    pll_rebase_kernel<<<1, 32, 0, s>>>(chunks, nch, base);
    count_launch();
    for (const ShardRange& r : rng) {
        if (r.nch == 0) continue;
        pll_out_kernel<<<(r.nch + 127) / 128, 128, 0, s>>>(err + r.off, r.len, out + r.off, r.L, r.nch, P, chunks + r.cb);
        count_launch();
    }
    LRB_CHECK(cudaGetLastError());
    return 0;
}

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
