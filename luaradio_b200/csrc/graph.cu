// Single-stream GPU flow graph: a connected chain of GPU blocks sharing device-resident buffers.
//
// Replaces, for a run of connected GPU blocks, the reference's fork-per-block scheduler and socketpair
// pipes (radio/core/composite.lua:568-636, radio/core/pipe.lua:53-88): intermediate sample vectors stay
// in a two-slot device ring; host<->device traffic exists only at the two ends, double-buffered on
// separate copy streams so chunk i+1 uploads while chunk i computes and chunk i-1 downloads.
// commit(fuse=1) rewrites runs of adjacent blocks into fused kernels, one rule function per rewrite (below).
#include "../../include/lrb200.h"
#include "common.cuh"
#include "blocks.h"

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <new>
#include <string>
#include <vector>

namespace lrb {

using Blocks = std::vector<std::unique_ptr<Block>>;

// What a rule made of the run starting at blocks[i]: one stage, or two, standing for the first `used` blocks.
struct Rewrite {
    std::unique_ptr<Block> stage, stage2;
    size_t used = 0;                 // 0: no match
};
// 0 (a match or none, see out->used), or -1 with the error set
using Rule = int (*)(const Blocks& blocks, size_t i, Rewrite* out);

// blocks[j] as a T, or nullptr (another type, or past the end)
template <class T> T* block_at(const Blocks& blocks, size_t j) {
    return j < blocks.size() ? dynamic_cast<T*>(blocks[j].get()) : nullptr;
}

// Rotator -> FIR(crcf, D = 1) -> Downsampler(8 B) [-> Discriminator]  =>  tuner kernel (composites/tuner.lua:40-47).
// No match when the tuner kernel has no instantiation for the (taps, decimation) shape.
static int fuse_tuner(const Blocks& blocks, size_t i, Rewrite* out) {
    RotatorBlock* rot = block_at<RotatorBlock>(blocks, i);
    FirBlock* fir = block_at<FirBlock>(blocks, i + 1);
    DownsampleBlock* down = block_at<DownsampleBlock>(blocks, i + 2);
    if (!rot || !fir || fir->kind != FIR_CRCF || fir->D != 1 || !down || down->in_size != 8) return 0;
    DiscrimBlock* disc = block_at<DiscrimBlock>(blocks, i + 3);
    out->stage = make_tuner(rot->turns, (const float*)fir->h_taps.data(), fir->M, down->D, disc ? disc->gain : 0.0f);
    if (out->stage) out->used = disc ? 4 : 3;
    return 0;
}

// Rotator -> FIR(crcf or cccf, D = 1, M <= 513) [-> Downsampler(8 B)]  =>  overlap-save FIR with the translator folded in
// (any taps, complex taps included)
static int fuse_rotator_overlap_save(const Blocks& blocks, size_t i, Rewrite* out) {
    RotatorBlock* rot = block_at<RotatorBlock>(blocks, i);
    FirBlock* fir = block_at<FirBlock>(blocks, i + 1);
    if (!rot || !fir || (fir->kind != FIR_CRCF && fir->kind != FIR_CCCF) || fir->D != 1 || fir->M > 513) return 0;
    DownsampleBlock* down = block_at<DownsampleBlock>(blocks, i + 2);
    if (down && down->in_size != 8) down = nullptr;
    out->stage = make_block<FirBlock>(fir->kind, fir->h_taps.data(), (unsigned)fir->M, (unsigned)(down ? down->D : 1), true, true,
                                      rot->turns);
    if (!out->stage) return -1;
    out->used = down ? 3 : 2;
    return 0;
}

// [MultiplyConstant(real c) ->] Upsampler(L) -> FIR(crcf or rrrf, D = 1) [-> Downsampler(D)]  =>  polyphase interpolating
// FIR (composites/interpolator.lua:31-41, composites/rationalresampler.lua:33-46).  A complex constant is not absorbed.
static int fuse_interpolator(const Blocks& blocks, size_t i, Rewrite* out) {
    ScaleBlock* sc = block_at<ScaleBlock>(blocks, i);
    if (sc && sc->complex_const) sc = nullptr;
    const size_t j = sc ? i + 1 : i;
    UpsampleBlock* up = block_at<UpsampleBlock>(blocks, j);
    FirBlock* fir = block_at<FirBlock>(blocks, j + 1);
    if (!up || !fir || fir->D != 1 || (fir->kind != FIR_CRCF && fir->kind != FIR_RRRF) || fir->in_size != up->out_size) return 0;
    DownsampleBlock* down = block_at<DownsampleBlock>(blocks, j + 2);
    if (down && down->in_size != fir->out_size) down = nullptr;
    out->stage = make_block<InterpFirBlock>(fir->kind == FIR_CRCF, (const float*)fir->h_taps.data(), fir->M, up->L,
                                            down ? down->D : 1, sc != nullptr, sc ? sc->cre : 1.0f, true);
    if (!out->stage) return -1;
    out->used = (j - i) + 2 + (down ? 1 : 0);
    return 0;
}

// FIR(h, rrrf, D = 1) -> single-pole IIR(b, c, real) -> Downsampler(D > 1): the chain's audio tail
// (examples/rtlsdr_wbfm_mono.lua:15-18; iirfilter.lua:147-179; downsampler.lua:45-53).
// y[n] = c y[n-1] + v[n], v = b * u, u = h * x.  Unrolling the recurrence D times:
//     y[n] = c^D y[n-D] + sum_{i<D} c^i v[n-i]
// so the kept samples z[m] = y[mD] obey  z[m] = c^D z[m-1] + w[mD]  with  w = (h * b * [1, c, .., c^(D-1)]) * x:
// ONE decimating FIR with M + nb + D - 2 taps (only kept outputs computed) and a pole c^D at the
// output rate, instead of a full-rate FIR and a full-rate recurrence that both compute D times more
// samples than the Downsampler keeps.  Zero initial state on both sides, so the streams are equal
// from the first sample; the taps are designed in float64 from the float32 coefficients.
// One stage with the pole fused in when its memory fits the polyphase kernel's warm-up, else two stages
// `fir*iir1_rrrf(..) | pole_rrrf`; no match when the polyphase kernel has no shape for the composed taps.
static int fuse_noble_identity(const Blocks& blocks, size_t i, Rewrite* out) {
    FirBlock* fir = block_at<FirBlock>(blocks, i);
    IirBlock* iir = block_at<IirBlock>(blocks, i + 1);
    DownsampleBlock* down = block_at<DownsampleBlock>(blocks, i + 2);
    if (!fir || fir->D != 1 || fir->kind != FIR_RRRF || !iir || iir->complex_data || iir->D != 1 || !down || down->in_size != 4 ||
        down->D <= 1)
        return 0;
    const int Dd = down->D, nbb = iir->nb;
    std::vector<double> g((size_t)(nbb + Dd - 1), 0.0);
    double cp = 1.0;
    for (int k = 0; k < Dd; ++k) {
        for (int j = 0; j < nbb; ++j) g[(size_t)(k + j)] += cp * (double)iir->b[j];
        cp *= (double)iir->c;
    }
    const float* h = (const float*)fir->h_taps.data();
    const int Mc = fir->M + (int)g.size() - 1;
    std::vector<float> hc((size_t)Mc);
    for (int t = 0; t < Mc; ++t) {
        double acc = 0.0;
        for (int k = 0; k < (int)g.size(); ++k)
            if (t - k >= 0 && t - k < fir->M) acc += g[(size_t)k] * (double)h[t - k];
        hc[(size_t)t] = (float)acc;
    }
    auto nf = make_block<FirBlock>(FIR_RRRF, hc.data(), (unsigned)Mc, (unsigned)Dd, true);
    if (!nf) return -1;
    // only worth it when the polyphase kernel has this shape (at AUTO, the block runs it whenever it has it)
    if (!nf->always_polyphase()) return 0;
    nf->set_algorithm(fir->algo);
    nf->name = "fir*iir1_rrrf(" + std::to_string(Mc) + ",/" + std::to_string(Dd) + ")";
    if (nf->always_polyphase() && polyphase_pole_ok((float)cp)) {
        // the pole's memory (|c^D|^64 <= 1e-8) fits the kernel's own warm-up: ONE stage
        if (nf->set_pole((float)cp) != 0) return -1;
        nf->name += "+pole";
    } else {
        const float one = 1.0f, a2[2] = {1.0f, (float)(-cp)};     // cp == c^D
        out->stage2 = make_block<IirBlock>(false, &one, 1u, a2, 2u, true);
        if (!out->stage2) return -1;
        out->stage2->name = "pole_rrrf";
    }
    out->stage = std::move(nf);
    out->used = 3;
    return 0;
}

// ComplexMagnitude -> FIR(rrrf, D = 1) -> Downsampler(4 B, D > 1), or ComplexMagnitude -> FIR(rrrf, D > 1)  =>  overlap-save
// FIR that takes |x| at its load (the ERT receiver's front end, composites/ertreceiver.lua:38-43).  The magnitude stream
// never goes through HBM: 8 B read per input sample instead of 8 + 4 + 4.  No match for an undecimated FIR, or where the
// decimating FIR fuse_fir_decimator would make does not run the overlap-save kernel on long calls (a polyphase shape, a
// forced direct form, taps the single-block plan does not cover): those keep their own kernel choice.
static int fuse_magnitude_fir(const Blocks& blocks, size_t i, Rewrite* out) {
    C2fBlock* mag = block_at<C2fBlock>(blocks, i);
    FirBlock* fir = block_at<FirBlock>(blocks, i + 1);
    if (!mag || mag->op != 0 || !fir || fir->kind != FIR_RRRF || fir->rotate || fir->magnitude || fir->has_pole) return 0;
    DownsampleBlock* down = fir->D == 1 ? block_at<DownsampleBlock>(blocks, i + 2) : nullptr;
    if (down && down->in_size != 4) down = nullptr;
    const int D = fir->D * (down ? down->D : 1);
    if (D <= 1) return 0;
    auto plain = make_block<FirBlock>(FIR_RRRF, fir->h_taps.data(), (unsigned)fir->M, (unsigned)D, true);
    if (!plain) return -1;
    if (plain->set_algorithm(fir->algo) != 0) return -1;
    if (plain->effective_algorithm() != LRB200_FIR_FFT) return 0;
    out->stage = make_block<FirBlock>(FIR_RRRF, fir->h_taps.data(), (unsigned)fir->M, (unsigned)D, true, false, 0.0, true);
    if (!out->stage) return -1;
    out->used = down ? 3 : 2;
    return 0;
}

// FIR(D = 1, not Hilbert) -> Downsampler(D)  =>  decimating FIR (composites/decimator.lua:34-41)
static int fuse_fir_decimator(const Blocks& blocks, size_t i, Rewrite* out) {
    FirBlock* fir = block_at<FirBlock>(blocks, i);
    DownsampleBlock* down = block_at<DownsampleBlock>(blocks, i + 1);
    if (!fir || fir->D != 1 || fir->kind == FIR_HILBERT || !down || down->in_size != fir->out_size) return 0;
    auto nf = make_block<FirBlock>(fir->kind, fir->h_taps.data(), (unsigned)fir->M, (unsigned)down->D, true);
    if (!nf) return -1;
    nf->set_algorithm(fir->algo);    // FIRFilterBlock(taps, use_fft) survives the fusion
    out->stage = std::move(nf);
    out->used = 2;
    return 0;
}

// single-pole IIR(D = 1) -> Downsampler(D)  =>  scan with strided store
static int fuse_iir_decimator(const Blocks& blocks, size_t i, Rewrite* out) {
    IirBlock* iir = block_at<IirBlock>(blocks, i);
    DownsampleBlock* down = block_at<DownsampleBlock>(blocks, i + 1);
    if (!iir || iir->D != 1 || !down || down->in_size != iir->out_size) return 0;
    const float a[2] = {1.0f, -iir->c};
    auto ni = make_block<IirBlock>(iir->complex_data, iir->b, (unsigned)iir->nb, a, 2u, true);
    if (!ni) return -1;
    ni->D = down->D;
    out->stage = std::move(ni);
    out->used = 2;
    return 0;
}

// in priority order: the first rule that matches at a block wins
static const Rule FUSION_RULES[] = {fuse_tuner, fuse_rotator_overlap_save, fuse_interpolator, fuse_noble_identity,
                                   fuse_magnitude_fir, fuse_fir_decimator, fuse_iir_decimator};

// The host <-> device boundary of a device run: a linear graph, a device DAG, or a block created without LRB200_DEVICE.
// The owner gives its run, a bound on a run's outputs per port, its ports' element sizes and its chunk length.  A host
// call of at most one chunk is one upload per input, the run, one download per output and one synchronize, all on the
// library stream (every call of the reference's per-vector regime, pipe.lua:73: nothing to overlap); a longer call is
// cut into chunks pipelined over two slots on three streams, so that chunk i + 1 uploads while chunk i runs and chunk
// i - 1 downloads.  Where a stream is cut changes output bits (PllBlock::parallel and FirBlock::path choose by call
// length, the IIR scan places its warm-up restarts from a call's start), so each owner keeps its own chunk length.
// Super-chunk mode (SURVEY.md 8e "streaming mode"), for an owner with one input: small host vectors are packed into
// pinned slots of `samples` input samples; a full slot is processed asynchronously while the next one fills, and its
// outputs (one stream per output port) are handed back when that next slot is submitted (or at flush) -- the per-vector
// cost is one host memcpy instead of copies + launches + a sync.  Every port's outputs come from the same slots.  While
// the mode is on, the stream runs through the slots only: a direct device or shard run is refused, and a reset waits for
// and drops the slots in flight and the partial slot.
struct HostBoundary {
    // device ins / outs of one run of n samples, asynchronous on s: dy[k] receives n_out[k] samples of port k
    using Run = std::function<int(const void* const* dx, size_t n, void* const* dy, size_t* n_out, cudaStream_t s)>;
    struct HostFree { void operator()(char* p) const { cudaFreeHost(p); } };
    using PinnedSlot = std::unique_ptr<char, HostFree>;
    Run run;
    std::function<size_t(size_t)> max_out;        // samples any output port may receive from a run of n inputs
    std::vector<size_t> in_size, out_size;        // bytes per sample of each input and output port
    size_t chunk;                                 // input samples per chunk of a host call
    std::vector<DeviceBuffer> din[2], dout[2];    // per slot: the device staging of each port
    std::vector<const void*> pin[2];
    std::vector<void*> pout[2];
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;   // the copy streams of calls longer than one chunk
    cudaEvent_t ev_h2d[2] = {nullptr, nullptr}, ev_comp[2] = {nullptr, nullptr}, ev_d2h[2] = {nullptr, nullptr};
    // super-chunk mode
    size_t samples = 0;                           // input samples per slot; 0 = off
    size_t outcap = 0;                            // samples a slot can produce in any port
    PinnedSlot hin[2];
    std::vector<PinnedSlot> hout[2];
    cudaEvent_t done[2] = {nullptr, nullptr};
    bool pending[2] = {false, false};
    std::vector<size_t> nout[2];
    size_t fill = 0;
    int cur = 0;
    bool fed = false;                             // an execute since the mode was set, or since the last flush / reset

    HostBoundary(Run r, std::function<size_t(size_t)> mo, size_t chunk_) : run(std::move(r)), max_out(std::move(mo)), chunk(chunk_) {}
    ~HostBoundary() {
        release();
        for (int i = 0; i < 2; ++i)
            for (cudaEvent_t e : {ev_h2d[i], ev_comp[i], ev_d2h[i]})
                if (e) cudaEventDestroy(e);
        if (s_h2d) cudaStreamDestroy(s_h2d);
        if (s_d2h) cudaStreamDestroy(s_d2h);
    }

    // launches in flight may still read a staging buffer that grows: the device drains first
    static int grow(DeviceBuffer& b, size_t bytes) {
        if (bytes <= b.capacity()) return 0;
        LRB_CHECK(cudaDeviceSynchronize());
        return b.reserve(bytes);
    }
    // the slot's device staging for a run of n inputs
    int reserve(int slot, size_t n) {
        const size_t mo = max_out(n);
        din[slot].resize(in_size.size());
        dout[slot].resize(out_size.size());
        pin[slot].resize(in_size.size());
        pout[slot].resize(out_size.size());
        for (size_t i = 0; i < in_size.size(); ++i) {
            if (grow(din[slot][i], (n ? n : 1) * in_size[i]) != 0) return -1;
            pin[slot][i] = din[slot][i].get();
        }
        for (size_t k = 0; k < out_size.size(); ++k) {
            if (grow(dout[slot][k], (mo ? mo : 1) * out_size[k]) != 0) return -1;
            pout[slot][k] = dout[slot][k].get();
        }
        return 0;
    }
    // one run through the slot on s: the host ins x[i] up, the run, the outs down to y[k] (no synchronize)
    int stage(int slot, const void* const* x, size_t n, void* const* y, size_t* n_out, cudaStream_t s) {
        for (size_t i = 0; i < in_size.size(); ++i)
            if (n) LRB_CHECK(cudaMemcpyAsync(din[slot][i].get(), x[i], n * in_size[i], cudaMemcpyHostToDevice, s));
        if (run(pin[slot].data(), n, pout[slot].data(), n_out, s) != 0) return -1;
        for (size_t k = 0; k < out_size.size(); ++k)
            if (n_out[k]) LRB_CHECK(cudaMemcpyAsync(y[k], pout[slot][k], n_out[k] * out_size[k], cudaMemcpyDeviceToHost, s));
        return 0;
    }

    int ensure_pipeline() {
        if (s_h2d) return 0;
        LRB_CHECK(cudaStreamCreateWithFlags(&s_h2d, cudaStreamNonBlocking));
        LRB_CHECK(cudaStreamCreateWithFlags(&s_d2h, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
            LRB_CHECK(cudaEventCreateWithFlags(&ev_h2d[i], cudaEventDisableTiming));
            LRB_CHECK(cudaEventCreateWithFlags(&ev_comp[i], cudaEventDisableTiming));
            LRB_CHECK(cudaEventCreateWithFlags(&ev_d2h[i], cudaEventDisableTiming));
        }
        return 0;
    }

    // host ins x[i] of n samples, host outs y[k] receiving n_out[k] samples -- or, in super-chunk mode, the vector appended
    // to the current slot (y[k] then receives the outputs of the slots completed meanwhile)
    int execute(const void* const* x, size_t n, void* const* y, size_t* n_out) {
        if (samples) {
            fed = true;
            return accumulate((const char*)x[0], n, (char* const*)y, n_out);
        }
        cudaStream_t s = ctx().stream;
        if (n <= chunk) {
            if (reserve(0, n) != 0 || stage(0, x, n, y, n_out, s) != 0) return -1;
            LRB_CHECK(cudaStreamSynchronize(s));
            return 0;
        }
        if (ensure_pipeline() != 0) return -1;
        std::vector<size_t> no(out_size.size());
        for (size_t k = 0; k < out_size.size(); ++k) n_out[k] = 0;
        for (size_t done_in = 0, it = 0; done_in < n; ++it) {
            const int slot = (int)(it & 1);
            const size_t nc = n - done_in < chunk ? n - done_in : chunk;
            if (reserve(slot, nc) != 0) return -1;
            if (it >= 2) LRB_CHECK(cudaStreamWaitEvent(s_h2d, ev_comp[slot], 0));     // the slot's inputs free again
            for (size_t i = 0; i < in_size.size(); ++i)
                LRB_CHECK(cudaMemcpyAsync(din[slot][i].get(), (const char*)x[i] + done_in * in_size[i], nc * in_size[i],
                                          cudaMemcpyHostToDevice, s_h2d));
            LRB_CHECK(cudaEventRecord(ev_h2d[slot], s_h2d));
            LRB_CHECK(cudaStreamWaitEvent(s, ev_h2d[slot], 0));
            if (it >= 2) LRB_CHECK(cudaStreamWaitEvent(s, ev_d2h[slot], 0));          // the slot's outputs drained
            if (run(pin[slot].data(), nc, pout[slot].data(), no.data(), s) != 0) return -1;
            LRB_CHECK(cudaEventRecord(ev_comp[slot], s));
            LRB_CHECK(cudaStreamWaitEvent(s_d2h, ev_comp[slot], 0));
            for (size_t k = 0; k < out_size.size(); ++k) {
                if (no[k]) LRB_CHECK(cudaMemcpyAsync((char*)y[k] + n_out[k] * out_size[k], pout[slot][k], no[k] * out_size[k],
                                                     cudaMemcpyDeviceToHost, s_d2h));
                n_out[k] += no[k];
            }
            LRB_CHECK(cudaEventRecord(ev_d2h[slot], s_d2h));
            done_in += nc;
        }
        // the last download is behind every upload and every run (event chain), so one synchronize drains all three
        LRB_CHECK(cudaStreamSynchronize(s_d2h));
        LRB_CHECK(cudaStreamSynchronize(s));     // (returns at once; keeps the compute stream's error state observable)
        return 0;
    }

    // ---- super-chunk mode -----------------------------------------------------------------------------------------------
    void release() {
        for (int i = 0; i < 2; ++i) {
            hin[i].reset(); hout[i].clear();
            if (done[i]) cudaEventDestroy(done[i]);
            done[i] = nullptr;
            pending[i] = false; nout[i].clear();
        }
        samples = 0; fill = 0; cur = 0;
    }
    // slots of n input samples (0: off), only while none is pending or partly filled
    int set_superchunk(size_t n, const char* who) {
        if (pending[0] || pending[1] || fill) { set_error("%s: flush before changing the super-chunk size", who); return -1; }
        release();
        fed = false;
        if (n == 0) return 0;
        outcap = max_out(n) + 1;
        for (int i = 0; i < 2; ++i) {
            if (reserve(i, n) != 0) return -1;
            char* p = nullptr;
            LRB_CHECK(cudaHostAlloc((void**)&p, n * in_size[0], cudaHostAllocDefault));
            hin[i].reset(p);
            hout[i].resize(out_size.size());
            nout[i].assign(out_size.size(), 0);
            for (size_t k = 0; k < out_size.size(); ++k) {
                LRB_CHECK(cudaHostAlloc((void**)&p, outcap * out_size[k], cudaHostAllocDefault));
                hout[i][k].reset(p);
            }
            LRB_CHECK(cudaEventCreateWithFlags(&done[i], cudaEventDisableTiming));
        }
        samples = n;
        return 0;
    }
    // reset: wait for the slots in flight and forget them and the partial slot (the super-chunk size stays)
    int drop() {
        for (int i = 0; i < 2; ++i) {
            if (pending[i] && !cuda_ok(cudaEventSynchronize(done[i]), "cudaEventSynchronize")) return -1;
            pending[i] = false;
        }
        fill = 0; cur = 0; fed = false;
        return 0;
    }
    // append a finished slot's outputs to y[k] + produced[k]
    int collect(int slot, char* const* y, size_t* produced) {
        if (!pending[slot]) return 0;
        if (!cuda_ok(cudaEventSynchronize(done[slot]), "cudaEventSynchronize")) return -1;
        for (size_t k = 0; k < out_size.size(); ++k) {
            if (nout[slot][k]) memcpy(y[k] + produced[k] * out_size[k], hout[slot][k].get(), nout[slot][k] * out_size[k]);
            produced[k] += nout[slot][k];
        }
        pending[slot] = false;
        return 0;
    }
    int submit(int slot, size_t count) {
        cudaStream_t s = ctx().stream;
        const void* hx = hin[slot].get();
        std::vector<void*> hy(out_size.size());
        for (size_t k = 0; k < out_size.size(); ++k) hy[k] = hout[slot][k].get();
        if (stage(slot, &hx, count, hy.data(), nout[slot].data(), s) != 0) return -1;
        LRB_CHECK(cudaEventRecord(done[slot], s));
        pending[slot] = true;
        return 0;
    }
    int accumulate(const char* x, size_t n, char* const* y, size_t* n_out) {
        for (size_t k = 0; k < out_size.size(); ++k) n_out[k] = 0;
        while (n > 0) {
            const size_t take = n < samples - fill ? n : samples - fill;
            memcpy(hin[cur].get() + fill * in_size[0], x, take * in_size[0]);
            fill += take; x += take * in_size[0]; n -= take;
            if (fill == samples) {
                // the other slot was submitted one super-chunk ago: its results are (long) ready
                if (collect(cur ^ 1, y, n_out) != 0) return -1;
                if (submit(cur, samples) != 0) return -1;
                cur ^= 1;
                fill = 0;
            }
        }
        return 0;
    }
    // the pending slot's outputs and the partial slot's; 0 samples when the mode is off
    int flush(void* const* yv, size_t* n_out) {
        char* const* y = (char* const*)yv;
        for (size_t k = 0; k < out_size.size(); ++k) n_out[k] = 0;
        fed = false;
        if (!samples) return 0;
        if (collect(cur ^ 1, y, n_out) != 0) return -1;
        if (fill) {
            if (submit(cur, fill) != 0) return -1;
            if (collect(cur, y, n_out) != 0) return -1;
            fill = 0;
        }
        return 0;
    }
    // a run past the boundary (device pointers, a shard) would overtake the samples waiting in the slots
    int refuse_direct(const char* who, const char* what) const {
        if (!samples) return 0;
        set_error("%s: %s runs the stream directly; switch super-chunk mode off first (set_superchunk 0)", who, what);
        return -1;
    }
    // room one host call of n inputs may need in any output port
    size_t max_output(size_t n) const { return samples ? (n / samples + 2) * outcap : max_out(n); }
};

void HostBoundaryFree::operator()(HostBoundary* h) const { delete h; }

static constexpr size_t HOST_CHUNK = (size_t)1 << 24;   // input samples per chunk of a host-mode block's call

int Block::execute_multi(const void* const* x, int nin, size_t n, void* const* y, int nout, size_t* n_out) {
    if (nin != num_inputs || nout != num_outputs) {
        set_error("%s: expected %d input(s) and %d output(s), got %d and %d", name.c_str(), num_inputs, num_outputs, nin, nout);
        return -1;
    }
    size_t produced = 0;
    if (dev_ptrs) {
        if (run_multi(x, nin, n, y, nout, &produced, ctx().stream) != 0) return -1;
        if (n_out) *n_out = produced;
        return 0;
    }
    if (!host) {
        host.reset(new HostBoundary([this](const void* const* dx, size_t m, void* const* dy, size_t* no, cudaStream_t s) {
            if (run_multi(dx, num_inputs, m, dy, num_outputs, no, s) != 0) return -1;
            for (int o = 1; o < num_outputs; ++o) no[o] = no[0];      // every port produces the same count
            return 0;
        }, [this](size_t m) { return max_output(m); }, HOST_CHUNK));
        host->in_size.assign((size_t)nin, in_size);
        for (int o = 0; o < nout; ++o) host->out_size.push_back(out_size_of(o));
    }
    std::vector<size_t> counts((size_t)nout);
    if (host->execute(x, n, y, counts.data()) != 0) return -1;
    if (n_out) *n_out = counts[0];
    return 0;
}

// ---- time-chunk sharding (SURVEY.md 8e): where a stream can be cut, for graphs and DAGs alike ---------------------------
int Block::need_in(double need_out, double* need) const {
    const long long mem = memory_in();
    if (mem < 0) { set_error("%s has unbounded memory, the stream cannot be cut", name.c_str()); return -1; }
    unsigned bu, bd;
    rate(&bu, &bd);
    *need = std::ceil(need_out * (double)bd / (double)bu) + (double)mem + 1.0;
    return 0;
}

// The halo of a left-context need: whole output periods, and a multiple of 4 samples so that a chunk placed `halo`
// samples into a 16-byte aligned buffer stays 16-byte aligned (float32 and complex streams alike): the vectorised interior
// kernels need that.  `need` is a whole number (need_in adds whole numbers to a ceil), so the ceil only converts it.
static long long round_halo(double need, unsigned long long period) {
    const long long q = 4 * (long long)period;
    const long long h = (long long)std::ceil(need);
    return ((h + q - 1) / q) * q;
}

// The arguments of one shard of a stream whose output period is `period` input samples: 0 with *first set for the
// stream's first chunk (no halo, or start 0: nothing to its left), or -1 with the error set
static int shard_args(const char* who, size_t halo, uint64_t start, unsigned long long period, bool* first) {
    if (halo % period || start % period) { set_error("%s: halo and start must be multiples of %llu input samples", who, period); return -1; }
    *first = halo == 0 || start == 0;
    if (!*first && start < halo) { set_error("%s: chunk starts inside the halo", who); return -1; }
    return 0;
}

// A committed linear run of blocks, itself a one-port Block (a node of a Dag).  Its name is the description.
struct Graph : Block {
    Blocks blocks;                   // as appended
    Blocks fused;                    // blocks created by fusion
    std::vector<Block*> stages;      // execution order after commit (not owned)
    bool committed = false;
    DeviceBuffer ring[2];
    // time-chunk sharding (run_shard): scratch for the outputs that belong to the halo
    DeviceBuffer head_out;
    // optional per-stage timing
    bool timing = false;
    std::vector<std::vector<cudaEvent_t>> tev;   // per stage: [start0, stop0, start1, stop1, ...]
    std::vector<int> tcount;

    // element sizes and name (the description) are set by commit; host calls go in chunks of 2^23 samples
    Graph() : Block("", 8, 8, true) {
        host.reset(new HostBoundary([this](const void* const* dx, size_t n, void* const* dy, size_t* n_out, cudaStream_t s) {
            return run(dx[0], n, dy[0], n_out, s);
        }, [this](size_t n) { return max_output(n); }, (size_t)1 << 23));
    }
    // the boundary of host calls and super-chunk mode, sized for the committed stages
    HostBoundary* boundary() {
        if (ensure_committed() != 0) return nullptr;
        if (stages.empty()) { set_error("graph: no blocks"); return nullptr; }
        host->in_size.assign(1, in_size);
        host->out_size.assign(1, out_size);
        return host.get();
    }

    cudaEvent_t timing_event(size_t stage, size_t idx) {
        auto& v = tev[stage];
        while (v.size() <= idx) { cudaEvent_t e; cudaEventCreate(&e); v.push_back(e); }
        return v[idx];
    }
    // per-stage timing: events recorded on s around stage k's launches
    void timing_start(size_t k, cudaStream_t s) {
        if (!timing) return;
        if (tcount.size() < stages.size()) { tev.resize(stages.size()); tcount.assign(stages.size(), 0); }
        cudaEventRecord(timing_event(k, 2 * (size_t)tcount[k]), s);
    }
    void timing_stop(size_t k, cudaStream_t s) {
        if (!timing) return;
        cudaEventRecord(timing_event(k, 2 * (size_t)tcount[k] + 1), s);
        tcount[k]++;
    }

    ~Graph() override {
        for (auto& v : tev) for (cudaEvent_t e : v) cudaEventDestroy(e);
    }

    size_t max_output(size_t n) const override {
        for (Block* b : stages) n = b->max_output(n);
        return n;
    }
    uint64_t outputs_before(uint64_t idx) const override {
        for (Block* b : stages) idx = b->outputs_before(idx);
        return idx;
    }
    void rate(unsigned* up, unsigned* down) const override {
        const Rate r = total_rate();
        *up = (unsigned)r.up; *down = (unsigned)r.down;
    }

    int commit(int fuse) {
        stages.clear();
        fused.clear();
        name.clear();
        for (size_t i = 0; i < blocks.size();) {
            Rewrite rw;
            if (fuse)
                for (Rule rule : FUSION_RULES) {
                    if (rule(blocks, i, &rw) != 0) return -1;
                    if (rw.used) break;
                }
            Block* st = blocks[i].get();
            if (rw.used) { st = rw.stage.get(); fused.push_back(std::move(rw.stage)); }
            stages.push_back(st);
            if (!name.empty()) name += " | ";
            name += st->name;
            if (rw.used > 1) name += "[fused x" + std::to_string(rw.used) + "]";
            if (rw.stage2) {
                stages.push_back(rw.stage2.get());
                name += " | " + rw.stage2->name;
                fused.push_back(std::move(rw.stage2));
            }
            i += rw.used ? rw.used : 1;
        }
        for (size_t k = 0; k + 1 < stages.size(); ++k) {
            if (stages[k]->out_size != stages[k + 1]->in_size) {
                set_error("graph: %s (out %zu B) cannot feed %s (in %zu B)", stages[k]->name.c_str(), stages[k]->out_size,
                          stages[k + 1]->name.c_str(), stages[k + 1]->in_size);
                return -1;
            }
        }
        if (!stages.empty()) { in_size = stages.front()->in_size; out_size = stages.back()->out_size; }
        committed = true;
        return 0;
    }
    int ensure_committed() { return committed ? 0 : commit(1); }

    // grow the two-slot ring for a call of n inputs; a stage still in flight may be reading the old buffer
    int reserve_ring(size_t n, cudaStream_t s) {
        for (size_t k = 0; k + 1 < stages.size(); ++k) {
            n = stages[k]->max_output(n);
            const size_t bytes = (n ? n : 1) * stages[k]->out_size;
            DeviceBuffer& slot = ring[k & 1];
            if (bytes > slot.capacity()) {
                LRB_CHECK(cudaStreamSynchronize(s));
                if (slot.reserve(bytes) != 0) return -1;
            }
        }
        return 0;
    }

    // device in/out, asynchronous on s
    int run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) override {
        if (ensure_committed() != 0) return -1;
        if (stages.empty()) { set_error("graph: no blocks"); return -1; }
        if (reserve_ring(n, s) != 0) return -1;
        const void* in = dx;
        size_t cnt = n;
        for (size_t k = 0; k < stages.size(); ++k) {
            void* out = (k + 1 == stages.size()) ? dy : ring[k & 1].get();
            size_t no = 0;
            timing_start(k, s);
            if (stages[k]->run(in, cnt, out, &no, s) != 0) return -1;
            timing_stop(k, s);
            in = out;
            cnt = no;
        }
        *n_out = cnt;
        return 0;
    }

    // Block::reset for every block, with ONE launch zeroing the carried state of them all
    int reset(cudaStream_t s) {
        std::vector<void*> ptrs;
        std::vector<size_t> bytes;
        for (auto* list : {&blocks, &fused})
            for (auto& b : *list) {
                b->rewind();
                for (auto& sg : b->carried) { ptrs.push_back(sg.first); bytes.push_back(sg.second); }
            }
        if (ptrs.empty()) return 0;
        return launch_zero_segments(ptrs.data(), bytes.data(), (int)ptrs.size(), s);
    }
    int reset() override { return host->drop() != 0 ? -1 : reset(ctx().stream); }

    // ---- time-chunk sharding (SURVEY.md 8e) -------------------------------------------------------------------
    Rate total_rate() const {
        Rate r;
        for (Block* b : stages) r = r.then(*b);
        return r;
    }
    // the stages walked back from the output, each by the plain rule (a PLL's state is handed over only in a DAG)
    int need_in(double need_out, double* need) const override {
        for (size_t k = stages.size(); k-- > 0;)
            if (stages[k]->Block::need_in(need_out, &need_out) != 0) return -1;
        *need = need_out;
        return 0;
    }
    // input samples of left context a cold start needs so that the outputs equal the streaming ones to float32
    // resolution, as a halo; -1 when a stage's memory is unbounded
    long long halo() {
        double need = 0.0;
        if (ensure_committed() != 0 || need_in(0.0, &need) != 0) return -1;
        return round_halo(need, total_rate().down);
    }

    // One time chunk of a sharded stream.  dx -> [halo samples of the left neighbour | n samples of this chunk], the chunk
    // starting at global input index `start` (a multiple of the output period, like halo).  The stream is run COLD from
    // start - halo over halo + n samples -- every stage's memory has died out by `start` (halo()) -- and the halo's outputs
    // are dropped.  Only what reads the neighbour's samples waits for `halo_ready`: the first stage keeps the few tiles
    // that touch dx[0, halo) out of its interior kernel and runs them as edge tiles on the side stream behind the event
    // (Ctx::lead_samples / lead_event); everything else starts at once, so the exchange overlaps the chunk's kernels.
    // A first stage that cannot do that makes the compute stream wait for the event (the exchange is then serial).
    // The last stage runs as two streaming calls -- the inputs that belong to the halo (their outputs go to a scratch
    // buffer), then the rest straight into dy -- so dy receives exactly the chunk's outputs.
    int run_shard(const void* dx, size_t halo_n, size_t n, uint64_t start, void* dy, size_t* n_out, cudaEvent_t halo_ready) {
        if (ensure_committed() != 0) return -1;
        if (stages.empty()) { set_error("graph: no blocks"); return -1; }
        cudaStream_t s = ctx().stream;
        const size_t isz = in_size, osz = out_size;
        bool first;
        if (shard_args("graph", halo_n, start, total_rate().down, &first) != 0) return -1;
        if (first) {
            if (reset(s) != 0 || seek(start) != 0) return -1;
            return run((const char*)dx + halo_n * isz, n, dy, n_out, s);
        }
        if (reset(s) != 0 || seek(start - halo_n) != 0) return -1;
        const size_t K = stages.size();
        // inputs of every stage that belong to the halo: lead[k] = (stage-k input index of `start`) - (that of start - halo)
        std::vector<size_t> lead(K + 1);
        {
            uint64_t a = start - halo_n, b = start;
            for (size_t k = 0; k < K; ++k) {
                lead[k] = (size_t)(b - a);
                a = stages[k]->outputs_before(a);
                b = stages[k]->outputs_before(b);
            }
            lead[K] = (size_t)(b - a);                       // outputs of the halo: dropped
        }
        const size_t ho = lead[K];
        if ((ho + 1) * osz > head_out.capacity()) {
            LRB_CHECK(cudaStreamSynchronize(s));
            if (head_out.reserve((ho + 1) * osz) != 0) return -1;
        }
        const size_t n_tot = halo_n + n;
        if (reserve_ring(n_tot, s) != 0) return -1;
        const bool overlap = halo_ready && K >= 2 && stages[0]->supports_lead_wait();
        if (halo_ready && !overlap) LRB_CHECK(cudaStreamWaitEvent(s, halo_ready, 0));
        const void* in = dx;
        size_t cnt = n_tot;
        int rc = 0;
        for (size_t k = 0; k < K && rc == 0; ++k) {
            const bool last = k + 1 == K;
            timing_start(k, s);
            if (k == 0 && overlap) { ctx().lead_samples = (long long)halo_n; ctx().lead_event = halo_ready; ctx().reserve_ctas = 4; }
            size_t no = 0;
            if (!last) {
                void* out = ring[k & 1].get();
                rc = stages[k]->run(in, cnt, out, &no, s);
                in = out;
                cnt = no;
            } else {
                // two streaming calls: the halo's share of the inputs -> scratch, the chunk's -> dy
                // (the short first call goes to the side stream when the stage keeps every state access there: the second
                // call's interior kernel then starts without waiting for the first call's latency-bound edge kernel)
                size_t no1 = 0;
                const size_t m1 = lead[k] < cnt ? lead[k] : cnt;
                cudaStream_t s1 = (stages[k]->state_only_on_side_stream() && cnt - m1 >= SIDE_STREAM_MIN) ? side_fork(s) : s;
                rc = stages[k]->run(in, m1, head_out.get(), &no1, s1);
                if (rc == 0 && no1 != ho) { set_error("graph: halo produced %zu outputs, expected %zu", no1, ho); rc = -1; }
                if (rc == 0) rc = stages[k]->run((const char*)in + m1 * stages[k]->in_size, cnt - m1, dy, &no, s);
                side_join(s, s1);
                cnt = no;
            }
            if (k == 0) { ctx().lead_samples = 0; ctx().lead_event = nullptr; ctx().reserve_ctas = 0; }
            timing_stop(k, s);
        }
        if (rc != 0) return -1;
        *n_out = cnt;
        return 0;
    }

    int seek(uint64_t idx) override {
        if (ensure_committed() != 0) return -1;
        for (Block* b : stages) {
            if (b->seek(idx) != 0) return -1;
            idx = b->outputs_before(idx);
        }
        return 0;
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// Device DAG: fan-out / fan-in between GPU nodes without host hops.  A node is a multi-port block (MultiplyConjugate, Add,
// Subtract, PLL, ...), a single block, or a committed LINEAR flow graph (so the fused kernels keep doing the work inside
// every linear run).  Nodes are added in topological order; an input reference is (producer node, output port) or the
// DAG's own input.  Every edge is a grow-only device buffer; all inputs of a node must deliver the same number of samples
// per call (true whenever the converging paths have the same rate changes -- every block here is zero-latency; the
// reference's PipeMux would buffer a surplus instead, radio/core/pipe.lua:495-615).  Host in, host out(s) through the
// HostBoundary above, a whole call as one chunk: one upload, the node launches in order on the library stream, one
// download per output, one synchronize; or host vectors packed into super-chunks; or the same launches on device-resident
// input and outputs with no synchronize.
// This is what composites/wbfmstereodemodulator.lua:22-64 and amsynchronousdemodulator.lua:25-45 need on the device.
// ---------------------------------------------------------------------------------------------------------------------
// An output port of a node, or (node -1) the DAG's input.  The C ABI encodes it as node * 4 + port, or -1.
struct PortRef {
    int node = -1, port = 0;
    bool is_input() const { return node < 0; }
};

struct DagNode {
    std::unique_ptr<Block> blk;    // a block, or a committed linear Graph
    int members = 1;               // the blocks a DAG rewrite folded into this node (the description's [fused xN])
    std::vector<PortRef> ins;
    std::vector<DeviceBuffer> out_buf;
    std::vector<size_t> out_cnt;
    std::vector<void*> out_ptr;    // where each port's samples of the current call are (out_buf, or a caller's dy)
    // time-chunk sharding, from the DAG's shape (Dag::plan)
    double need_out = 0.0;         // outputs of left context its consumers and ports need
    bool below_pll = false;        // a transitive consumer of a PLL
    PllBlock* pll = nullptr;       // the block as a PLL whose state is handed over (set by add), with its record's index
    int rec = -1;
    long long probe = -1;          // a PLL's probe point in the first shard's run (shard_begin), or -1
};

// What a DAG rule made of the nodes around nodes[at]: one node standing for `members` blocks, fed by `in`, in the place of
// nodes[at]; the nodes in `gone` go.  No match: node stays null.
struct DagRewrite {
    std::unique_ptr<Block> node;
    PortRef in;
    std::vector<int> gone;
    int members = 0;
};
struct Dag;
// 0 (a match or none, see out->node), or -1 with the error set
using DagRule = int (*)(const Dag& dag, size_t at, DagRewrite* out);
extern const DagRule DAG_RULES[1];

struct Dag {
    std::vector<DagNode> nodes;
    std::vector<PortRef> outputs;  // never the DAG input
    size_t in_size = 0;
    std::string desc;
    // commit applies the DAG rules (fuse != 0) once the nodes and outputs are known.  A DAG not committed by the caller is
    // committed with fuse = 1 by its first run, halo, seek, super-chunk size or description.  Once a rule has rewritten
    // nodes, node ids have changed: adding nodes or setting outputs is refused from then on.
    bool committed = false, rewritten = false;
    int fuse = 1;

    int refuse_after_rewrite(const char* what) const {
        if (!rewritten) return 0;
        set_error("dag: %s after commit fused nodes (node ids have changed)", what);
        return -1;
    }
    // how many node inputs and DAG outputs read port p
    int consumers(PortRef p) const {
        int c = 0;
        for (const DagNode& nd : nodes)
            for (PortRef q : nd.ins) c += (!q.is_input() && q.node == p.node && q.port == p.port);
        for (PortRef q : outputs) c += (q.node == p.node && q.port == p.port);
        return c;
    }
    int commit(int fuse_);
    int ensure_committed() { return committed ? 0 : commit(fuse); }
    // nodes[at] becomes rw.node, the nodes in rw.gone go, and every reference follows the renumbering
    void apply(size_t at, DagRewrite& rw) {
        std::vector<int> remap(nodes.size(), -1);
        std::vector<bool> drop(nodes.size(), false);
        for (int g : rw.gone) drop[(size_t)g] = true;
        std::vector<DagNode> kept;
        for (size_t j = 0; j < nodes.size(); ++j) {
            if (drop[j]) continue;
            remap[j] = (int)kept.size();
            if (j != at) { kept.push_back(std::move(nodes[j])); continue; }
            DagNode nd;
            nd.blk = std::move(rw.node);
            nd.members = rw.members;
            nd.ins.assign(1, rw.in);
            nd.out_buf.resize((size_t)nd.blk->num_outputs);
            nd.out_cnt.assign((size_t)nd.blk->num_outputs, 0);
            nd.out_ptr.assign((size_t)nd.blk->num_outputs, nullptr);
            kept.push_back(std::move(nd));
        }
        for (DagNode& nd : kept)
            for (PortRef& q : nd.ins) if (!q.is_input()) q.node = remap[(size_t)q.node];
        for (PortRef& q : outputs) q.node = remap[(size_t)q.node];
        nodes = std::move(kept);
    }
    // host calls and super-chunk mode; the run writes each output port straight into the boundary's staging
    HostBoundary host{[this](const void* const* dx, size_t n, void* const* dy, size_t* n_out, cudaStream_t s) {
        return run_nodes(dx[0], n, dy, n_out, s);
    }, [this](size_t n) { return max_output(n); }, ~(size_t)0};

    // the boundary, sized for the current input and output ports
    HostBoundary* boundary() {
        if (nodes.empty() || outputs.empty()) { set_error("dag: no nodes / no outputs"); return nullptr; }
        if (ensure_committed() != 0) return nullptr;
        host.in_size.assign(1, in_size);
        host.out_size.resize(outputs.size());
        for (size_t k = 0; k < outputs.size(); ++k) host.out_size[k] = out_size(k);
        return &host;
    }

    // on success the DAG owns blk; on failure the caller keeps it
    int add(Block* blk, const int* refs, unsigned nin) {
        if (refuse_after_rewrite("add") != 0) return -1;
        committed = false;
        DagNode nd;
        nd.blk.reset(blk);
        nd.pll = blk->as_pll();
        if (wire(nd, refs, nin) != 0) { nd.blk.release(); return -1; }
        nd.out_buf.resize((size_t)blk->num_outputs);
        nd.out_cnt.assign((size_t)blk->num_outputs, 0);
        nd.out_ptr.assign((size_t)blk->num_outputs, nullptr);
        sh.planned = false;
        if (!desc.empty()) desc += " ; ";
        desc += blk->name;
        nodes.push_back(std::move(nd));
        return (int)nodes.size() - 1;
    }

    int wire(DagNode& nd, const int* refs, unsigned nin) {
        const Block& b = *nd.blk;
        if ((int)nin != b.num_inputs) { set_error("dag: %s takes %d input(s), got %u", b.name.c_str(), b.num_inputs, nin); return -1; }
        for (unsigned i = 0; i < nin; ++i) {
            PortRef r;
            size_t esz;
            if (refs[i] == -1) {
                if (in_size && in_size != b.in_size) { set_error("dag: the input feeds nodes of different sample sizes"); return -1; }
                in_size = b.in_size;
                esz = in_size;
            } else {
                if (decode(refs[i], &r) != 0) { set_error("dag: bad input reference %d", refs[i]); return -1; }
                esz = node(r).blk->out_size_of(r.port);
            }
            if (esz != b.in_size) { set_error("dag: %zu-byte samples cannot feed %s (%zu-byte input)", esz, b.name.c_str(), b.in_size); return -1; }
            nd.ins.push_back(r);
        }
        return 0;
    }

    // an ABI reference to an existing node's output port: 0, or -1 (no such port)
    int decode(int ref, PortRef* r) const {
        if (ref < 0 || (ref >> 2) >= (int)nodes.size() || (ref & 3) >= nodes[(size_t)(ref >> 2)].blk->num_outputs) return -1;
        *r = PortRef{ref >> 2, ref & 3};
        return 0;
    }
    const DagNode& node(PortRef r) const { return nodes[(size_t)r.node]; }
    // where port r's samples of the current call are, and how many (the DAG input: dx, n)
    const void* port_ptr(PortRef r, const void* dx) const { return r.is_input() ? dx : node(r).out_ptr[(size_t)r.port]; }
    size_t port_cnt(PortRef r, size_t n) const { return r.is_input() ? n : node(r).out_cnt[(size_t)r.port]; }

    size_t out_size(size_t k) const { return node(outputs[k]).blk->out_size_of(outputs[k].port); }
    // conservative: no node here produces more samples than its input times the interpolation factors on the way
    size_t max_output(size_t n) const {
        size_t m = n;
        for (const DagNode& nd : nodes) { const size_t c = nd.blk->max_output(n); if (c > m) m = c; }
        return m;
    }

    // back to the state after creation: the slots in flight are waited for and dropped with the partial slot (the
    // super-chunk size stays), then every node's carried state is zeroed
    int reset() {
        if (host.drop() != 0) return -1;
        for (DagNode& nd : nodes)
            if (nd.blk->reset() != 0) return -1;
        return 0;
    }

    // The node launches of one call, asynchronous on s: the DAG input is dx (n samples, device).  With dy, output k's
    // n_out[k] samples go to dy[k] (the producing node writes there, and its consumers read them there); without, they
    // stay in the producer's edge buffer.  Every count is host arithmetic, so nothing here synchronizes except growing
    // an edge buffer.
    int run_nodes(const void* dx, size_t n, void* const* dy, size_t* n_out, cudaStream_t s) {
        if (nodes.empty() || outputs.empty()) { set_error("dag: no nodes / no outputs"); return -1; }
        for (size_t i = 0; i < nodes.size(); ++i)
            if (run_node(i, dx, n, dy, s) != 0) return -1;
        for (size_t k = 0; k < outputs.size(); ++k) {
            const void* p = port_ptr(outputs[k], nullptr);
            const size_t c = port_cnt(outputs[k], 0);
            // an output listed twice: the producer wrote the first dy only
            if (dy && c && p != dy[k]) LRB_CHECK(cudaMemcpyAsync(dy[k], p, c * out_size(k), cudaMemcpyDeviceToDevice, s));
            n_out[k] = c;
        }
        return 0;
    }

    // node i's inputs (all of the same length *cnt) and the places its ports write: a caller's dy[k] for output port k,
    // else its grown edge buffer
    int node_io(size_t i, const void* dx, size_t n, void* const* dy, std::vector<const void*>& ins, size_t* cnt, void** outs,
                cudaStream_t s) {
        DagNode& nd = nodes[i];
        ins.clear();
        *cnt = 0;
        for (size_t j = 0; j < nd.ins.size(); ++j) {
            const size_t c = port_cnt(nd.ins[j], n);
            if (j && c != *cnt) { set_error("dag: %s received inputs of different lengths (%zu, %zu)", nd.blk->name.c_str(), *cnt, c); return -1; }
            *cnt = c;
            ins.push_back(port_ptr(nd.ins[j], dx));
        }
        const size_t mo = nd.blk->max_output(*cnt);
        for (int o = 0; o < nd.blk->num_outputs; ++o) {
            void* ext = nullptr;
            for (size_t k = 0; dy && k < outputs.size() && !ext; ++k)
                if (outputs[k].node == (int)i && outputs[k].port == o) ext = dy[k];
            if (!ext) {
                DeviceBuffer& buf = nd.out_buf[(size_t)o];
                const size_t bytes = (mo ? mo : 1) * nd.blk->out_size_of(o);
                if (bytes > buf.capacity()) {
                    LRB_CHECK(cudaStreamSynchronize(s));
                    if (buf.reserve(bytes) != 0) return -1;
                }
                ext = buf.get();
            }
            outs[o] = nd.out_ptr[(size_t)o] = ext;
        }
        return 0;
    }

    // One node's launches.  A PLL with a probe point (the first rank of a sharded stream) also leaves its state there in
    // its record.
    int run_node(size_t i, const void* dx, size_t n, void* const* dy, cudaStream_t s) {
        DagNode& nd = nodes[i];
        std::vector<const void*> ins;
        size_t cnt = 0;
        void* outs[4];                 // a port is two bits of a reference
        if (node_io(i, dx, n, dy, ins, &cnt, outs, s) != 0) return -1;
        size_t no = 0;
        if (nd.probe >= 0) {
            if (nd.pll->run_probe(ins[0], cnt, outs, nd.probe, rec_dev(nd), s) != 0) return -1;
            no = cnt;
        } else if (nd.blk->run_multi(ins.data(), (int)ins.size(), cnt, outs, nd.blk->num_outputs, &no, s) != 0) {
            return -1;
        }
        for (int o = 0; o < nd.blk->num_outputs; ++o) nd.out_cnt[(size_t)o] = no;
        return 0;
    }

    // ---- time-chunk sharding (SURVEY.md 8e) ---------------------------------------------------------------------------
    // A shard runs the stream cold from start - halo and drops every port's outputs of the halo, as Graph::run_shard.  A
    // PLL's multiplied phase integrates the whole past, so its state is handed over instead: at the PLL input index h of
    // a shard's start, less what everything behind the PLL needs of left context (from h on, the PLL's outputs reach the
    // shard's kept outputs), the loop is speculated from a lead-in over the halo (the chunk-parallel form's speculation,
    // pll.cu), checked against the left shard's state at h, re-run from that state on a miss, and the VCO output is
    // started from the sum of the left shards' advances of the multiplied phase.  A shard's record is one
    // PllShardRecord per PLL, in node order.
    struct ShardState {
        std::vector<int> plls;                 // node ids of the PLLs
        unsigned long long period = 1;         // lcm of every output port's total decimation
        double need = 0.0;                     // input samples of left context, unrounded
        // the shard between begin and end
        bool pending = false, first = false;
        const void* dx = nullptr;              // the DAG input (a PLL or a node behind one may read it)
        uint64_t start = 0;
        size_t halo = 0, n = 0;
        std::vector<size_t> skip;              // per port: outputs of the halo
        bool planned = false;
    };
    ShardState sh;
    DeviceBuffer d_rec;
    std::vector<PllShardRecord> h_rec;     // host copy of this shard's record

    PllShardRecord* rec_dev(const DagNode& nd) { return d_rec.as<PllShardRecord>() + nd.rec; }
    size_t record_bytes() { return plan() != 0 ? 0 : sizeof(PllShardRecord) * sh.plls.size(); }

    // needs, PLLs and the period, from the shape alone; -1 with the error set when the stream cannot be cut
    int plan() {
        if (sh.planned) return 0;
        if (nodes.empty() || outputs.empty()) { set_error("dag: no nodes / no outputs"); return -1; }
        if (ensure_committed() != 0) return -1;
        sh.plls.clear();
        std::vector<Rate> rate(nodes.size());                  // total rate at each node's output
        for (size_t i = 0; i < nodes.size(); ++i) {
            DagNode& nd = nodes[i];
            nd.need_out = 0.0;
            nd.below_pll = false;
            nd.rec = -1;
            Rate r;
            for (PortRef p : nd.ins)
                if (!p.is_input()) {
                    if (node(p).below_pll || node(p).pll) nd.below_pll = true;
                    r = rate[(size_t)p.node];
                }
            if (nd.pll && nd.below_pll) { set_error("dag: %s behind another pll, the stream cannot be cut", nd.blk->name.c_str()); return -1; }
            if (nd.pll) { nd.rec = (int)sh.plls.size(); sh.plls.push_back((int)i); }
            rate[i] = r.then(*nd.blk);
        }
        sh.period = 1;
        for (PortRef p : outputs) sh.period = std::lcm(sh.period, rate[(size_t)p.node].down);
        // walk back from the ports: each node's need at its input from its need at its output
        sh.need = 0.0;
        for (size_t i = nodes.size(); i-- > 0;) {
            double need;
            if (nodes[i].blk->need_in(nodes[i].need_out, &need) != 0) return -1;
            for (PortRef p : nodes[i].ins) {
                double& t = p.is_input() ? sh.need : nodes[(size_t)p.node].need_out;
                t = need > t ? need : t;
            }
        }
        sh.planned = true;
        return 0;
    }

    long long halo() { return plan() != 0 ? -1 : round_halo(sh.need, sh.period); }

    // every node's input index once the DAG input's first `g` samples are consumed
    std::vector<uint64_t> in_index(uint64_t g) const {
        std::vector<uint64_t> idx(nodes.size());
        for (size_t i = 0; i < nodes.size(); ++i) {
            const PortRef r = nodes[i].ins.empty() ? PortRef{} : nodes[i].ins[0];
            idx[i] = r.is_input() ? g : node(r).blk->outputs_before(idx[(size_t)r.node]);
        }
        return idx;
    }

    int seek(uint64_t g) {
        if (ensure_committed() != 0) return -1;
        const std::vector<uint64_t> idx = in_index(g);
        for (size_t i = 0; i < nodes.size(); ++i)
            if (nodes[i].blk->seek(idx[i]) != 0) return -1;
        return 0;
    }

    int check_record(size_t bytes) {
        const size_t want = record_bytes();
        if (bytes != want) { set_error("dag: a record of this DAG is %zu bytes, got %zu", want, bytes); return -1; }
        return 0;
    }

    // the kept outputs of port k (from its node's edge buffer) to dy[k]
    int copy_port(size_t k, void* const* dy, size_t* n_out, cudaStream_t s) {
        const size_t c = port_cnt(outputs[k], 0), sk = sh.skip[k];
        if (c < sk) { set_error("dag: output %zu: the halo produced %zu outputs, expected %zu", k, c, sk); return -1; }
        if (c > sk) LRB_CHECK(cudaMemcpyAsync(dy[k], (const char*)port_ptr(outputs[k], nullptr) + sk * out_size(k),
                                              (c - sk) * out_size(k), cudaMemcpyDeviceToDevice, s));
        n_out[k] = c - sk;
        return 0;
    }

    bool port_in_phase_b(size_t k) const {
        const DagNode& nd = node(outputs[k]);
        return nd.below_pll || nd.pll;
    }

    int shard_begin(const void* dx, size_t halo_n, size_t n, uint64_t start, void* const* dy, size_t* n_out, void* record,
                    size_t record_bytes_) {
        if (host.refuse_direct("dag", "sharding") != 0 || plan() != 0 || check_record(record_bytes_) != 0) return -1;
        bool first;
        if (shard_args("dag", halo_n, start, sh.period, &first) != 0) return -1;
        sh.pending = false;
        if (reset() != 0) return -1;
        cudaStream_t s = ctx().stream;
        const size_t npll = sh.plls.size();
        if (npll && d_rec.reserve(sizeof(PllShardRecord) * npll) != 0) return -1;
        const uint64_t g0 = first ? start : start - halo_n;
        if (seek(g0) != 0) return -1;
        const std::vector<uint64_t> a0 = in_index(g0), a1 = in_index(start), a2 = in_index(start + n);
        // handoff points of each PLL, as indices into this call's PLL input
        std::vector<long long> lh(nodes.size(), -1), le(nodes.size(), -1);
        for (int p : sh.plls) {
            const long long D = (long long)std::ceil(nodes[(size_t)p].need_out);
            lh[(size_t)p] = (long long)a1[(size_t)p] - D - (long long)a0[(size_t)p];
            le[(size_t)p] = (long long)a2[(size_t)p] - D - (long long)a0[(size_t)p];
            if (le[(size_t)p] < (first ? 0 : lh[(size_t)p])) { set_error("dag: the chunk is shorter than what follows %s needs", nodes[(size_t)p].blk->name.c_str()); return -1; }
        }
        sh.skip.assign(outputs.size(), 0);
        int rc = 0;
        if (first) {
            // the plain run, with each PLL's state at the next shard's handoff point
            for (int p : sh.plls) nodes[(size_t)p].probe = le[(size_t)p];
            rc = run_nodes((const char*)dx + halo_n * in_size, n, dy, n_out, s);
            for (int p : sh.plls) nodes[(size_t)p].probe = -1;
        } else {
            for (size_t k = 0; k < outputs.size(); ++k) {
                const size_t i = (size_t)outputs[k].node;
                sh.skip[k] = (size_t)(nodes[i].blk->outputs_before(a1[i]) - nodes[i].blk->outputs_before(a0[i]));
            }
            const size_t N = halo_n + n;
            for (size_t i = 0; i < nodes.size() && rc == 0; ++i) {
                DagNode& nd = nodes[i];
                if (nd.below_pll) continue;
                if (!nd.pll) { rc = run_node(i, dx, N, nullptr, s); continue; }
                std::vector<const void*> ins;
                size_t cnt = 0;
                void* outs[4];
                rc = node_io(i, dx, N, nullptr, ins, &cnt, outs, s);
                if (rc == 0) rc = nd.pll->shard_loop(ins[0], cnt, (float*)outs[1], lh[i], le[i], rec_dev(nd), s);
                nd.out_cnt[0] = nd.out_cnt[1] = cnt;
            }
            for (size_t k = 0; k < outputs.size() && rc == 0; ++k) {
                n_out[k] = 0;
                if (!port_in_phase_b(k)) rc = copy_port(k, dy, n_out, s);
            }
        }
        if (rc != 0) return -1;
        h_rec.assign(npll, PllShardRecord{});
        if (npll) {
            LRB_CHECK(cudaMemcpyAsync(h_rec.data(), d_rec.get(), sizeof(PllShardRecord) * npll, cudaMemcpyDeviceToHost, s));
            LRB_CHECK(cudaStreamSynchronize(s));
            for (PllShardRecord& r : h_rec) {
                r.first = first ? 1.0 : 0.0;
                if (first) r.spec_phi = r.spec_freq = 0.0;      // no speculated start
            }
            memcpy(record, h_rec.data(), sizeof(PllShardRecord) * npll);
        }
        sh.pending = true;
        sh.first = first;
        sh.start = start; sh.halo = halo_n; sh.n = n; sh.dx = dx;
        return 0;
    }

    // does this shard's speculated start agree with the left shard's end state, for every PLL?
    int shard_accepts(const PllShardRecord* left, const PllShardRecord* own) {
        for (size_t j = 0; j < sh.plls.size(); ++j) {
            if (own[j].first != 0.0) continue;                      // a first shard starts from the reset state
            const PllBlock* p = nodes[(size_t)sh.plls[j]].pll;
            if (!p->accepts(left[j].end_phi, left[j].end_freq, own[j].spec_phi, own[j].spec_freq)) return 0;
        }
        return 1;
    }

    int shard_end(const PllShardRecord* left, unsigned num_left, void* const* dy, size_t* n_out, void* record_out, size_t record_bytes_) {
        if (!sh.pending) { set_error("dag: shard_end without shard_begin"); return -1; }
        if (check_record(record_bytes_) != 0) return -1;
        const size_t npll = sh.plls.size();
        cudaStream_t s = ctx().stream;
        if (sh.first) {
            for (size_t k = 0; k < outputs.size(); ++k) n_out[k] = port_cnt(outputs[k], 0);
            if (npll) memcpy(record_out, h_rec.data(), sizeof(PllShardRecord) * npll);
            sh.pending = false;
            return 0;
        }
        if (npll && num_left == 0) { set_error("dag: a shard after the first needs the records of the shards to its left"); return -1; }
        bool rerun = false;
        int rc = 0;
        for (size_t j = 0; j < npll && rc == 0; ++j) {
            DagNode& nd = nodes[(size_t)sh.plls[j]];
            const PllShardRecord& l = left[npll * (size_t)(num_left - 1) + j];
            const PllShardRecord& o = h_rec[j];
            const double base = PllBlock::fold_advances(left, num_left, npll, j);
            if (!nd.pll->accepts(l.end_phi, l.end_freq, o.spec_phi, o.spec_freq)) {
                rerun = true;
                rc = nd.pll->shard_rerun(port_ptr(nd.ins[0], sh.dx), (float*)nd.out_ptr[1], l.end_phi, l.end_freq, rec_dev(nd), s);
            }
            if (rc == 0) rc = nd.pll->shard_out((const float*)nd.out_ptr[1], (float2*)nd.out_ptr[0], base, s);
        }
        const size_t N = sh.halo + sh.n;
        for (size_t i = 0; i < nodes.size() && rc == 0; ++i)
            if (nodes[i].below_pll) rc = run_node(i, sh.dx, N, nullptr, s);
        for (size_t k = 0; k < outputs.size() && rc == 0; ++k) {
            if (port_in_phase_b(k)) rc = copy_port(k, dy, n_out, s);
            else n_out[k] = port_cnt(outputs[k], 0) - sh.skip[k];
        }
        if (rc != 0) return -1;
        if (rerun) {
            // only the end states are the device's: the speculated start and the first-shard flag stay the host's
            std::vector<PllShardRecord> dev(npll);
            LRB_CHECK(cudaMemcpyAsync(dev.data(), d_rec.get(), sizeof(PllShardRecord) * npll, cudaMemcpyDeviceToHost, s));
            LRB_CHECK(cudaStreamSynchronize(s));
            for (size_t j = 0; j < npll; ++j) {
                h_rec[j].end_phi = dev[j].end_phi;
                h_rec[j].end_dP = dev[j].end_dP;
                h_rec[j].end_freq = dev[j].end_freq;
            }
        }
        if (npll) memcpy(record_out, h_rec.data(), sizeof(PllShardRecord) * npll);
        sh.pending = false;
        return rerun ? 1 : 0;
    }
};

// ---- device DAG rewrites: one rule function per rewrite, tried at every node when the DAG is committed ------------------

// The FIR -> ComplexMagnitude branch whose magnitude is port p: a committed graph node `fir | cmag`, or a FIR node read only
// by a magnitude node.  The FIR is cccf, D = 1, no fused translator, M <= FFT_MAX_TAPS; no port inside the branch has
// another reader or is a DAG output.
struct FskBranch {
    FirBlock* fir = nullptr;
    PortRef in;                      // what the FIR reads
    std::vector<int> nodes;
};
static bool fsk_branch(const Dag& d, PortRef p, FskBranch* b) {
    if (p.is_input() || d.consumers(p) != 1) return false;
    const DagNode& m = d.nodes[(size_t)p.node];
    C2fBlock* mag = nullptr;
    if (Graph* g = dynamic_cast<Graph*>(m.blk.get())) {
        if (g->stages.size() != 2) return false;
        b->fir = dynamic_cast<FirBlock*>(g->stages[0]);
        mag = dynamic_cast<C2fBlock*>(g->stages[1]);
        b->in = m.ins[0];
        b->nodes = {p.node};
    } else if ((mag = dynamic_cast<C2fBlock*>(m.blk.get())) != nullptr) {
        const PortRef q = m.ins[0];
        if (q.is_input() || d.consumers(q) != 1) return false;
        b->fir = dynamic_cast<FirBlock*>(d.nodes[(size_t)q.node].blk.get());
        b->in = d.nodes[(size_t)q.node].ins[0];
        b->nodes = {q.node, p.node};
    }
    const FirBlock* f = b->fir;
    return mag && mag->op == 0 && f && f->kind == FIR_CCCF && f->D == 1 && !f->rotate && f->M <= FFT_MAX_TAPS && f->fast;
}

// ComplexBandpass(h_a) -> ComplexMagnitude and ComplexBandpass(h_b) -> ComplexMagnitude on one input, into Subtract's in1
// and in2  =>  FskDetectBlock, |x * h_a| - |x * h_b| in one kernel (the POCSAG receiver's mark/space detector,
// composites/pocsagreceiver.lua:28-45): the input is read once, and neither the two complex FIR outputs nor the two
// magnitudes go through HBM.  Any two tap sets of equal length; the FIRs' algorithm settings carry over.
static int fuse_fsk_detector(const Dag& d, size_t at, DagRewrite* out) {
    const DagNode& sub = d.nodes[at];
    const BinaryBlock* bin = dynamic_cast<const BinaryBlock*>(sub.blk.get());
    if (!bin || bin->op != BIN_SUB || bin->cplx) return 0;
    FskBranch br[2];
    if (!fsk_branch(d, sub.ins[0], &br[0]) || !fsk_branch(d, sub.ins[1], &br[1])) return 0;
    if (br[0].fir == br[1].fir || br[0].fir->M != br[1].fir->M) return 0;
    if (br[0].in.node != br[1].in.node || br[0].in.port != br[1].in.port) return 0;
    std::unique_ptr<FirBlock> member[2];
    for (int k = 0; k < 2; ++k) {
        const FirBlock& f = *br[k].fir;
        member[k] = make_block<FirBlock>(FIR_CCCF, f.h_taps.data(), (unsigned)f.M, 1u, true);
        if (!member[k] || member[k]->set_algorithm(f.algo) != 0) return -1;
    }
    out->node = make_block<FskDetectBlock>(std::move(member[0]), std::move(member[1]), true);
    if (!out->node) return -1;
    out->in = br[0].in;
    out->gone = br[0].nodes;
    out->gone.insert(out->gone.end(), br[1].nodes.begin(), br[1].nodes.end());
    out->members = 5;
    return 0;
}

const DagRule DAG_RULES[1] = {fuse_fsk_detector};

int Dag::commit(int fuse_) {
    if (rewritten && !fuse_) { set_error("dag: commit(0) after commit fused nodes"); return -1; }
    fuse = fuse_;
    if (fuse && !outputs.empty()) {
        for (size_t i = 0; i < nodes.size(); ++i)
            for (DagRule rule : DAG_RULES) {
                DagRewrite rw;
                if (rule(*this, i, &rw) != 0) return -1;
                if (!rw.node) continue;
                apply(i, rw);
                rewritten = true;
                sh.planned = false;
                i = (size_t)-1;              // from the start: the renumbered nodes may match again
                break;
            }
    }
    desc.clear();
    for (const DagNode& nd : nodes) {
        if (!desc.empty()) desc += " ; ";
        desc += nd.blk->name;
        if (nd.members > 1) desc += "[fused x" + std::to_string(nd.members) + "]";
    }
    committed = true;
    return 0;
}

}  // namespace lrb

using namespace lrb;

struct lrb200_graph_s { std::unique_ptr<Graph> g; };
struct lrb200_dag_s { Dag d; };

extern "C" {

lrb200_graph_t* lrb200_graph_create(void) {
    if (lrb200_device_count() <= 0) { set_error("no CUDA device available; libluaradio_b200 has no CPU fallback"); return nullptr; }
    if (ctx().device < 0 && lrb200_init(0) != 0) return nullptr;
    std::unique_ptr<Graph> impl(new (std::nothrow) Graph());
    lrb200_graph_t* g = impl ? new (std::nothrow) lrb200_graph_s{std::move(impl)} : nullptr;
    if (!g) set_error("out of memory");
    return g;
}

int lrb200_graph_append(lrb200_graph_t* g, lrb200_block_t* q) {
    if (!g || !q || !q->impl) { set_error("graph_append: null handle"); return -1; }
    if (!q->impl->dev_ptrs) { set_error("graph_append: block %s was not created with LRB200_DEVICE", q->impl->name.c_str()); return -1; }
    Blocks& blocks = g->g->blocks;
    if (!blocks.empty() && blocks.back()->out_size != q->impl->in_size) {
        set_error("graph_append: %s (out %zu B) cannot feed %s (in %zu B)", blocks.back()->name.c_str(),
                  blocks.back()->out_size, q->impl->name.c_str(), q->impl->in_size);
        return -1;
    }
    blocks.emplace_back(q->impl);
    g->g->committed = false;
    q->impl = nullptr;          // ownership moves to the graph
    delete q;
    return 0;
}

int lrb200_graph_commit(lrb200_graph_t* g, int fuse) {
    if (!g) { set_error("null graph"); return -1; }
    return g->g->commit(fuse);
}

int lrb200_graph_execute(lrb200_graph_t* g, const void* x, size_t n, void* y, size_t* n_out) {
    if (!g) { set_error("null graph"); return -1; }
    size_t no = 0;
    HostBoundary* hb = g->g->boundary();
    int rc = hb ? hb->execute(&x, n, &y, &no) : -1;
    if (n_out) *n_out = no;
    return rc;
}

int lrb200_graph_execute_device(lrb200_graph_t* g, const void* dx, size_t n, void* dy, size_t* n_out) {
    if (!g) { set_error("null graph"); return -1; }
    size_t no = 0;
    int rc = g->g->host->refuse_direct("graph", "execute_device") != 0 ? -1 : g->g->run(dx, n, dy, &no, ctx().stream);
    if (n_out) *n_out = no;
    return rc;
}

size_t lrb200_graph_max_output(const lrb200_graph_t* g, size_t n) {
    if (!g) return 0;
    Graph& gr = *g->g;
    if (gr.ensure_committed() != 0) return 0;
    // super-chunk mode: one call may hand back the results of the slots completed while n samples were appended
    return gr.host->max_output(n);
}

int lrb200_graph_set_superchunk(lrb200_graph_t* g, size_t samples) {
    if (!g) { set_error("null graph"); return -1; }
    HostBoundary* hb = g->g->boundary();
    return hb ? hb->set_superchunk(samples, "graph") : -1;
}

int lrb200_graph_flush(lrb200_graph_t* g, void* y, size_t* n_out) {
    if (!g) { set_error("null graph"); return -1; }
    size_t no = 0;
    int rc = g->g->host->flush(&y, &no);     // 0 samples with super-chunk mode off or nothing fed
    if (n_out) *n_out = no;
    return rc;
}

long long lrb200_graph_halo(lrb200_graph_t* g) {
    if (!g) { set_error("null graph"); return -1; }
    return g->g->halo();
}

int lrb200_graph_execute_shard(lrb200_graph_t* g, lrb200_graph_t* g_head, const void* dx, size_t halo, size_t n,
                               uint64_t start, void* dy, size_t* n_out, void* halo_ready_event) {
    if (!g) { set_error("null graph"); return -1; }
    size_t no = 0;
    (void)g_head;
    int rc = g->g->host->refuse_direct("graph", "sharding") != 0 ? -1 : g->g->run_shard(dx, halo, n, start, dy, &no, (cudaEvent_t)halo_ready_event);
    if (n_out) *n_out = no;
    return rc;
}

int lrb200_graph_reset(lrb200_graph_t* g) {
    if (!g) { set_error("null graph"); return -1; }
    return g->g->reset();
}

int lrb200_graph_seek(lrb200_graph_t* g, uint64_t sample_index) {
    if (!g) { set_error("null graph"); return -1; }
    return g->g->seek(sample_index);
}

int lrb200_graph_num_stages(const lrb200_graph_t* g) {
    if (!g) return 0;
    if (g->g->ensure_committed() != 0) return -1;
    return (int)g->g->stages.size();
}

const char* lrb200_graph_describe(const lrb200_graph_t* g) {
    if (!g) return "";
    if (g->g->ensure_committed() != 0) return "";
    return g->g->name.c_str();
}

const char* lrb200_graph_stage_name(const lrb200_graph_t* g, int stage) {
    if (!g) return "";
    Graph& gr = *g->g;
    if (gr.ensure_committed() != 0) return "";
    if (stage < 0 || stage >= (int)gr.stages.size()) return "";
    return gr.stages[stage]->name.c_str();
}

int lrb200_graph_set_timing(lrb200_graph_t* g, int enable) {
    if (!g) { set_error("null graph"); return -1; }
    g->g->timing = enable != 0;
    return 0;
}

double lrb200_graph_stage_time_ms(lrb200_graph_t* g, int stage, int* executions) {
    if (executions) *executions = 0;
    if (!g || stage < 0 || stage >= (int)g->g->tcount.size()) return 0.0;
    if (cudaStreamSynchronize(ctx().stream) != cudaSuccess) return 0.0;
    double total = 0.0;
    int cnt = g->g->tcount[stage];
    for (int i = 0; i < cnt; ++i) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, g->g->tev[stage][2 * i], g->g->tev[stage][2 * i + 1]) == cudaSuccess) total += ms;
    }
    if (executions) *executions = cnt;
    g->g->tcount[stage] = 0;
    return total;
}

void lrb200_graph_destroy(lrb200_graph_t* g) { delete g; }

// ---- device DAG ------------------------------------------------------------------------------------------------------
lrb200_dag_t* lrb200_dag_create(void) {
    if (lrb200_device_count() <= 0) { set_error("no CUDA device available; libluaradio_b200 has no CPU fallback"); return nullptr; }
    if (ctx().device < 0 && lrb200_init(0) != 0) return nullptr;
    lrb200_dag_t* d = new (std::nothrow) lrb200_dag_s();
    if (!d) set_error("out of memory");
    return d;
}

int lrb200_dag_add_block(lrb200_dag_t* d, lrb200_block_t* q, const int* inputs, unsigned num_inputs) {
    if (!d || !q || !q->impl || (!inputs && num_inputs)) { set_error("dag_add_block: null argument"); return -1; }
    if (!q->impl->dev_ptrs) { set_error("dag_add_block: block %s was not created with LRB200_DEVICE", q->impl->name.c_str()); return -1; }
    const int id = d->d.add(q->impl, inputs, num_inputs);
    if (id < 0) return -1;
    q->impl = nullptr;          // ownership moves to the DAG
    delete q;
    return id;
}

int lrb200_dag_add_graph(lrb200_dag_t* d, lrb200_graph_t* g, int input) {
    if (!d || !g) { set_error("dag_add_graph: null argument"); return -1; }
    if (g->g->ensure_committed() != 0) return -1;
    if (g->g->stages.empty()) { set_error("dag_add_graph: empty graph"); return -1; }
    const int id = d->d.add(g->g.get(), &input, 1);
    if (id < 0) return -1;
    g->g.release();             // ownership moves to the DAG
    delete g;
    return id;
}

int lrb200_dag_set_outputs(lrb200_dag_t* d, const int* outputs, unsigned num_outputs) {
    if (!d || !outputs || !num_outputs) { set_error("dag_set_outputs: null argument"); return -1; }
    if (d->d.host.samples) { set_error("dag_set_outputs: the super-chunk slots are sized for the outputs; set them first"); return -1; }
    if (d->d.refuse_after_rewrite("set_outputs") != 0) return -1;
    std::vector<PortRef> refs(num_outputs);
    for (unsigned k = 0; k < num_outputs; ++k)
        if (d->d.decode(outputs[k], &refs[k]) != 0) { set_error("dag_set_outputs: bad reference %d", outputs[k]); return -1; }
    d->d.outputs = std::move(refs);
    d->d.sh.planned = false;
    d->d.committed = false;
    return 0;
}

int lrb200_dag_commit(lrb200_dag_t* d, int fuse) {
    if (!d) { set_error("null dag"); return -1; }
    if (d->d.nodes.empty() || d->d.outputs.empty()) { set_error("dag: no nodes / no outputs"); return -1; }
    return d->d.commit(fuse);
}

int lrb200_dag_execute(lrb200_dag_t* d, const void* x, size_t n, void* const* y, size_t* n_out) {
    if (!d || !y || !n_out || (n && !x)) { set_error("dag_execute: null argument"); return -1; }
    HostBoundary* hb = d->d.boundary();
    return hb ? hb->execute(&x, n, y, n_out) : -1;
}

int lrb200_dag_execute_device(lrb200_dag_t* d, const void* dx, size_t n, void* const* dy, size_t* n_out) {
    if (!d || !dy || !n_out || (n && !dx)) { set_error("dag_execute_device: null argument"); return -1; }
    if (d->d.host.refuse_direct("dag", "execute_device") != 0 || d->d.ensure_committed() != 0) return -1;
    return d->d.run_nodes(dx, n, dy, n_out, ctx().stream);
}

size_t lrb200_dag_max_output(const lrb200_dag_t* d, unsigned output, size_t n) {
    if (!d || output >= d->d.outputs.size()) return 0;
    // super-chunk mode: one call may hand back the results of the slots completed while n samples were appended
    return d->d.host.max_output(n);
}

int lrb200_dag_set_superchunk(lrb200_dag_t* d, size_t samples) {
    if (!d) { set_error("null dag"); return -1; }
    HostBoundary* hb = d->d.boundary();
    return hb ? hb->set_superchunk(samples, "dag") : -1;
}

int lrb200_dag_flush(lrb200_dag_t* d, void* const* y, size_t* n_out) {
    if (!d || !y || !n_out) { set_error("dag_flush: null argument"); return -1; }
    HostBoundary& hb = d->d.host;
    for (size_t k = 0; k < d->d.outputs.size(); ++k) n_out[k] = 0;
    if (!hb.samples) { set_error("dag: flush needs super-chunk mode (set_superchunk)"); return -1; }
    if (!hb.fed) { set_error("dag: nothing to flush: no execute since super-chunk mode was set, the last flush or reset"); return -1; }
    return hb.flush(y, n_out);
}

int lrb200_dag_reset(lrb200_dag_t* d) {
    if (!d) { set_error("null dag"); return -1; }
    return d->d.reset();
}

long long lrb200_dag_halo(lrb200_dag_t* d) {
    if (!d) { set_error("null dag"); return -1; }
    return d->d.halo();
}

int lrb200_dag_seek(lrb200_dag_t* d, uint64_t sample_index) {
    if (!d) { set_error("null dag"); return -1; }
    if (d->d.nodes.empty()) { set_error("dag: no nodes"); return -1; }
    return d->d.seek(sample_index);
}

size_t lrb200_dag_shard_record_bytes(lrb200_dag_t* d) { return d ? d->d.record_bytes() : 0; }

int lrb200_dag_shard_begin(lrb200_dag_t* d, const void* dx, size_t halo, size_t n, uint64_t start, void* const* dy,
                           size_t* n_out, void* record, size_t record_bytes) {
    if (!d || !dy || !n_out || (n && !dx) || (record_bytes && !record)) { set_error("dag_shard_begin: null argument"); return -1; }
    return d->d.shard_begin(dx, halo, n, start, dy, n_out, record, record_bytes);
}

int lrb200_dag_shard_accepts(lrb200_dag_t* d, const void* left_record, const void* record, size_t record_bytes) {
    if (!d || (record_bytes && (!left_record || !record))) { set_error("dag_shard_accepts: null argument"); return -1; }
    if (d->d.check_record(record_bytes) != 0) return -1;
    return d->d.shard_accepts((const PllShardRecord*)left_record, (const PllShardRecord*)record);
}

int lrb200_dag_shard_end(lrb200_dag_t* d, const void* left_records, unsigned num_left, void* const* dy, size_t* n_out,
                         void* record_out, size_t record_bytes) {
    if (!d || !dy || !n_out || (record_bytes && (!record_out || (num_left && !left_records)))) { set_error("dag_shard_end: null argument"); return -1; }
    return d->d.shard_end((const PllShardRecord*)left_records, num_left, dy, n_out, record_out, record_bytes);
}

const char* lrb200_dag_describe(const lrb200_dag_t* d) {
    if (!d) return "";
    Dag& dag = const_cast<lrb200_dag_t*>(d)->d;          // describing commits, as lrb200_graph_describe does
    if (!dag.nodes.empty() && !dag.outputs.empty() && dag.ensure_committed() != 0) return "";
    return dag.desc.c_str();
}

void lrb200_dag_destroy(lrb200_dag_t* d) { delete d; }

}  // extern "C"
