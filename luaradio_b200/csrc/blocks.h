// Block objects behind the opaque C handles (internal).
#pragma once
#include "../../include/lrb200.h"
#include "common.cuh"
#include <cmath>
#include <memory>
#include <new>
#include <vector>
#include <string>
#include <utility>

namespace lrb {

struct Block {
    std::string name;
    size_t in_size, out_size;         // element sizes in bytes
    bool dev_ptrs;                    // run on device pointers (LRB200_DEVICE); else execute stages host vectors
    uint64_t consumed = 0;            // global index of the next input sample

    Block(std::string name_, size_t in, size_t out, bool dev) : name(std::move(name_)), in_size(in), out_size(out), dev_ptrs(dev) {}
    virtual ~Block() = default;
    virtual int init() { return 0; }
    virtual size_t max_output(size_t n) const { return n; }
    int num_inputs = 1, num_outputs = 1;
    // device pointers in/out, asynchronous on s; consumes n, produces *n_out, advances the carried state
    virtual int run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) = 0;
    // blocks with several input / output ports (all inputs the same length n and element size in_size, block.lua:516-532)
    virtual int run_multi(const void* const* dx, int nin, size_t n, void* const* dy, int nout, size_t* n_out, cudaStream_t s) {
        if (nin != 1 || nout != 1) { set_error("%s has one input and one output", name.c_str()); return -1; }
        return run(dx[0], n, dy[0], n_out, s);
    }
    int execute_multi(const void* const* x, int nin, size_t n, void* const* y, int nout, size_t* n_out);
    int execute(const void* x, size_t n, void* y, size_t* n_out) { return execute_multi(&x, 1, n, &y, 1, n_out); }
    virtual size_t out_size_of(int port) const { (void)port; return out_size; }    // element size of output port `port`
    std::vector<DeviceBuffer> staging;  // host-mode staging of execute_multi: nin + nout grow-only device buffers
    // Carried state: init() declares each buffer once with carry(), which allocates it zeroed.  reset() zeroes exactly
    // the declared buffers, puts every ping-pong index back to 0 and sets consumed = 0; a graph zeroes every stage's
    // buffers with ONE kernel (a 256 Mi-sample chain step is ~1 ms: a dozen cudaMemsetAsync nodes per step were 1.5 % of
    // it).  Look-back scratch whose counters live on the host is not state and is not declared.
    std::vector<std::pair<void*, size_t>> carried;
    std::vector<int*> carried_index;
    int carry(DeviceBuffer& buf, size_t bytes);
    int carry(DeviceBuffer (&pair)[2], size_t bytes, int& cur);    // ping-pong pair, buffer `cur` is read
    void rewind();                    // the host side of reset: indices and consumed
    virtual int reset();
    virtual int seek(uint64_t idx) { consumed = idx; return 0; }
    // number of outputs this block has produced once `idx` inputs are consumed (for graph seek)
    virtual uint64_t outputs_before(uint64_t idx) const { return idx; }
    // time-chunk sharding (SURVEY.md 8e): how many INPUT samples of left context a cold start needs before this block's
    // outputs equal the streaming ones to float32 resolution (FIR history, IIR decay to 1e-12, ...); < 0 = unbounded
    virtual long long memory_in() const { return 0; }
    // output rate / input rate = up / down
    virtual void rate(unsigned* up, unsigned* down) const { *up = 1; *down = 1; }
    // sharded runs: can this block's launch keep the launches that read the first Ctx::lead_samples inputs behind
    // Ctx::lead_event while everything else starts at once?  (else the whole stream waits for the neighbour exchange)
    virtual bool supports_lead_wait() const { return false; }
    // is all carried state (history, previous output, pole state) read ONLY by launches this block puts on the side
    // stream for a long call (edge tiles, history update)?  Then a short call may run entirely on the side stream and the
    // next long call's interior kernel need not wait for it (run_shard's split of the last stage).
    virtual bool state_only_on_side_stream() const { return false; }
};

// Construct and init() a block: nullptr, with the error set, on failure
template <typename B, typename... A>
std::unique_ptr<B> make_block(A&&... args) {
    std::unique_ptr<B> b(new (std::nothrow) B(std::forward<A>(args)...));
    if (!b) { set_error("out of memory"); return nullptr; }
    if (b->init() != 0) return nullptr;
    return b;
}

// downsampler.lua:45-53 in global-index form: outputs sit at global input index == 0 (mod D)
inline void decim_plan(uint64_t consumed, unsigned D, size_t n, long long* first, long long* n_out) {
    uint64_t r = consumed % D;
    long long f = (long long)((D - r) % D);
    *first = f;
    *n_out = ((long long)n > f) ? (((long long)n - f + D - 1) / D) : 0;
}

inline long long decay_samples(double c) {        // samples until |c|^k < 1e-12; < 0 if it never gets there
    const double a = std::fabs(c);
    if (a == 0.0) return 0;
    if (a >= 1.0) return -1;
    return (long long)std::ceil(std::log(1e-12) / std::log(a)) + 1;
}

// fir_fft.cu: a FIR's overlap-save plan, made at creation (*out stays null when no overlap-save kernel covers the
// shape), and the two ways to run a call through it.  0, or -1 with the error set.
constexpr int FIR_FFT_N = 1024;
constexpr int FFT_MAX_TAPS = 513;       // L >= 512: at most half of every block is overlap
struct FirFast {
    int in_mode = 0;           // 0: complex in; 1: real in, two blocks packed per transform (rrrf); 2: Hilbert
    int M = 0, D = 1;
    int nparts = 1;            // > 1: uniformly partitioned overlap-save for filters longer than one block allows
    int part_taps = 0;         // taps per partition (M unless partitioned)
    bool rotate = false;       // a translator of rot_fix turns per sample fused in front
    uint64_t rot_fix = 0;
    DeviceBuffer d_H;          // nparts tap spectra, FIR_FFT_N each
    DeviceBuffer d_tw;
    DeviceBuffer d_E;
    int block_len() const { return FIR_FFT_N - (part_taps - 1); }     // L: outputs per block
};
int fir_fast_prepare(FirKind kind, const void* taps, int M, int D, bool rotate, uint64_t rot_fix,
                     std::unique_ptr<FirFast>* out);
int launch_overlap_save(const FirFast& f, const void* x, const void* hist, long long n, void* y, long long first,
                        uint64_t g0, cudaStream_t s);
int launch_delay_line(const FirFast& f, const void* x, const void* hist, long long n, void* y, cudaStream_t s);

struct PolyTaps;  // polyphase decimator taps (tuner.cu)

// The kernel a FirBlock call runs: register-tiled polyphase (tuner.cu), generic-shape polyphase (poly_generic.cu),
// single-block overlap-save or partitioned delay line (fir_fft.cu), catch-all direct form (fir_direct.cu)
enum class FirPath { Polyphase, PolyGeneric, OverlapSave, DelayLine, Direct };

struct FirBlock : Block {
    FirKind kind;
    int M = 0, D = 1;
    size_t tap_size = 4;
    std::vector<char> h_taps;
    DeviceBuffer d_taps;
    DeviceBuffer d_hist[2];
    int cur = 0;
    int algo = 0;                     // LRB200_FIR_AUTO / DIRECT / FFT
    bool rotate = false;              // fused FrequencyTranslator in front (graph fusion; FFT path only)
    double rot_turns = 0.0;
    uint64_t rot_fix = 0;
    // the kernels that cover this block, decided at init: overlap-save plan, polyphase taps, generic polyphase shape
    std::unique_ptr<FirFast> fast;
    PolyTaps* poly = nullptr;
    bool gen_poly = false;
    // output-rate pole fused behind a real polyphase decimator (graph rewrite of FIR -> IIR1 -> Downsampler)
    bool has_pole = false;
    float pole_c = 0.f;
    DeviceBuffer d_pole[2];
    int pcur = 0;
    int set_pole(float c);

    // rotate: a FrequencyTranslator of turns_per_sample fused in front (graph fusion)
    FirBlock(FirKind k, const void* taps_host, unsigned ntaps, unsigned decim, bool dev, bool rotate = false,
             double turns_per_sample = 0.0);
    ~FirBlock() override;
    int init() override;
    size_t max_output(size_t n) const override;
    int run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) override;
    uint64_t outputs_before(uint64_t idx) const override { return (idx + D - 1) / D; }
    long long memory_in() const override;
    void rate(unsigned* up, unsigned* down) const override { *up = 1; *down = (unsigned)D; }
    bool supports_lead_wait() const override { return always_polyphase(); }
    bool state_only_on_side_stream() const override { return always_polyphase(); }
    int set_algorithm(int a);
    FirPath path(size_t n) const;     // the kernel a call of n inputs runs
    bool always_polyphase() const { return poly != nullptr && algo != LRB200_FIR_FFT; }    // path(n) for every n
    int effective_algorithm() const;  // path() of a long call as LRB200_FIR_DIRECT / FFT (lrb200_fir_get_algorithm)
};

struct RotatorBlock : Block {
    double turns = 0;
    uint64_t turns_fix = 0;
    RotatorBlock(double turns_per_sample, bool dev);
    int run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) override;
};

struct DiscrimBlock : Block {
    float gain = 1.f;
    DeviceBuffer d_prev;
    DiscrimBlock(float gain, bool dev);
    int init() override { return carry(d_prev, sizeof(float2)); }
    int run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) override;
    long long memory_in() const override { return 1; }
};

struct DownsampleBlock : Block {
    int D = 1;
    DownsampleBlock(unsigned factor, unsigned elem, bool dev);
    size_t max_output(size_t n) const override;
    int run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) override;
    uint64_t outputs_before(uint64_t idx) const override { return (idx + D - 1) / D; }
    void rate(unsigned* up, unsigned* down) const override { *up = 1; *down = (unsigned)D; }
};

struct IirBlock : Block {
    bool complex_data = false;
    float b[9] = {0};
    int nb = 1;
    float c = 0.f;
    int D = 1;                        // fused Downsampler behind the filter (graph fusion)
    DeviceBuffer d_xhist[2];
    DeviceBuffer d_ystate[2];
    int cur = 0;
    IirScanWork work;
    IirBlock(bool cplx, const float* b, unsigned nb, const float* a, unsigned na, bool dev);
    int init() override;
    size_t max_output(size_t n) const override;
    int run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) override;
    uint64_t outputs_before(uint64_t idx) const override { return (idx + D - 1) / D; }
    long long memory_in() const override;
    void rate(unsigned* up, unsigned* down) const override { *up = 1; *down = (unsigned)D; }
};

// IIRFilterBlock of any order (na > 2): direct form I, time-parallel chunks with a measured warm-up
struct IirGeneralBlock : Block {
    bool complex_data = false;
    float b[10] = {0}, a[10] = {0};
    int nb = 1, na = 1;
    long long warm = -1;               // samples until the impulse response of 1/A(z) is below 1e-10 of its peak
    DeviceBuffer d_xhist[2];
    DeviceBuffer d_yhist[2];
    int cur = 0;
    IirGeneralBlock(bool cplx, const float* b, unsigned nb, const float* a, unsigned na, bool dev);
    int init() override;
    int run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) override;
    long long memory_in() const override { return warm < 0 ? -1 : warm + nb; }
};

// iir_order.cu: IIRFilterBlock with more than 10 taps on either side (up to 64 each): a state-space scan in double with a
// decoupled look-back over 2048-sample tiles, exact for any pole radius
constexpr int IIR_ORDER_MAX_TAPS = 64;
constexpr int IIR_ORDER_MAX_TILES = 1 << 17;        // 2048-sample tiles per launch (256 Mi samples)
struct IirOrderBlock : Block {
    bool complex_data = false;
    int nb = 1, q = 0;                                // feed-forward taps, feedback order na - 1
    std::vector<double> b, cdiv;                      // b[j] / a0;  cdiv[j] = -a[j] / a0 (j >= 1)
    long long decay = -1;                             // samples until the impulse response of 1/A(z) is below 1e-10 of its peak
    DeviceBuffer d_xhist[2];                          // last nb - 1 inputs (exact in the input type), oldest first
    DeviceBuffer d_ystate[2];                         // last q outputs in double, most recent first
    int cur = 0;
    DeviceBuffer d_mats, d_hom;                       // M^V, M^(T e) for e < look-back window; homogeneous response table
    // look-back scratch, not state (as LevelBlock): tickets count up from ticket_base, records are tagged with epoch
    DeviceBuffer d_ticket, d_flags, d_agg, d_pfx;
    unsigned long long ticket_base = 0;
    unsigned epoch = 0;
    IirOrderBlock(bool cplx, const float* b, unsigned nb, const float* a, unsigned na, bool dev);
    int init() override;
    int run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) override;
    long long memory_in() const override { return decay; }
};

struct C2fBlock : Block {
    int op = 0;                       // 0 = magnitude, 1 = real part
    C2fBlock(int op, bool dev);
    int run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) override;
};

// resample.cu ---------------------------------------------------------------------------------
struct ScaleBlock : Block {           // MultiplyConstantBlock
    float cre, cim;
    bool complex_data, complex_const;
    ScaleBlock(float re, float im, bool cdata, bool cconst, bool dev);
    int run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) override;
};

struct UpsampleBlock : Block {        // UpsamplerBlock
    int L = 1;
    UpsampleBlock(unsigned factor, unsigned elem, bool dev);
    size_t max_output(size_t n) const override { return n * (size_t)L; }
    uint64_t outputs_before(uint64_t idx) const override { return idx * (uint64_t)L; }
    void rate(unsigned* up, unsigned* down) const override { *up = (unsigned)L; *down = 1; }
    int run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) override;
};

struct InterpFirBlock : Block {       // [MultiplyConstant ->] Upsampler -> FIR(real taps) [-> Downsampler], fused
    bool complex_data;
    int L, D, M, Hn = 0, cur = 0;
    bool has_scale;
    float scale;
    std::vector<float> h_taps;
    DeviceBuffer d_taps;
    DeviceBuffer d_taps_tp;              // [t][phase] layout for the register-tiled interpolator (D == 1, L <= 8)
    int Tt = 0;
    bool rs_ok = false;                  // the register-tiled (L, D) polyphase kernel covers this shape (resample.cu)
    DeviceBuffer d_hist[2];
    InterpFirBlock(bool cdata, const float* taps_host, int ntaps, int interp, int decim, bool has_scale, float scale, bool dev);
    int init() override;
    size_t max_output(size_t n) const override;
    uint64_t outputs_before(uint64_t idx) const override;
    int run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) override;
    long long memory_in() const override { return Hn + 1; }
    void rate(unsigned* up, unsigned* down) const override { *up = (unsigned)L; *down = (unsigned)D; }
};

// level.cu: AGCBlock (agc = true) and PowerSquelchBlock, one block-parallel scan kernel per call
constexpr int LEVEL_MAX_TILES = 1 << 17;   // 2048-sample tiles per launch (256 Mi samples)
struct LevelBlock : Block {
    bool agc = false, complex_data = false;
    double pa = 0, ga = 0, T = 0, theta = 0;  // power / gain alphas, linear target and threshold
    DeviceBuffer d_state[2];                  // (P, g) after the last sample, ping-ponged per launch
    int cur = 0;
    DeviceBuffer d_pw;                        // (1-ga)^k, k <= one tile
    // look-back scratch, not state: the tickets count up across launches from ticket_base and the records are tagged
    // with epoch, both kept on the host and never reset (zeroing d_ticket alone would leave tiles waiting for ever)
    DeviceBuffer d_ticket;                    // tile tickets
    unsigned long long ticket_base = 0;
    DeviceBuffer d_rec;                       // per-tile look-back records, 16 bytes per tile and stage
    size_t rec_bytes() const { return (size_t)16 * (agc ? 2 : 1) * LEVEL_MAX_TILES; }
    unsigned epoch = 0;
    LevelBlock(bool agc, double power_alpha, double gain_alpha, double target, double threshold, bool cplx, bool dev);
    int init() override;
    int run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) override;
    long long memory_in() const override;
};

// phasecorr.cu: BinaryPhaseCorrectorBlock, a reduce / scan / apply over 2048-sample tiles (three launches per call)
constexpr int PC_MAX_TILES = 1 << 17;      // 2048-sample tiles per launch (256 Mi samples)
struct PhaseCorrectorBlock : Block {
    unsigned N = 1, I = 1;                  // num_samples, sample_interval
    DeviceBuffer d_state[2];                // {average (double), window[N] (float32, slot = measurement number mod N)}
    int cur = 0;
    DeviceBuffer d_tiles;                   // scratch: per-tile term sums and starting averages
    PhaseCorrectorBlock(unsigned num_samples, unsigned sample_interval, bool dev);
    int init() override;
    int run(const void* dx, size_t n, void* dy, size_t* n_out, cudaStream_t s) override;
    long long memory_in() const override;
};

// psd_long.cu: the PSD transform of frames of 8192 <= N <= 2^20 points (power of two) for PsdBlock
constexpr int PSD_LONG_MIN = 8192, PSD_LONG_MAX = 1 << 20;
constexpr int PSD_LONG_SINGLE_MAX = 16384;           // one CTA per frame up to here, two passes through scratch above
constexpr long long PSD_LONG_BATCH = 1LL << 25;      // samples per two-pass batch: 256 MiB of complex64 scratch
struct PsdLong {
    int N = 0;
    DeviceBuffer d_tw;                               // twiddle tables (psd_long.cu)
    DeviceBuffer d_scratch;                          // two-pass form: the column pass's output
    int init(int N);
    int run(const void* x, const float* window, float* y, long long frames, bool cplx, double inv_scale, bool logarithmic,
            cudaStream_t s);
};

}  // namespace lrb

// the opaque public handle
struct lrb200_block_s { lrb::Block* impl; };

namespace lrb {
// a new C handle owning b; nullptr when b is (the error is set)
inline lrb200_block_s* block_handle(std::unique_ptr<Block> b) {
    if (!b) return nullptr;
    lrb200_block_s* h = new (std::nothrow) lrb200_block_s{b.get()};
    if (!h) { set_error("out of memory"); return nullptr; }
    b.release();
    return h;
}
// the lrb200_*_create tail: block B from args and the LRB200_DEVICE bit of flags, behind a new handle
template <typename B, typename... A>
lrb200_block_s* create_block(unsigned flags, A&&... args) {
    return block_handle(make_block<B>(std::forward<A>(args)..., (flags & LRB200_DEVICE) != 0));
}

// tuner.cu: register-tiled polyphase decimating FIR with real taps.  polyphase_prepare returns nullptr when no kernel
// is instantiated for the shape: complex data, for the TunerBlock's fused translator of turns_per_sample if
// `translator`, or a float32 stream if `real_data`.
PolyTaps* polyphase_prepare(const float* taps, int M, int D, double turns_per_sample, bool translator = false,
                            bool real_data = false);
void polyphase_release(PolyTaps* p);
// FirBlock's kernel for taps prepared without a translator: x / hist / y are float2, or float32 for real_data.  A real
// decimator with pole_in != nullptr additionally fuses the output-rate pole z[m] = pole_c z[m-1] + w[m], its state
// z[-1] read from pole_in and the last z written to pole_out.  0, or -1 with the error set.
int launch_polyphase(const PolyTaps* p, const void* x, const void* hist, long long n, void* y, long long first,
                     long long n_out, cudaStream_t s, float pole_c = 0.f, const float* pole_in = nullptr,
                     float* pole_out = nullptr);
bool polyphase_pole_ok(float c);     // the pole's memory fits the kernel's warm-up
// tuner.cu: fused FrequencyTranslator -> FIR(crcf) -> Downsampler; returns nullptr (with the error set) on failure
// iqconv.cu: IQFileSource sample format -> ComplexFloat32 (nullptr + error for an unknown format)
std::unique_ptr<Block> make_iqconv(const char* format, bool dev);
// RealFileSource (to_file = false, comps = 1), RealFileSink/WAVFileSink (true, 1), IQFileSink (true, 2)
std::unique_ptr<Block> make_fileconv(const char* format, bool to_file, int comps, bool dev);
// disc_gain != 0 additionally fuses a FrequencyDiscriminator(gain) behind it (float output)
std::unique_ptr<Block> make_tuner(double turns_per_sample, const float* taps, int ntaps, int decim, float disc_gain);
}  // namespace lrb
