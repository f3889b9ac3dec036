// Internal declarations shared by the kernels and the C ABI (not installed; the public surface is
// include/lrb200.h).  All launchers are asynchronous on the given stream.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <atomic>
#include <math.h>

namespace lrb {

#define LRB_MAX_DEVICES 16        // per-device "function attributes set" flags (power of two)

struct Ctx {
    int device = -1;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    std::atomic<uint64_t> launches{0};
    // persistent kernels leave this many CTA slots free while the first stage of a sharded run keeps its edge tiles waiting
    // for the neighbour's halo on the side stream (graph.cu: run_shard) -- otherwise those few tiles only get an SM once
    // the persistent grid drains
    int reserve_ctas = 0;
    // time-chunk sharding: the first `lead_samples` input samples of the launch in flight come from the left neighbour and
    // are only valid after `lead_event`; the polyphase launcher keeps every tile that touches them out of the interior
    // kernel and makes its edge launch (side stream) wait for the event -- so only those few tiles wait for the exchange
    long long lead_samples = 0;
    cudaEvent_t lead_event = nullptr;
    // side stream for the few-CTA edge kernels, so they overlap the interior kernel instead of trailing it
    cudaStream_t side = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
};
Ctx& ctx();
void set_error(const char* fmt, ...);
bool cuda_ok(cudaError_t e, const char* what);

#define LRB_CHECK(call)                                   \
    do {                                                  \
        if (!::lrb::cuda_ok((call), #call)) return -1;    \
    } while (0)

// One cudaMalloc region, freed with the object.  The int-returning members follow LRB_CHECK: 0, or -1 with the error set.
class DeviceBuffer {
public:
    DeviceBuffer() = default;
    DeviceBuffer(const DeviceBuffer&) = delete;
    DeviceBuffer& operator=(const DeviceBuffer&) = delete;
    DeviceBuffer(DeviceBuffer&& o) noexcept : p_(o.p_), cap_(o.cap_) { o.p_ = nullptr; o.cap_ = 0; }
    DeviceBuffer& operator=(DeviceBuffer&& o) noexcept {
        if (this != &o) { cudaFree(p_); p_ = o.p_; cap_ = o.cap_; o.p_ = nullptr; o.cap_ = 0; }
        return *this;
    }
    ~DeviceBuffer() { cudaFree(p_); }
    void* get() const { return p_; }
    template <typename T> T* as() const { return static_cast<T*>(p_); }
    size_t capacity() const { return cap_; }
    // grow-only (like Vector:resize): a larger request drops the contents and allocates anew
    int reserve(size_t bytes) {
        if (bytes <= cap_) return 0;
        cudaFree(p_);
        p_ = nullptr;
        cap_ = 0;
        LRB_CHECK(cudaMalloc(&p_, bytes));
        cap_ = bytes;
        return 0;
    }
    int alloc_zeroed(size_t bytes) {
        if (reserve(bytes) != 0) return -1;
        LRB_CHECK(cudaMemset(p_, 0, bytes));
        return 0;
    }
    int upload(const void* host, size_t bytes) {
        if (reserve(bytes) != 0) return -1;
        LRB_CHECK(cudaMemcpy(p_, host, bytes, cudaMemcpyHostToDevice));
        return 0;
    }

private:
    void* p_ = nullptr;
    size_t cap_ = 0;
};

// cycles-per-sample (any sign / magnitude) -> fraction of a turn in 2^-64 units.  Done in 80-bit long double
// so that removing the integer part does not round the 53-bit fraction (a 2^-54 error per sample is
// 3e-6 rad after 2^33 samples).
inline uint64_t turns_to_fix(double turns) {
    long double t = (long double)turns;
    t -= floorl(t);                         // [0,1), exact
    long double f = ldexpl(t, 64);
    if (f >= 18446744073709551616.0L) return 0;
    return (uint64_t)f;
}

// fork: returns a stream that has waited for everything enqueued on `s` so far (or `s` itself if unavailable);
// join: makes `s` wait for the side stream.  Used as  side = side_fork(s); edge<<<..., side>>>; main<<<..., s>>>; side_join(s).
constexpr size_t SIDE_STREAM_MIN = (size_t)1 << 18;   // below this many samples the few-CTA kernels stay on the main stream
cudaStream_t side_fork(cudaStream_t s);
void side_join(cudaStream_t s, cudaStream_t side);

inline void count_launch(int n = 1) { ctx().launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

enum FirKind { FIR_CRCF = 0, FIR_CCCF = 1, FIR_RRRF = 2, FIR_HILBERT = 3 };

// ---- fir_direct.cu ----------------------------------------------------------------------------
// Generic direct form: any ntaps, any decimation.  Logical input index i in [-(M-1), n): i < 0
// reads hist[M-1+i].  Output j (0 <= j < n_out) is the filter output at input index first + j*D.
int launch_fir_generic(FirKind kind, const void* x, const void* hist, const void* taps, int M, int D,
                       long long first, long long n_out, void* y, cudaStream_t s);
// new_hist[j] = logical(n - H + j), j in [0,H), over the concatenation [old_hist | x].
int launch_hist_update(const void* x, long long n, const void* hist_old, void* hist_new, int H,
                       int elem_size, cudaStream_t s);

// ---- poly_generic.cu --------------------------------------------------------------------------
// register-tiled polyphase decimating FIR for any covered (kind, M, D); taps_host in natural order
bool poly_generic_supports(FirKind kind, int M, int D);
int launch_poly_generic(FirKind kind, const void* x, const void* hist, const void* taps_host, int M, int D,
                        long long first, long long n, long long n_out, void* y, cudaStream_t s);

// ---- elementwise.cu ---------------------------------------------------------------------------
int launch_rotator(const float2* x, float2* y, long long n, uint64_t turns_fix, uint64_t g0, cudaStream_t s);
int launch_discrim(const float2* x, const float2* prev, float* y, long long n, float inv_gain, cudaStream_t s);
int launch_downsample(const void* x, void* y, long long first, long long n_out, int D, int elem_size, cudaStream_t s);
int launch_cmag(const float2* x, float* y, long long n, cudaStream_t s);
int launch_c2r(const float2* x, float* y, long long n, cudaStream_t s);
int launch_copy_last(const void* x, long long n, void* dst, int elem_size, cudaStream_t s);
// zero up to 32 small device buffers with one launch (graph reset)
int launch_zero_segments(void* const* ptrs, const size_t* bytes, int count, cudaStream_t s);

// ---- iir.cu -----------------------------------------------------------------------------------
// y[n] = sum_{j<nb} b[j] x[n-j] + c*y[n-1]   (c = -a1/a0, b already divided by a0)
// xhist: nb-1 previous inputs (oldest first), ystate: previous output.  State buffers are
// ping-ponged by the caller: *_in is read, *_out written.  Fused decimation: only outputs whose
// index (first + j*D) are written when D > 1.
struct IirScanWork {           // device-side scratch for the decoupled look-back
    DeviceBuffer ticket;       // 1 int
    DeviceBuffer flags;        // max_tiles ints
    DeviceBuffer agg;          // max_tiles elements
    DeviceBuffer pfx;          // max_tiles elements
    int max_tiles = 0;
    unsigned epoch = 0;
};
int iir_work_alloc(IirScanWork* w, int elem_size);
long long iir_max_per_launch(const IirScanWork& w);
int launch_iir1(bool complex_data, const void* x, long long n, void* y, const float* b_host, int nb, float c,
                const void* xhist_in, void* xhist_out, const void* ystate_in, void* ystate_out,
                long long first, int D, IirScanWork* w, cudaStream_t s);

// general order (direct form I), time-parallel with a warm-up of `warm` samples (< 0: unknown -> sequential)
int launch_iir_general(bool complex_data, const void* x, long long n, void* y, const float* b, int nb, const float* a, int na,
                       const void* xhist, const void* yhist, long long warm, cudaStream_t s);

// ---- synth.cu ---------------------------------------------------------------------------------
int launch_synth_white(float2* dst, uint64_t n0, long long n, uint32_t seed, cudaStream_t s);
int launch_synth_fm(float2* dst, uint64_t n0, long long n, uint32_t seed, double rate, double carrier,
                    double deviation, float amp, float noise, cudaStream_t s);

// ---- device helpers ---------------------------------------------------------------------------
#ifdef __CUDACC__
// Two-lane float2 multiply-add / multiply.  sm_90 has no packed FP32 FMA: each lane is one FFMA (FMUL), written with the
// explicit round-to-nearest intrinsics so that the compiler neither contracts nor reassociates them.
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fsub2(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
// |v| as ComplexMagnitudeBlock computes it (complexmagnitude.lua:28-36): sqrt(re*re + im*im), one FMA, correctly rounded
// square root.  The magnitude kernel and the overlap-save FIR's magnitude prologue both use it, so they agree bit for bit.
__device__ __forceinline__ float cmag_of(float2 v) { return __fsqrt_rn(__fmaf_rn(v.x, v.x, __fmul_rn(v.y, v.y))); }
// exp(j*2*pi*turns) for turns given as a 64-bit fixed-point fraction of a cycle.
__device__ __forceinline__ float2 phasor_from_fix(uint64_t ph) {
    // top 32 bits as a signed fraction of a half-turn: t in [-1, 1)
    int t = (int)(uint32_t)(ph >> 32);
    float half_turns = (float)t * 4.656612873077393e-10f;  // 2^-31
    float s, c;
    sincospif(half_turns, &s, &c);
    return make_float2(c, s);
}
// atan2 for the fused discriminator epilogue: one fast division, a degree-8 polynomial in a^2 on [0, 1]
// (max abs error 1.1e-7 rad, fitted and checked in float32) and three selects -- a few dozen instructions instead
// of the ~110 of atan2f, whose 8 calls per thread made up a third of the tuner kernel's instruction stream.
__device__ __forceinline__ float fast_atan2f(float y, float x) {
    const float ax = fabsf(x), ay = fabsf(y);
    const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
    const float a = mx > 0.f ? __fdividef(mn, mx) : 0.f;
    const float z = a * a;
    float r = 0.0028340641874819994f;
    r = fmaf(r, z, -0.016005029901862144f);
    r = fmaf(r, z, 0.042587608098983765f);
    r = fmaf(r, z, -0.07495445758104324f);
    r = fmaf(r, z, 0.10636754333972931f);
    r = fmaf(r, z, -0.14202570915222168f);
    r = fmaf(r, z, 0.19992484152317047f);
    r = fmaf(r, z, -0.3333306610584259f);
    r = fmaf(r, z, 1.0f);
    r *= a;
    r = ay > ax ? 1.57079632679489662f - r : r;
    r = x < 0.f ? 3.14159265358979324f - r : r;
    return copysignf(r, y);
}
// Two atan2 at once on the lanes of a float2 (y = (y0, y1), x = (x0, x1)), the two polynomial chains interleaved for ILP.
__device__ __forceinline__ float2 fast_atan2f_x2(float2 y, float2 x) {
    const float ax0 = fabsf(x.x), ay0 = fabsf(y.x), ax1 = fabsf(x.y), ay1 = fabsf(y.y);
    const float mx0 = fmaxf(ax0, ay0), mn0 = fminf(ax0, ay0), mx1 = fmaxf(ax1, ay1), mn1 = fminf(ax1, ay1);
    const float2 a = make_float2(mx0 > 0.f ? __fdividef(mn0, mx0) : 0.f, mx1 > 0.f ? __fdividef(mn1, mx1) : 0.f);
    const float2 z = fmul2(a, a);
    float2 r = make_float2(0.0028340641874819994f, 0.0028340641874819994f);
    r = ffma2(r, z, make_float2(-0.016005029901862144f, -0.016005029901862144f));
    r = ffma2(r, z, make_float2(0.042587608098983765f, 0.042587608098983765f));
    r = ffma2(r, z, make_float2(-0.07495445758104324f, -0.07495445758104324f));
    r = ffma2(r, z, make_float2(0.10636754333972931f, 0.10636754333972931f));
    r = ffma2(r, z, make_float2(-0.14202570915222168f, -0.14202570915222168f));
    r = ffma2(r, z, make_float2(0.19992484152317047f, 0.19992484152317047f));
    r = ffma2(r, z, make_float2(-0.3333306610584259f, -0.3333306610584259f));
    r = ffma2(r, z, make_float2(1.0f, 1.0f));
    r = fmul2(r, a);
    float r0 = ay0 > ax0 ? 1.57079632679489662f - r.x : r.x;
    float r1 = ay1 > ax1 ? 1.57079632679489662f - r.y : r.y;
    r0 = x.x < 0.f ? 3.14159265358979324f - r0 : r0;
    r1 = x.y < 0.f ? 3.14159265358979324f - r1 : r1;
    return make_float2(copysignf(r0, y.x), copysignf(r1, y.y));
}
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
    // (a.x + j a.y)(b.x + j b.y): two FMUL + two FFMA
    float2 t = fmul2(make_float2(-a.y, a.x), make_float2(b.y, b.y));
    return ffma2(a, make_float2(b.x, b.x), t);
}
#endif

}  // namespace lrb
