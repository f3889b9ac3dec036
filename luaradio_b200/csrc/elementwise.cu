// Element-wise / 1-sample-stencil kernels: FrequencyTranslator, FrequencyDiscriminator, Downsampler,
// ComplexMagnitude, ComplexToReal.  All are HBM-streaming kernels: 128-bit coalesced loads where the
// pointers allow, grid sized to a few waves of the SMs (132 on H100), no shared memory (no reuse to exploit).
#include "common.cuh"

namespace lrb {

namespace {

constexpr int EW_THREADS = 256;

inline int ew_grid(long long work_items) {
    long long blocks = (work_items + EW_THREADS - 1) / EW_THREADS;
    long long cap = (long long)ctx().sm_count * 16;   // grid-stride beyond ~16 CTAs/SM
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (int)blocks;
}

// frequencytranslator.lua:93-110 -- y[n] = x[n] * exp(j*omega*(g0+n)); phase from the global index.
// Each thread handles 2 consecutive samples (one 128-bit load/store) per grid-stride step.
__global__ void __launch_bounds__(EW_THREADS)
rotator_kernel(const float2* __restrict__ x, float2* __restrict__ y, long long n, uint64_t turns_fix, uint64_t g0, int vec_ok) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (vec_ok) {
        const long long npairs = n >> 1;
        const float4* x4 = reinterpret_cast<const float4*>(x);
        float4* y4 = reinterpret_cast<float4*>(y);
        for (; p < npairs; p += stride) {
            float4 v = __ldcs(x4 + p);
            uint64_t g = g0 + (uint64_t)(2 * p);
            float2 r0 = cmul(make_float2(v.x, v.y), phasor_from_fix(turns_fix * g));
            float2 r1 = cmul(make_float2(v.z, v.w), phasor_from_fix(turns_fix * (g + 1)));
            __stcs(y4 + p, make_float4(r0.x, r0.y, r1.x, r1.y));
        }
        if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) {
            long long i = n - 1;
            y[i] = cmul(x[i], phasor_from_fix(turns_fix * (g0 + (uint64_t)i)));
        }
    } else {
        for (; p < n; p += stride) y[p] = cmul(x[p], phasor_from_fix(turns_fix * (g0 + (uint64_t)p)));
    }
}

// frequencydiscriminator.lua:68-88 -- y[n] = atan2(im, re of x[n]*conj(x[n-1])) * (1/gain)
__device__ __forceinline__ float discrim_one(float2 cur, float2 prev, float inv_gain) {
    // x * conj(p) = (xr*pr + xi*pi) + j(xi*pr - xr*pi)
    float re = fmaf(cur.x, prev.x, cur.y * prev.y);
    float im = fmaf(cur.y, prev.x, -cur.x * prev.y);
    return atan2f(im, re) * inv_gain;
}

__global__ void __launch_bounds__(EW_THREADS)
discrim_kernel(const float2* __restrict__ x, const float2* __restrict__ prev, float* __restrict__ y, long long n, float inv_gain, int vec_ok) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (vec_ok) {
        // 4 samples per step: two 128-bit loads + the sample before, one 128-bit store
        const long long nquads = n >> 2;
        const float4* x4 = reinterpret_cast<const float4*>(x);
        float4* y4 = reinterpret_cast<float4*>(y);
        for (; p < nquads; p += stride) {
            float4 a = __ldg(x4 + 2 * p), b = __ldg(x4 + 2 * p + 1);
            float2 pv = (p == 0) ? __ldg(prev) : __ldg(x + 4 * p - 1);
            float4 o;
            o.x = discrim_one(make_float2(a.x, a.y), pv, inv_gain);
            o.y = discrim_one(make_float2(a.z, a.w), make_float2(a.x, a.y), inv_gain);
            o.z = discrim_one(make_float2(b.x, b.y), make_float2(a.z, a.w), inv_gain);
            o.w = discrim_one(make_float2(b.z, b.w), make_float2(b.x, b.y), inv_gain);
            __stcs(y4 + p, o);
        }
        long long i = (nquads << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x;
        if (i < n) {
            float2 pv = (i == 0) ? __ldg(prev) : __ldg(x + i - 1);
            y[i] = discrim_one(__ldg(x + i), pv, inv_gain);
        }
    } else {
        for (; p < n; p += stride) {
            float2 pv = (p == 0) ? __ldg(prev) : __ldg(x + p - 1);
            y[p] = discrim_one(__ldg(x + p), pv, inv_gain);
        }
    }
}

// downsampler.lua:45-53 -- y[j] = x[first + j*D].  The whole input stream is touched for small D
// (32-byte sectors), so this is an input-bandwidth-bound gather.
template <typename T>
__global__ void __launch_bounds__(EW_THREADS)
downsample_kernel(const T* __restrict__ x, T* __restrict__ y, long long first, long long n_out, int D) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n_out; j += stride)
        y[j] = __ldg(x + first + j * (long long)D);
}

// complexmagnitude.lua:28-36 / complexfloat32.lua:163-165: sqrt(re*re + im*im)
__global__ void __launch_bounds__(EW_THREADS)
cmag_kernel(const float2* __restrict__ x, float* __restrict__ y, long long n, int vec_ok) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (vec_ok) {
        const long long nquads = n >> 2;
        const float4* x4 = reinterpret_cast<const float4*>(x);
        float4* y4 = reinterpret_cast<float4*>(y);
        for (; p < nquads; p += stride) {
            float4 a = __ldcs(x4 + 2 * p), b = __ldcs(x4 + 2 * p + 1);
            float4 o;
            o.x = cmag_of(make_float2(a.x, a.y));
            o.y = cmag_of(make_float2(a.z, a.w));
            o.z = cmag_of(make_float2(b.x, b.y));
            o.w = cmag_of(make_float2(b.z, b.w));
            __stcs(y4 + p, o);
        }
        long long i = (nquads << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x;
        if (i < n) y[i] = cmag_of(x[i]);
    } else {
        for (; p < n; p += stride) y[p] = cmag_of(x[p]);
    }
}

// complextoreal.lua:27-35
__global__ void __launch_bounds__(EW_THREADS)
c2r_kernel(const float2* __restrict__ x, float* __restrict__ y, long long n, int vec_ok) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (vec_ok) {
        const long long nquads = n >> 2;
        const float4* x4 = reinterpret_cast<const float4*>(x);
        float4* y4 = reinterpret_cast<float4*>(y);
        for (; p < nquads; p += stride) {
            float4 a = __ldcs(x4 + 2 * p), b = __ldcs(x4 + 2 * p + 1);
            __stcs(y4 + p, make_float4(a.x, a.z, b.x, b.z));
        }
        long long i = (nquads << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x;
        if (i < n) y[i] = x[i].x;
    } else {
        for (; p < n; p += stride) y[p] = x[p].x;
    }
}

inline int aligned16(const void* a, const void* b) {
    return ((((uintptr_t)a) | ((uintptr_t)b)) & 15) == 0;
}

}  // namespace

int launch_rotator(const float2* x, float2* y, long long n, uint64_t turns_fix, uint64_t g0, cudaStream_t s) {
    if (n <= 0) return 0;
    int v = aligned16(x, y);
    rotator_kernel<<<ew_grid(v ? (n + 1) / 2 : n), EW_THREADS, 0, s>>>(x, y, n, turns_fix, g0, v);
    count_launch();
    LRB_CHECK(cudaGetLastError());
    return 0;
}

int launch_discrim(const float2* x, const float2* prev, float* y, long long n, float inv_gain, cudaStream_t s) {
    if (n <= 0) return 0;
    int v = aligned16(x, y);
    discrim_kernel<<<ew_grid(v ? (n + 3) / 4 : n), EW_THREADS, 0, s>>>(x, prev, y, n, inv_gain, v);
    count_launch();
    LRB_CHECK(cudaGetLastError());
    return 0;
}

int launch_downsample(const void* x, void* y, long long first, long long n_out, int D, int elem_size, cudaStream_t s) {
    if (n_out <= 0) return 0;
    if (elem_size == 8)
        downsample_kernel<float2><<<ew_grid(n_out), EW_THREADS, 0, s>>>((const float2*)x, (float2*)y, first, n_out, D);
    else
        downsample_kernel<float><<<ew_grid(n_out), EW_THREADS, 0, s>>>((const float*)x, (float*)y, first, n_out, D);
    count_launch();
    LRB_CHECK(cudaGetLastError());
    return 0;
}

int launch_cmag(const float2* x, float* y, long long n, cudaStream_t s) {
    if (n <= 0) return 0;
    int v = aligned16(x, y);
    cmag_kernel<<<ew_grid(v ? (n + 3) / 4 : n), EW_THREADS, 0, s>>>(x, y, n, v);
    count_launch();
    LRB_CHECK(cudaGetLastError());
    return 0;
}

int launch_c2r(const float2* x, float* y, long long n, cudaStream_t s) {
    if (n <= 0) return 0;
    int v = aligned16(x, y);
    c2r_kernel<<<ew_grid(v ? (n + 3) / 4 : n), EW_THREADS, 0, s>>>(x, y, n, v);
    count_launch();
    LRB_CHECK(cudaGetLastError());
    return 0;
}

}  // namespace lrb
