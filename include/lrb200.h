/*
 * lrb200.h -- C ABI of libluaradio_b200.so: the H100 (sm_90a) implementation of LuaRadio's
 * per-block sample-stream DSP hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  Every entry point replaces one FFI
 * binding (or pure-Lua loop) of the reference, cited as `file:line` relative to the reference
 * root (vsergeev/luaradio v0.11.0).  The conventions are the ones the reference's own FFI
 * bindings use (liquid-dsp style, radio/blocks/signal/firfilter.lua:167-226):
 *
 *   - plain C: `extern "C"`, pointers and sizes only, no C++/torch types, no exceptions;
 *   - sample types are binary-compatible with radio/types/complexfloat32.lua:19-24 and
 *     radio/types/float32.lua:17-21 (interleaved I/Q float32 == CUDA float2; float32);
 *   - stateful objects are an opaque handle with a  create / execute / reset / destroy  quartet;
 *     create returns NULL on failure (the Lua wrapper raises error(), firfilter.lua:199-201);
 *   - the CALLER owns every sample buffer; the library owns only its opaque state;
 *   - execute consumes exactly n input samples (any n >= 0, including 1: tests/jigs.lua:226-243),
 *     writes *n_out output samples and carries the block's streaming state (FIR history,
 *     translator phase, discriminator previous sample, IIR state, downsampler index) to the
 *     next call, exactly as the reference's process() does;
 *   - execute returns 0 on success, <0 on failure with a message in lrb200_last_error();
 *   - handles are not thread-safe (the reference runs one single-threaded process per block,
 *     radio/core/composite.lua:568-636); different handles may be used from different threads.
 *
 * Pointer mode is fixed per handle at create time by `flags`:
 *   LRB200_HOST    x / y are HOST pointers (pageable or pinned): drop-in mode, the call stages
 *                  host->device, runs the kernels, copies device->host and synchronises.
 *   LRB200_DEVICE  x / y are DEVICE pointers: the call only enqueues kernels on the library
 *                  stream (lrb200_set_stream / lrb200_sync) -- graph mode, used when connected
 *                  GPU blocks share device-resident buffers (lrb200_graph_*).
 *                  The pointers reach the kernels as given (so do dx / dy of
 *                  lrb200_graph_execute_device).  They need only the natural alignment of their
 *                  element: 4 bytes for float32, 8 for complex, a component's width for the raw
 *                  file formats (a 16-byte aligned pointer may select faster kernels, never other
 *                  results beyond float32 rounding).  A call reads no byte outside [x, x + n
 *                  samples) and writes no byte outside [y, y + *n_out samples); the buffers may
 *                  sit inside larger allocations next to live data (tests/test_gpu_bounds.py).
 *
 * There is NO CPU fallback anywhere in this library: without a CUDA device every create fails.
 */
#ifndef LRB200_H
#define LRB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* radio/types/complexfloat32.lua:19-24, radio/types/float32.lua:17-21 */
typedef struct { float real; float imag; } complex_float32_t;
typedef struct { float value; } float32_t;

#define LRB200_HOST   0u
#define LRB200_DEVICE 1u

/* ---- library / device ---------------------------------------------------------------------
 * Replaces the feature probe + ffi.load in radio/core/platform.lua:277-299 (platform.features.X,
 * platform.libs.X).  lrb200_init is lazy-safe: create functions call it with the current device. */
int         lrb200_init(int device);                 /* 0 ok, <0 error (no device, wrong arch)   */
int         lrb200_device_count(void);               /* 0 when no CUDA device is usable          */
int         lrb200_current_device(void);             /* device of the last successful lrb200_init, -1 before */
const char* lrb200_last_error(void);                 /* thread-local, never NULL                 */
const char* lrb200_version(void);
int         lrb200_set_stream(void* cuda_stream);    /* use the caller's cudaStream_t (NULL = own) */
void*       lrb200_get_stream(void);
int         lrb200_sync(void);                       /* cudaStreamSynchronize on the library stream */
uint64_t    lrb200_launch_count(void);               /* kernels launched by this library so far  */

/* device / pinned memory for graph mode and source/sink boundaries (the reference's
 * platform.alloc, radio/core/platform.lua:268-274, is the host analogue) */
void* lrb200_malloc(size_t bytes);
void  lrb200_free(void* dptr);
void* lrb200_host_alloc(size_t bytes);               /* pinned */
void  lrb200_host_free(void* hptr);
int   lrb200_memcpy_h2d(void* dst, const void* src, size_t bytes);   /* async on the library stream */
int   lrb200_memcpy_d2h(void* dst, const void* src, size_t bytes);   /* async on the library stream */
int   lrb200_memset(void* dptr, int value, size_t bytes);
/* peer access between the per-GPU processes of a sharded stream (lrb200_graph_execute_shard): export a 64-byte handle of
 * an lrb200_malloc allocation, import it in the neighbour process, and let the copy engine move the halo over NVLink
 * (lrb200_memcpy_d2d on `cuda_stream`, NULL = the library stream) -- no SM and no collective kernel involved. */
int   lrb200_ipc_export(void* dptr, void* handle_out64);
void* lrb200_ipc_import(const void* handle64);
int   lrb200_ipc_close(void* imported);
int   lrb200_memcpy_d2d(void* dst, const void* src, size_t bytes, void* cuda_stream);

/* ---- generic block handle ------------------------------------------------------------------
 * Every block below is an lrb200_block_t; the typed names are aliases so the Lua cdef reads like
 * the liquid bindings it sits beside.  lrb200_block_execute is what Block:process() calls
 * (radio/core/block.lua:585). */
typedef struct lrb200_block_s lrb200_block_t;

int    lrb200_block_execute(lrb200_block_t* q, const void* x, size_t n, void* y, size_t* n_out);
/* blocks with several ports (block.lua:516-532 hands process() one vector per input, all of the same length n):
 * x[i] / y[o] are the port buffers, in the handle's pointer mode */
int    lrb200_block_execute_multi(lrb200_block_t* q, const void* const* x, unsigned num_inputs, size_t n, void* const* y,
                                  unsigned num_outputs, size_t* n_out);
unsigned lrb200_block_num_inputs(const lrb200_block_t* q);
unsigned lrb200_block_num_outputs(const lrb200_block_t* q);
size_t lrb200_block_max_output(const lrb200_block_t* q, size_t n); /* upper bound on *n_out for n inputs */
size_t lrb200_block_in_size(const lrb200_block_t* q);              /* bytes per input sample  */
size_t lrb200_block_out_size(const lrb200_block_t* q);             /* bytes per output sample */
int    lrb200_block_reset(lrb200_block_t* q);                      /* back to the state after create */
int    lrb200_block_seek(lrb200_block_t* q, uint64_t sample_index); /* set the global input sample index
                                                                       (translator phase, decimation phase)
                                                                       for time-chunk sharding */
void   lrb200_block_destroy(lrb200_block_t* q);
const char* lrb200_block_name(const lrb200_block_t* q);

/* ---- FIRFilterBlock (+ Lowpass/Highpass/Bandpass/Bandstop/ComplexBandpass/ComplexBandstop) ---
 * Replaces: volk_32fc_32f_dot_prod_32fc / volk_32fc_x2_dot_prod_32fc / volk_32f_x2_dot_prod_32f
 * called once per output sample (firfilter.lua:111-163), firfilt_{crcf,cccf,rrrf}_create /
 * _execute_block (firfilter.lua:167-226), the pure-Lua loops (:244-305) and the FFTW/VOLK
 * overlap-save path process_fft (:320-398).
 *   y[n] = sum_{k<ntaps} taps[k] * x[n-k], zero initial history, history carried across calls.
 * `taps` are in natural order (NOT reversed).  decim >= 1 fuses a DownsamplerBlock(decim)
 * (downsampler.lua:40-56) behind the filter: only outputs at global input index == 0 mod decim
 * are computed and written (this is what Tuner/Decimator need, composites/decimator.lua:34-41).
 * Unlike process_fft the output is length-preserving with zero latency (n_out == n for decim 1),
 * i.e. the dot-product semantics, whichever algorithm runs inside (SURVEY.md 7f). */
typedef lrb200_block_t lrb200_fir_t;
lrb200_fir_t* lrb200_fir_create_crcf(const float32_t* taps, unsigned ntaps, unsigned decim, unsigned flags);         /* complex in, real taps    */
lrb200_fir_t* lrb200_fir_create_cccf(const complex_float32_t* taps, unsigned ntaps, unsigned decim, unsigned flags); /* complex in, complex taps */
lrb200_fir_t* lrb200_fir_create_rrrf(const float32_t* taps, unsigned ntaps, unsigned decim, unsigned flags);         /* real in, real taps       */
int  lrb200_fir_execute(lrb200_fir_t* q, const void* x, size_t n, void* y, size_t* n_out);
int  lrb200_fir_reset(lrb200_fir_t* q);
void lrb200_fir_destroy(lrb200_fir_t* q);
/* algorithm selection (FIRFilterBlock(taps, use_fft), firfilter.lua:43,55-62):
 * 0 = automatic, 1 = force direct form, 2 = force fused overlap-save FFT */
#define LRB200_FIR_AUTO   0
#define LRB200_FIR_DIRECT 1
#define LRB200_FIR_FFT    2
int  lrb200_fir_set_algorithm(lrb200_fir_t* q, int algo);
int  lrb200_fir_get_algorithm(const lrb200_fir_t* q);   /* the algorithm that will run (1 or 2) */

/* ---- HilbertTransformBlock -------------------------------------------------------------------
 * Replaces volk_32f_x2_dot_prod_32f / dotprod_rrrf_execute per sample (hilberttransform.lua:39-128)
 * and the Lua loop (:132-167): out.real = x[n-(ntaps-1)/2], out.imag = sum_k taps[k] x[n-k].
 * float32 in -> complex out; ntaps must be odd. */
typedef lrb200_block_t lrb200_hilbert_t;
lrb200_hilbert_t* lrb200_hilbert_create(const float32_t* taps, unsigned ntaps, unsigned flags);

/* ---- FrequencyTranslatorBlock ---------------------------------------------------------------
 * Replaces volk_32fc_s32fc_x2_rotator_32fc (frequencytranslator.lua:26-53), nco_crcf_mix_block_up
 * (:55-89) and the Lua loop (:93-110): y[n] = x[n] * exp(j*omega*n_global).
 * `turns_per_sample` = offset/rate (cycles per sample, any sign); the phase is the closed form of
 * the global sample index in 64-bit fixed point, so it never drifts and any chunk can be
 * processed independently (lrb200_block_seek). */
typedef lrb200_block_t lrb200_rotator_t;
lrb200_rotator_t* lrb200_rotator_create(double turns_per_sample, unsigned flags);

/* ---- FrequencyDiscriminatorBlock -------------------------------------------------------------
 * Replaces volk_32fc_x2_multiply_conjugate_32fc + volk_32fc_s32f_atan2_32f_a
 * (frequencydiscriminator.lua:40-64) and the Lua loop (:68-88):
 * y[n] = atan2(im, re of x[n]*conj(x[n-1])) / gain, gain = 2*pi*modulation_index; prev sample carried. */
typedef lrb200_block_t lrb200_discrim_t;
lrb200_discrim_t* lrb200_discrim_create(float gain, unsigned flags);

/* ---- DownsamplerBlock -------------------------------------------------------------------------
 * Replaces the LuaJIT gather loop (downsampler.lua:40-56): y[m] = x[index + m*factor], index carried.
 * elem_size is 8 (complex) or 4 (float32). */
typedef lrb200_block_t lrb200_downsample_t;
lrb200_downsample_t* lrb200_downsample_create(unsigned factor, unsigned elem_size, unsigned flags);

/* ---- IIRFilterBlock / SinglepoleLowpass / SinglepoleHighpass / FMDeemphasisFilterBlock --------
 * Replaces iirfilt_{rrrf,crcf}_create/_execute_block (iirfilter.lua:63-109) and the Lua recurrence
 * (:113-179): y[n] = (sum_j b[j] x[n-j] - sum_{j>=1} a[j] y[n-j]) / a[0], zero initial state.
 * Single pole (na <= 2): block-parallel affine scan (decoupled look-back, or a warm-up restart when the pole's
 * memory is shorter than 512 samples).  Higher orders (na, nb <= 10): direct form I in time-parallel chunks
 * with a warm-up measured from the filter's impulse response; short calls are the plain sequential recurrence.
 * Longer filters (nb or na in 11..64): state-space scan in double with a decoupled look-back, exact up to rounding for
 * any pole radius.  More than 64 taps on either side, or a[0] == 0, is refused. */
typedef lrb200_block_t lrb200_iir_t;
lrb200_iir_t* lrb200_iir_create_rrrf(const float32_t* b, unsigned nb, const float32_t* a, unsigned na, unsigned flags);
lrb200_iir_t* lrb200_iir_create_crcf(const float32_t* b, unsigned nb, const float32_t* a, unsigned na, unsigned flags);

/* ---- ComplexMagnitudeBlock / ComplexToRealBlock -----------------------------------------------
 * Replace the LuaJIT loops complexmagnitude.lua:28-36 (sqrt(re^2+im^2)) and complextoreal.lua:27-35. */
lrb200_block_t* lrb200_cmag_create(unsigned flags);
lrb200_block_t* lrb200_c2r_create(unsigned flags);

/* ---- Resampling family (SURVEY.md 8f row 4) ------------------------------------------------------------
 * lrb200_mulconst_create replaces MultiplyConstantBlock:process (radio/blocks/signal/multiplyconstant.lua: complex x
 * complex, complex x real, real x real); lrb200_upsample_create replaces UpsamplerBlock:process
 * (radio/blocks/signal/upsampler.lua:44-52: y[i*L] = x[i], zeros in between; output length n*L).  In a graph,
 * [mulconst(real c) ->] upsample(L) -> fir(real taps) [-> downsample(D)] -- InterpolatorBlock
 * (radio/composites/interpolator.lua:31-41) and RationalResamplerBlock (radio/composites/rationalresampler.lua:33-46)
 * -- commit to ONE polyphase kernel that touches only the non-zero products of kept outputs. */
lrb200_block_t* lrb200_mulconst_create(float re, float im, unsigned complex_data, unsigned complex_constant, unsigned flags);
lrb200_block_t* lrb200_upsample_create(unsigned factor, unsigned elem_size, unsigned flags);

/* ---- Two-input element-wise blocks, DelayBlock, PSD (SURVEY.md 8f rows 3 and 4) -------------------------------------
 * lrb200_binary_create replaces MultiplyBlock / MultiplyConjugateBlock / AddBlock / SubtractBlock:process
 * (radio/blocks/signal/multiply.lua, multiplyconjugate.lua:26-51, add.lua, subtract.lua; VOLK or Lua loops):
 * op = "multiply" | "multiplyconjugate" (y = a * conj(b), complex only) | "add" | "subtract"; both inputs and the output
 * are ComplexFloat32 (complex_data != 0) or Float32.  Execute through lrb200_block_execute_multi with two inputs.
 * lrb200_delay_create replaces DelayBlock:process (radio/blocks/signal/delay.lua:26-60): y[n] = x[n - num_samples],
 * zeros first, the last num_samples inputs carried.
 * lrb200_psd_create replaces spectrum_utils.PSD:compute (radio/utilities/spectrum_utils.lua:524-642), the engine of the
 * spectrum sinks: every whole frame of num_samples inputs (power of two, 2..2^20) is multiplied by `window`
 * (window_utils.window(N, type, true)), transformed, and |X_k|^2 / scale (scale = sample_rate * window energy) is written,
 * as 10*log10 of it when logarithmic != 0; n must be a multiple of num_samples.
 * lrb200_pll_create replaces PLLBlock:process (radio/blocks/signal/pll.lua:113-170): loop constants from
 * (loop_bandwidth, frequency_min, frequency_max) in Hz at `rate`, output 0 = exp(j phi_multiplied) (ComplexFloat32),
 * output 1 = phase error (Float32); execute through lrb200_block_execute_multi with one input and two outputs.  The
 * recurrence is nonlinear and is run in stream order by one thread (exact, a few MS/s).  lrb200_pll_set_mode(q, 1) opts
 * into the chunk-parallel form for long calls: each chunk is simulated by its own thread after a lead-in of
 * 24 / (zeta * loop bandwidth) samples from the phase of the input and the centre frequency, and the multiplied phase is
 * rebuilt exactly from prefix sums of the per-chunk phase increments and errors -- equal to the sequential recurrence (to
 * float32 resolution) WHILE THE LOOP IS LOCKED, not while it acquires or free-runs on noise. */
lrb200_block_t* lrb200_binary_create(const char* op, unsigned complex_data, unsigned flags);
lrb200_block_t* lrb200_pll_create(double loop_bandwidth, double frequency_min, double frequency_max, double multiplier,
                                  double rate, unsigned flags);
int lrb200_pll_set_mode(lrb200_block_t* q, int mode);
lrb200_block_t* lrb200_delay_create(unsigned num_samples, unsigned elem_size, unsigned flags);
lrb200_block_t* lrb200_psd_create(unsigned num_samples, const float32_t* window, double scale, unsigned logarithmic,
                                  unsigned complex_data, unsigned flags);

/* ---- AGCBlock / PowerSquelchBlock (the reference's "Level Control" blocks) -------------------------------------------
 * lrb200_agc_create replaces AGCBlock:process_real / process_complex (radio/blocks/signal/agc.lua:72-115):
 *   P = (1-pa) P + pa |x|^2;  if P >= threshold: g = (1-ga) g + ga (target (1/P)), y = sqrt(g) x;  else y = x (g held)
 * with pa = 1/(1 + power_tau*rate), ga = 1/(1 + gain_tau*rate) and the dBFS target / threshold linearised as 10^(v/10)
 * (agc.lua:57-68), all in double; the output is rounded to float32 once.  lrb200_powersquelch_create replaces
 * PowerSquelchBlock:process_real / process_complex (radio/blocks/signal/powersquelch.lua:43-75): the same power estimator
 * with alpha = 1/(1 + tau*rate), y = x if P >= threshold else 0.  (The reference's PowerSquelchBlock always uses
 * tau = 0.001: powersquelch.lua:26 reads an undefined global, so its second argument is ignored -- its callers pass 0.001.)
 * complex_data != 0: ComplexFloat32, else Float32.  (P, g) start at zero and are carried across calls.  A block-parallel
 * scan with decoupled look-back: one kernel launch per call of up to 256 Mi samples. */
lrb200_block_t* lrb200_agc_create(double target_dbfs, double threshold_dbfs, double gain_tau, double power_tau, double rate,
                                  unsigned complex_data, unsigned flags);
lrb200_block_t* lrb200_powersquelch_create(double threshold_dbfs, double tau, double rate, unsigned complex_data, unsigned flags);

/* ---- BinaryPhaseCorrectorBlock ------------------------------------------------------------------------------------
 * Replaces BinaryPhaseCorrectorBlock:process (radio/blocks/signal/binaryphasecorrector.lua:43-77), ComplexFloat32 in and
 * out.  At every global sample index k*sample_interval (k = 0, 1, ..., whatever the call lengths):
 *   phi = atan2f(im, re) folded into (-pi/2, pi/2] in double;  avg = (avg + phi/N) - last/N
 * where N = num_samples and last is the float32 phi of measurement k-N (0 while the window fills); every sample is then
 * multiplied by ComplexFloat32(cos(-avg), sin(-avg)) with the average after the last measurement at or before it, the
 * product in double and rounded once.  The average and the N-entry window start at zero and are carried across calls;
 * the measurement grid follows the consumed sample count (so seek and sharded cold starts stay on it).  Three kernel
 * launches per call of up to 256 Mi samples.  num_samples and sample_interval must be >= 1. */
lrb200_block_t* lrb200_phasecorrector_create(unsigned num_samples, unsigned sample_interval, unsigned flags);

/* ---- IQFileSource sample formats (the source boundary, SURVEY.md 8f row 1) ------------------------------
 * Replaces the byte-swap + (value - offset) / scale loops of radio/blocks/sources/iqfile.lua:96-108 with the format
 * table of radio/utilities/format_utils.lua:82-97: u8 s8 u16le u16be s16le s16be u32le u32be s32le s32be f32le f32be
 * f64le f64be.  Input: interleaved I/Q in the file's own byte order (2 * sizeof(component) bytes per sample);
 * output: ComplexFloat32.  As the first stage of a graph it makes the host->device copy carry the file bytes
 * (2 B/sample for u8 instead of 8).  Unknown format -> NULL with "Unsupported format". */
lrb200_block_t* lrb200_iqconv_create(const char* format, unsigned flags);
/* RealFileSource (radio/blocks/sources/realfile.lua:86-104): one component per sample -> Float32. */
lrb200_block_t* lrb200_realconv_create(const char* format, unsigned flags);
/* The sink boundary: ComplexFloat32 -> interleaved I/Q (IQFileSink:process, radio/blocks/sinks/iqfile.lua:66-80) and
 * Float32 -> real samples (RealFileSink, radio/blocks/sinks/realfile.lua; WAVFileSink:process, sinks/wavfile.lua:170-186
 * with "u8" / "s16le" / "s32le" for 8 / 16 / 32 bits per sample): raw = x * scale + offset in double, truncated toward
 * zero into the C integer type, then the byte swap.  As the last stage of a graph the device->host copy carries the
 * file's bytes.  Inputs outside [-1, 1] saturate (undefined in the reference). */
lrb200_block_t* lrb200_iqsink_create(const char* format, unsigned flags);
lrb200_block_t* lrb200_realsink_create(const char* format, unsigned flags);

/* ---- GPU flow graph: connected GPU blocks on one stream with device-resident buffers ----------
 * Replaces, for a connected run of GPU blocks, the fork-per-block + socketpair plumbing of
 * radio/core/composite.lua:568-636 and radio/core/pipe.lua:53-88,495-615: the chain
 *   source -> b0 -> b1 -> ... -> sink
 * runs in one process on one CUDA stream; intermediate sample vectors live in a device-resident
 * ring of buffers and never touch the host; host<->device copies (pinned, cudaMemcpyAsync,
 * double-buffered) happen only at the source and sink ends.  Adjacent blocks are fused into single
 * kernels where the library has one (Translator->FIR->Downsampler == TunerBlock,
 * FIR->Downsampler == DecimatorBlock, Discriminator->FIR, IIR->Downsampler).  Blocks added to a
 * graph must have been created with LRB200_DEVICE and are owned by the graph afterwards. */
typedef struct lrb200_graph_s lrb200_graph_t;
lrb200_graph_t* lrb200_graph_create(void);
int    lrb200_graph_append(lrb200_graph_t* g, lrb200_block_t* q);   /* connect q after the current tail */
int    lrb200_graph_commit(lrb200_graph_t* g, int fuse);            /* fuse != 0: apply kernel fusion   */
int    lrb200_graph_execute(lrb200_graph_t* g, const void* x, size_t n, void* y, size_t* n_out);        /* HOST in/out   */
int    lrb200_graph_execute_device(lrb200_graph_t* g, const void* dx, size_t n, void* dy, size_t* n_out); /* DEVICE in/out, async */
size_t lrb200_graph_max_output(const lrb200_graph_t* g, size_t n);  /* room `y` of the next execute(n) must have  */
/* Super-chunk mode for the reference's per-vector regime (vectors of <= 131072 samples, typically 8192:
 * radio/core/pipe.lua:73, radio/blocks/sources/zero.lua:30).  With samples > 0, lrb200_graph_execute packs the host
 * vectors into pinned slots of `samples` input samples; a full slot is uploaded and processed asynchronously while the
 * next one fills, and execute hands back (possibly zero) output samples of slots completed earlier -- a block may
 * return any number of samples per process() call (docs/5.architecture.md:36-47; FIRFilterBlock:process_fft itself
 * emits whole blocks only, firfilter.lua:362).  lrb200_graph_flush pushes the partial slot through and drains
 * (call it at end of stream, where the reference's run loop sees EOF: radio/core/block.lua:588).  samples == 0
 * switches back to synchronous calls. */
int    lrb200_graph_set_superchunk(lrb200_graph_t* g, size_t samples);
int    lrb200_graph_flush(lrb200_graph_t* g, void* y, size_t* n_out);
int    lrb200_graph_reset(lrb200_graph_t* g);
int    lrb200_graph_seek(lrb200_graph_t* g, uint64_t sample_index);
/* Time-chunk sharding of one stream over several GPUs / processes (SURVEY.md 8e; the reference has no counterpart --
 * it parallelises by block, radio/core/composite.lua:568-636).  lrb200_graph_halo: input samples of left context a
 * cold start needs before the outputs equal the streaming ones to float32 resolution (FIR histories, single-pole
 * decay to 1e-12, one discriminator sample), rounded up to 4 whole output periods (keeps buffers 16-byte aligned); < 0 if some stage has unbounded
 * memory.  lrb200_graph_execute_shard runs one chunk: dx -> DEVICE [halo samples of the left neighbour | n samples of
 * this chunk], the chunk starting at global input index `start`.  The stream is run cold from start - halo and the halo's
 * outputs are dropped; only the first stage's few tiles that read the neighbour's samples wait for `halo_ready_event` (a
 * cudaEvent_t recorded after those samples landed, or NULL if they are already there) on a side stream, everything else
 * starts at once, so the exchange overlaps the chunk's kernels.  g_head is unused and may be NULL.  Asynchronous on the
 * library stream; dy receives exactly the outputs of a single-device run for this chunk. */
long long lrb200_graph_halo(lrb200_graph_t* g);
int    lrb200_graph_execute_shard(lrb200_graph_t* g, lrb200_graph_t* g_head, const void* dx, size_t halo, size_t n,
                                  uint64_t start, void* dy, size_t* n_out, void* halo_ready_event);
int    lrb200_graph_num_stages(const lrb200_graph_t* g);            /* kernels stages after fusion */
const char* lrb200_graph_describe(const lrb200_graph_t* g);         /* e.g. "tuner(128,/5) | discrim+fir(128) | iir1+down(/5)" */
const char* lrb200_graph_stage_name(const lrb200_graph_t* g, int stage);
/* per-stage device timing for roofline reporting: when enabled every execute brackets each stage with
 * CUDA events on the library stream; lrb200_graph_stage_time_ms sums them (synchronises) and resets. */
int    lrb200_graph_set_timing(lrb200_graph_t* g, int enable);
double lrb200_graph_stage_time_ms(lrb200_graph_t* g, int stage, int* executions);
void   lrb200_graph_destroy(lrb200_graph_t* g);

/* ---- device DAG: fan-out / fan-in between GPU nodes without host hops ------------------------------------------------
 * Replaces, for a connected set of GPU blocks that is not a straight line, the same fork-per-block + socketpair plumbing
 * (radio/core/composite.lua:568-636): composites/wbfmstereodemodulator.lua:22-64 and amsynchronousdemodulator.lua:25-45 run
 * with every edge in device memory.  A node is a block created with LRB200_DEVICE (any number of ports) or a linear
 * lrb200_graph_t (its fused kernels keep doing the work inside the run); nodes are added in topological order and are
 * owned by the DAG afterwards.  An input / output reference is  node_id * 4 + output_port,  or -1 for the DAG's single
 * input.  All inputs of a node must deliver the same number of samples per call (converging paths with equal rate
 * changes; the reference's PipeMux, radio/core/pipe.lua:495-615, would buffer a surplus).  lrb200_dag_execute: HOST in,
 * HOST outs -- one upload, the node launches in order, one download per output, one synchronize. */
typedef struct lrb200_dag_s lrb200_dag_t;
lrb200_dag_t* lrb200_dag_create(void);
int    lrb200_dag_add_block(lrb200_dag_t* d, lrb200_block_t* q, const int* inputs, unsigned num_inputs);   /* node id or -1 */
int    lrb200_dag_add_graph(lrb200_dag_t* d, lrb200_graph_t* g, int input);                                /* node id or -1 */
int    lrb200_dag_set_outputs(lrb200_dag_t* d, const int* outputs, unsigned num_outputs);
int    lrb200_dag_execute(lrb200_dag_t* d, const void* x, size_t n, void* const* y, size_t* n_out);        /* n_out[k] per output */
size_t lrb200_dag_max_output(const lrb200_dag_t* d, unsigned output, size_t n);
int    lrb200_dag_reset(lrb200_dag_t* d);
const char* lrb200_dag_describe(const lrb200_dag_t* d);
void   lrb200_dag_destroy(lrb200_dag_t* d);

/* ---- synthetic sources on the device (SURVEY.md 8d; the reference analogues are
 * radio/blocks/sources/{uniformrandom,signal}.lua) -- counter-based, so any window of the stream
 * can be regenerated on any GPU.  dst is a DEVICE pointer; async on the library stream. */
int lrb200_synth_white_iq(complex_float32_t* dst, uint64_t n0, size_t n, uint32_t seed);
int lrb200_synth_fm_iq(complex_float32_t* dst, uint64_t n0, size_t n, uint32_t seed,
                       double rate, double carrier, double deviation, float amp, float noise);

#ifdef __cplusplus
}
#endif
#endif /* LRB200_H */
