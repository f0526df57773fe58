/*
 * phastft_cuda.h -- C ABI of libphastft_cuda.so, the H100 (sm_90a) drop-in for PhastFT's
 * 1-D power-of-two FFT path.
 *
 * The reference (QuState/PhastFT @ 8cd3a39) has no FFI boundary: the path sits behind its
 * public Rust API.  Each entry point below names the reference item it stands in for; the
 * thin Rust wrappers that keep the reference's names and panics are in rust/src/lib.rs, the
 * C++ and Python mirrors in cpp/phastft.hpp and phastft_b200/api.py (see INTEGRATION.md).
 *
 * Conventions
 *   - plain pointers and sizes only; every function returns a phastft_status (int32_t), never
 *     aborts, never throws; phastft_last_error() gives a thread-local detail string.
 *   - planar data: separate re[] and im[] arrays of T, natural order in and out
 *     (README.md:174-178 of the reference); forward unscaled, reverse scaled by 1/N
 *     (algorithms/dit.rs:297-331).
 *   - `*_host` entry points take HOST pointers and are synchronous and in place from the
 *     caller's view (API parity with the Rust slices).  `*_dev` entry points take DEVICE
 *     pointers, enqueue on the given cudaStream_t (passed as void*), allocate nothing and do
 *     not synchronise: these are what bench.py's device-resident number measures.
 *   - plans are immutable after creation and may be shared between host threads (the Rust
 *     planners are Send + Sync); calls on one plan serialise on the plan's internal workspace.
 *   - there is NO CPU fallback: without a CUDA device every call returns PHASTFT_ERR_NO_DEVICE.
 */
#ifndef PHASTFT_CUDA_H
#define PHASTFT_CUDA_H

#include <stddef.h>
#include <stdint.h>

#include "phastft_status.h"

#ifdef __cplusplus
extern "C" {
#endif

#define PHASTFT_API __attribute__((visibility("default")))

/* ---- library -------------------------------------------------------------------------- */
PHASTFT_API const char* phastft_last_error(void);            /* thread-local, never NULL */
PHASTFT_API const char* phastft_version(void);
PHASTFT_API int32_t phastft_device_count(int* count);
/* number of CUDA kernels this library has launched in this process (bench.py "gpu_launches") */
PHASTFT_API uint64_t phastft_launch_count(void);
/* Thread-local, like phastft_last_error: the kernels the calling thread's most recent execution call (any *_host,
 * *_oneshot, *_dev, *_dev_profile or *_batch_sharded_host entry point) launched, one entry per launch, in order, separated
 * by "; ".  Each entry reads "<kind> R=<rows> C=<columns> NT=<threads> v<variant> <mode>[ pdl]": kind COL / TRANS (strided
 * passes), ROW (one CTA per transform), CLUSTER (both passes in one cluster launch: R=<R1>x<R2>, K=<CTAs per cluster>),
 * PIPE (both passes in one pipelined launch: R=<R1>x<R2>), R2C-UNTANGLE / C2R-PRE (the real transforms' elementwise
 * kernels), CHIRP-PRE / CHIRP-MUL / CHIRP-POST (the any-length transform's elementwise kernels: R=<M>, C=<members>); mode plain, tma (tile input by TMA), bulk (tile input by bulk copies), row-bulk (one-CTA tile in and out by bulk
 * copies), c2r-in (c2r pre-processing on load), cluster, pipe or pipe-tma; " pdl" marks programmatic dependent launch.
 * Reset at the start of every execution call; valid until the thread's next call. */
PHASTFT_API const char* phastft_last_launches(void);
/* The *_oneshot entry points (a planner per call, lib.rs:180 / r2c.rs:522,696) keep their most recent plan per
 * precision and reuse it when the next call has the same size and device; this releases those plans and their
 * device buffers. */
PHASTFT_API void phastft_oneshot_cache_clear(void);
/* Page-lock / release a caller-owned host range (cudaHostRegister / cudaHostUnregister).  The *_host entry points
 * accept any host memory, but copies from ordinary pageable memory run several times slower than from page-locked
 * memory, and the batched host pipeline only overlaps with page-locked memory.
 * Register long-lived buffers once; registration itself costs about as much as several copies. */
PHASTFT_API int32_t phastft_host_register(void* host_ptr, size_t bytes);
PHASTFT_API int32_t phastft_host_unregister(void* host_ptr);

/* ---- options.rs:10-43 : Options / guess_options ------------------------------------------
 * Kept for source compatibility.  On the GPU both fields are hints with no effect: there is
 * no separate bit-reversal step to thread and the grid is always full-chip parallel. */
typedef struct phastft_options {
    int32_t multithreaded_bit_reversal;     /* options.rs:16 */
    size_t smallest_parallel_chunk_size;    /* options.rs:23, default 16384 */
} phastft_options;
PHASTFT_API void phastft_options_default(phastft_options* out);            /* options.rs:26-33 */
PHASTFT_API void phastft_options_guess(size_t input_size, phastft_options* out); /* options.rs:38-43 */

/* ---- planner.rs:25-32 PlannerMode ------------------------------------------------------ */
#define PHASTFT_MODE_HEURISTIC 0
#define PHASTFT_MODE_TUNE 1   /* times a few pass decompositions / tile widths at plan time and keeps the fastest
                                 (the reference accepts the mode and ignores it, planner.rs:65) */

/* ---- planner.rs:34-114 : PlannerDit64 / PlannerDit32 -------------------------------------
 * num_points must be a non-zero power of two (planner.rs:66) else PHASTFT_ERR_NOT_POW2.
 * The plan owns the device twiddle tables (two-level W_N table + per-pass W_R tables) and,
 * lazily, a device workspace of N complex elements (multi-pass sizes only). */
typedef struct phastft_plan_dit_f64 phastft_plan_dit_f64;
typedef struct phastft_plan_dit_f32 phastft_plan_dit_f32;
PHASTFT_API int32_t phastft_plan_dit_f64_create(size_t num_points, int device, int mode, phastft_plan_dit_f64** out);
PHASTFT_API int32_t phastft_plan_dit_f32_create(size_t num_points, int device, int mode, phastft_plan_dit_f32** out);
PHASTFT_API void phastft_plan_dit_f64_destroy(phastft_plan_dit_f64* plan);
PHASTFT_API void phastft_plan_dit_f32_destroy(phastft_plan_dit_f32* plan);
PHASTFT_API size_t phastft_plan_dit_f64_size(const phastft_plan_dit_f64* plan);
PHASTFT_API size_t phastft_plan_dit_f32_size(const phastft_plan_dit_f32* plan);
/* Human-readable pass decomposition, e.g. "n=2^20 f64: COL R=1024 C=8 | TRANS R=1024 C=8". */
PHASTFT_API const char* phastft_plan_dit_f64_describe(const phastft_plan_dit_f64* plan);
PHASTFT_API const char* phastft_plan_dit_f32_describe(const phastft_plan_dit_f32* plan);

/* Sizes the plan's device workspace for calls of up to `batch` transforms now (the *_dev entry points otherwise
 * grow it on the first larger call, which synchronises the device and is an error inside a CUDA-graph capture). */
PHASTFT_API int32_t phastft_plan_dit_f64_reserve(const phastft_plan_dit_f64* plan, size_t batch);
PHASTFT_API int32_t phastft_plan_dit_f32_reserve(const phastft_plan_dit_f32* plan, size_t batch);

/* Host-only planning logic (no device needed): the pass decomposition N = 2^f0 * 2^f1 [* 2^f2] the
 * planner uses for `num_points` (one CTA per transform when *num_passes == 1; 0 passes for N == 1).
 * log2_factors must hold 3 ints. */
PHASTFT_API int32_t phastft_plan_factorization(size_t num_points, int precision_bits, int* log2_factors, int* num_passes);
/* Host-only: the alternative plans PHASTFT_MODE_TUNE times against the heuristic one for `num_points` (the tuner reads
 * this same list).  Candidate i has the pass sizes 2^log2_factors[3i + p] and tile widths pass_c[3i + p] (columns) for
 * p < its number of passes; unused slots are 0.  *count receives the number of candidates (0 for one-CTA sizes); at most
 * `max` are written. */
PHASTFT_API int32_t phastft_plan_tune_candidates(size_t num_points, int precision_bits, int* log2_factors, int* pass_c, int max, int* count);

/* Planner-table blob (multi-GPU init, SURVEY.md section 8e): rank 0 exports its tables into a
 * device buffer, the host framework broadcasts that buffer once (ncclBroadcast /
 * torch.distributed.broadcast), every other rank imports it.  No per-call collectives.
 * The blob starts with a 256-byte layout header (size, precision, pass sizes, each pass's tile width and first
 * radix): import / broadcast return PHASTFT_ERR_PLAN_MISMATCH when the receiving plan was built with a different
 * decomposition (PlannerMode::Tune or a PHASTFT_* override on one rank only) instead of installing foreign tables. */
PHASTFT_API size_t phastft_plan_dit_f64_tables_bytes(const phastft_plan_dit_f64* plan);
PHASTFT_API size_t phastft_plan_dit_f32_tables_bytes(const phastft_plan_dit_f32* plan);
PHASTFT_API int32_t phastft_plan_dit_f64_tables_export(const phastft_plan_dit_f64* plan, void* dst_dev, void* stream);
PHASTFT_API int32_t phastft_plan_dit_f32_tables_export(const phastft_plan_dit_f32* plan, void* dst_dev, void* stream);
PHASTFT_API int32_t phastft_plan_dit_f64_tables_import(phastft_plan_dit_f64* plan, const void* src_dev, void* stream);
PHASTFT_API int32_t phastft_plan_dit_f32_tables_import(phastft_plan_dit_f32* plan, const void* src_dev, void* stream);
/* Native NCCL path for the same broadcast: `comm` is an ncclComm_t created by the caller;
 * libnccl.so.2 is dlopen()ed on first use (PHASTFT_ERR_NCCL if absent). */
PHASTFT_API int32_t phastft_plan_dit_f64_tables_broadcast(phastft_plan_dit_f64* plan, void* nccl_comm, int root, void* stream);
PHASTFT_API int32_t phastft_plan_dit_f32_tables_broadcast(phastft_plan_dit_f32* plan, void* nccl_comm, int root, void* stream);

/* ---- lib.rs:143-226, algorithms/dit.rs:263-401 : fft_64_dit* / fft_32_dit* ----------------
 * Host-slice execution: fft_{64,32}_dit_with_planner[_and_opts](reals, imags, direction, planner[, opts]).
 * len_re / len_im are the slice lengths; the reference's asserts map to
 *   len_re != len_im -> PHASTFT_ERR_LEN_MISMATCH, not a power of two -> PHASTFT_ERR_NOT_POW2,
 *   log2(len) != plan -> PHASTFT_ERR_PLAN_MISMATCH.
 * `opts` may be NULL (= guess_options(len), lib.rs:149). */
PHASTFT_API int32_t phastft_fft_dit_f64_host(const phastft_plan_dit_f64* plan, double* reals, size_t len_re,
                                             double* imags, size_t len_im, int direction, const phastft_options* opts);
PHASTFT_API int32_t phastft_fft_dit_f32_host(const phastft_plan_dit_f32* plan, float* reals, size_t len_re,
                                             float* imags, size_t len_im, int direction, const phastft_options* opts);
/* fft_64_dit / fft_32_dit (lib.rs:180, 223): plans per call on `device`, like the reference. */
PHASTFT_API int32_t phastft_fft_dit_f64_oneshot(double* reals, size_t len_re, double* imags, size_t len_im,
                                                int direction, int device);
PHASTFT_API int32_t phastft_fft_dit_f32_oneshot(float* reals, size_t len_re, float* imags, size_t len_im,
                                                int direction, int device);

/* Device-resident execution (batched): `batch` transforms, transform b at d_re + b*batch_stride
 * (batch_stride >= N elements; the reference has no batch API -- a batch is a caller loop over
 * fft_32_dit_with_planner sharing one planner, examples/benchmark.rs:24-36).  In place. */
PHASTFT_API int32_t phastft_fft_dit_f64_dev(const phastft_plan_dit_f64* plan, double* d_reals, double* d_imags,
                                            int direction, size_t batch, size_t batch_stride, void* stream);
PHASTFT_API int32_t phastft_fft_dit_f32_dev(const phastft_plan_dit_f32* plan, float* d_reals, float* d_imags,
                                            int direction, size_t batch, size_t batch_stride, void* stream);
/* Profiling aid (bench.py's roofline): same as *_dev, but records CUDA events on `stream` around
 * every pass (kernel launch) of the first L2 chunk, synchronises, and returns the per-pass device
 * times in milliseconds (pass_ms must hold 3 floats). */
PHASTFT_API int32_t phastft_fft_dit_f64_dev_profile(const phastft_plan_dit_f64* plan, double* d_reals, double* d_imags,
                                                    int direction, size_t batch, size_t batch_stride, void* stream,
                                                    float* pass_ms, int* num_passes);
PHASTFT_API int32_t phastft_fft_dit_f32_dev_profile(const phastft_plan_dit_f32* plan, float* d_reals, float* d_imags,
                                                    int direction, size_t batch, size_t batch_stride, void* stream,
                                                    float* pass_ms, int* num_passes);
/* Host-slice batched execution sharded over devices (SURVEY.md section 8e): transforms
 * [g*batch/G, (g+1)*batch/G) run on plans[g] (one plan per device, tables made identical by the
 * init-time broadcast).  Synchronous. */
PHASTFT_API int32_t phastft_fft_dit_f32_batch_sharded_host(phastft_plan_dit_f32* const* plans, int num_plans,
                                                           float* reals, float* imags, size_t batch,
                                                           size_t batch_stride, int direction);
PHASTFT_API int32_t phastft_fft_dit_f64_batch_sharded_host(phastft_plan_dit_f64* const* plans, int num_plans,
                                                           double* reals, double* imags, size_t batch,
                                                           size_t batch_stride, int direction);

/* ---- planner.rs:164-212 : PlannerR2c64 / PlannerR2c32 -------------------------------------
 * n must be a power of two >= 4 else PHASTFT_ERR_R2C_N ("n must be a power of 2 >= 4"). */
typedef struct phastft_plan_r2c_f64 phastft_plan_r2c_f64;
typedef struct phastft_plan_r2c_f32 phastft_plan_r2c_f32;
PHASTFT_API int32_t phastft_plan_r2c_f64_create(size_t n, int device, phastft_plan_r2c_f64** out);
PHASTFT_API int32_t phastft_plan_r2c_f32_create(size_t n, int device, phastft_plan_r2c_f32** out);
PHASTFT_API void phastft_plan_r2c_f64_destroy(phastft_plan_r2c_f64* plan);
PHASTFT_API void phastft_plan_r2c_f32_destroy(phastft_plan_r2c_f32* plan);
PHASTFT_API size_t phastft_plan_r2c_f64_size(const phastft_plan_r2c_f64* plan);
PHASTFT_API size_t phastft_plan_r2c_f32_size(const phastft_plan_r2c_f32* plan);
/* The path c2r calls on this plan take under the current environment, then the first pass's c2r build and the inner
 * N/2-point plan's own description, e.g.
 *   "n=2^20 f64 r2c/c2r: c2r fused on load (the first pass loads the half-spectrum) | c2r-in build: COL R=512 C=8 NT=256 R1=32
 *    | inner: n=2^19 f64: ..."
 * "fused on load" (the first pass builds its input from the half-spectrum; launch record mode c2r-in) or "separate sweep"
 * (a C2R-PRE launch into scratch first), with the rule that decided in parentheses.  The string is rebuilt per call and stays
 * valid until the calling thread's next call of either describe function. */
PHASTFT_API const char* phastft_plan_r2c_f64_describe(const phastft_plan_r2c_f64* plan);
PHASTFT_API const char* phastft_plan_r2c_f32_describe(const phastft_plan_r2c_f32* plan);
/* The same for batched calls of `batch` transforms (phastft_{r2c,c2r}_*_batch_dev): the c2r path that batch takes, the rule that
 * decided, and the c2r build of the first pass such a call runs ("none" where it runs a kernel without one: the one-CTA
 * kernel, the cluster or pipelined launch, the TMA pair).  describe_batch(plan, 1) equals describe(plan). */
PHASTFT_API const char* phastft_plan_r2c_f64_describe_batch(const phastft_plan_r2c_f64* plan, size_t batch);
PHASTFT_API const char* phastft_plan_r2c_f32_describe_batch(const phastft_plan_r2c_f32* plan, size_t batch);
/* Makes, now and on this thread, every allocation a batched call of `batch` transforms would make: the inner plan's workspace
 * and, when that batch's c2r takes the separate sweep, the plan-owned c2r scratch (batch * N/2 per array).  A batched call that
 * would grow either while its stream is being captured into a CUDA graph returns PHASTFT_ERR_INVALID_ARG instead. */
PHASTFT_API int32_t phastft_plan_r2c_f64_reserve(const phastft_plan_r2c_f64* plan, size_t batch);
PHASTFT_API int32_t phastft_plan_r2c_f32_reserve(const phastft_plan_r2c_f32* plan, size_t batch);

/* ---- algorithms/r2c.rs:521-662 : r2c_fft_{f64,f32}[_with_planner] --------------------------
 * input (length N, not modified) -> output_re/output_im (length N/2+1 each).  Length checks in
 * the reference's order (r2c.rs:543-553). */
PHASTFT_API int32_t phastft_r2c_f64_host(const phastft_plan_r2c_f64* plan, const double* input, size_t len_in,
                                         double* output_re, size_t len_ore, double* output_im, size_t len_oim);
PHASTFT_API int32_t phastft_r2c_f32_host(const phastft_plan_r2c_f32* plan, const float* input, size_t len_in,
                                         float* output_re, size_t len_ore, float* output_im, size_t len_oim);
/* r2c_fft_f64 / r2c_fft_f32 (r2c.rs:521, 598): plans per call. */
PHASTFT_API int32_t phastft_r2c_f64_oneshot(const double* input, size_t len_in, double* output_re, size_t len_ore,
                                            double* output_im, size_t len_oim, int device);
PHASTFT_API int32_t phastft_r2c_f32_oneshot(const float* input, size_t len_in, float* output_re, size_t len_ore,
                                            float* output_im, size_t len_oim, int device);
/* Device-resident: d_input N reals, d_out_re/d_out_im N/2+1 each; asynchronous on `stream`.
 * d_input is read as N/2 (re, im) pairs: it must be aligned to 2 * sizeof(T) bytes (16 for f64, 8 for f32), else
 * PHASTFT_ERR_INVALID_ARG and nothing is launched. */
PHASTFT_API int32_t phastft_r2c_f64_dev(const phastft_plan_r2c_f64* plan, const double* d_input, double* d_out_re,
                                        double* d_out_im, void* stream);
PHASTFT_API int32_t phastft_r2c_f32_dev(const phastft_plan_r2c_f32* plan, const float* d_input, float* d_out_re,
                                        float* d_out_im, void* stream);

/* ---- algorithms/r2c.rs:695-895 : c2r_fft_{f64,f32}[_with_planner[_and_scratch]] -------------
 * input_re/input_im (N/2+1 each, not modified) -> output (N reals), fully normalised so that
 * c2r(r2c(x)) == x.  scratch_re/scratch_im: caller scratch of N/2 each, or both NULL with
 * len 0 to let the plan use its own device workspace (the reference's allocating variants,
 * r2c.rs:716-718).  Host scratch is only length-checked (r2c.rs:761-762): the work happens in
 * device memory. */
PHASTFT_API int32_t phastft_c2r_f64_host(const phastft_plan_r2c_f64* plan, const double* input_re, size_t len_ire,
                                         const double* input_im, size_t len_iim, double* output, size_t len_out,
                                         double* scratch_re, size_t len_sre, double* scratch_im, size_t len_sim);
PHASTFT_API int32_t phastft_c2r_f32_host(const phastft_plan_r2c_f32* plan, const float* input_re, size_t len_ire,
                                         const float* input_im, size_t len_iim, float* output, size_t len_out,
                                         float* scratch_re, size_t len_sre, float* scratch_im, size_t len_sim);
PHASTFT_API int32_t phastft_c2r_f64_oneshot(const double* input_re, size_t len_ire, const double* input_im,
                                            size_t len_iim, double* output, size_t len_out, int device);
PHASTFT_API int32_t phastft_c2r_f32_oneshot(const float* input_re, size_t len_ire, const float* input_im,
                                            size_t len_iim, float* output, size_t len_out, int device);
/* Device-resident: d_scratch_re/d_scratch_im N/2 each or both NULL (plan workspace).  d_output is written as N/2
 * (re, im) pairs: it must be aligned to 2 * sizeof(T) bytes, else PHASTFT_ERR_INVALID_ARG and nothing is launched. */
PHASTFT_API int32_t phastft_c2r_f64_dev(const phastft_plan_r2c_f64* plan, const double* d_in_re, const double* d_in_im,
                                        double* d_output, double* d_scratch_re, double* d_scratch_im, void* stream);
PHASTFT_API int32_t phastft_c2r_f32_dev(const phastft_plan_r2c_f32* plan, const float* d_in_re, const float* d_in_im,
                                        float* d_output, float* d_scratch_re, float* d_scratch_im, void* stream);

/* ---- batched r2c / c2r, device-resident (the reference has no batch API: a batch is a caller loop) --------------------
 * `batch` transforms in one call, asynchronous on `stream`; each member means exactly what the lone *_dev call means.
 * Strides are in elements of the array they describe: member b of a real array starts at b * stride reals, member b of a
 * spectrum array at b * stride bins.
 *   r2c: in_stride >= N and even, out_stride >= N/2 + 1; writes N/2 + 1 bins per member, never writes d_input.
 *   c2r: in_stride >= N/2 + 1, out_stride >= N and even; normalised so that c2r(r2c(x)) == x, never writes the spectra.
 *        d_scratch_re / d_scratch_im: batch * N/2 elements each, dense, or both NULL for the plan-owned scratch (grown to
 *        batch * N/2 on first use, or ahead of time by phastft_plan_r2c_*_reserve).
 * The real arrays are accessed as (re, im) pairs: their base must be aligned to 2 * sizeof(T) bytes, which is why the real
 * stride must be even.  A stride that is too small or odd, a misaligned base, one scratch pointer without the other or a
 * NULL pointer returns PHASTFT_ERR_INVALID_ARG (the detail names the argument) before anything is launched.  batch == 0
 * launches nothing; batch == 1 runs exactly the lone *_dev call.  The c2r path of a batch (fused into the first pass's loads
 * or the separate sweep) is stated by phastft_plan_r2c_*_describe_batch. */
PHASTFT_API int32_t phastft_r2c_f64_batch_dev(const phastft_plan_r2c_f64* plan, const double* d_input, size_t in_stride,
                                              double* d_out_re, double* d_out_im, size_t out_stride, size_t batch, void* stream);
PHASTFT_API int32_t phastft_r2c_f32_batch_dev(const phastft_plan_r2c_f32* plan, const float* d_input, size_t in_stride,
                                              float* d_out_re, float* d_out_im, size_t out_stride, size_t batch, void* stream);
PHASTFT_API int32_t phastft_c2r_f64_batch_dev(const phastft_plan_r2c_f64* plan, const double* d_in_re, const double* d_in_im,
                                              size_t in_stride, double* d_output, size_t out_stride, double* d_scratch_re,
                                              double* d_scratch_im, size_t batch, void* stream);
PHASTFT_API int32_t phastft_c2r_f32_batch_dev(const phastft_plan_r2c_f32* plan, const float* d_in_re, const float* d_in_im,
                                              size_t in_stride, float* d_output, size_t out_stride, float* d_scratch_re,
                                              float* d_scratch_im, size_t batch, void* stream);

/* ---- complex FFTs of any length (the reference accepts powers of two only) -------------------------------------------
 * n >= 1.  A power of two runs the n-point c2c plan exactly as phastft_fft_dit_*_dev does (same results, same launches).
 * Any other n up to 2^29 - 1 uses Bluestein's chirp-z algorithm: with w[j] = exp(-pi i (j^2 mod 2n) / n),
 * X[k] = w[k] sum_j (x[j] w[j]) conj(w[k - j]), a circular convolution of length M = 2^ceil(log2(2n - 1)) computed by two
 * forward M-point c2c transforms of the library between three elementwise kernels (CHIRP-PRE, CHIRP-MUL, CHIRP-POST in
 * phastft_last_launches).  The plan owns the chirp, the transform of the convolution kernel (computed once in f64) and a
 * workspace of batch * M complex values.  Any other n returns PHASTFT_ERR_INVALID_ARG before the device is touched.
 * Semantics of the fft_dit entry points: planar, in place, natural order, forward unscaled, reverse scaled by 1/n. */
typedef struct phastft_plan_any_f64 phastft_plan_any_f64;
typedef struct phastft_plan_any_f32 phastft_plan_any_f32;
PHASTFT_API int32_t phastft_plan_any_f64_create(size_t n, int device, phastft_plan_any_f64** out);
PHASTFT_API int32_t phastft_plan_any_f32_create(size_t n, int device, phastft_plan_any_f32** out);
PHASTFT_API void phastft_plan_any_f64_destroy(phastft_plan_any_f64* plan);
PHASTFT_API void phastft_plan_any_f32_destroy(phastft_plan_any_f32* plan);
PHASTFT_API size_t phastft_plan_any_f64_size(const phastft_plan_any_f64* plan);
PHASTFT_API size_t phastft_plan_any_f32_size(const phastft_plan_any_f32* plan);
/* "n=1000 f64 any: Bluestein M=2^11 | inner: n=2^11 f64: ..." or "n=2^20 f64 any: power of two | inner: n=2^20 f64: ..." */
PHASTFT_API const char* phastft_plan_any_f64_describe(const phastft_plan_any_f64* plan);
PHASTFT_API const char* phastft_plan_any_f32_describe(const phastft_plan_any_f32* plan);
/* Makes every allocation a call of `batch` transforms would make now: the inner plan's workspace and this plan's batch * M.
 * A call that would grow either while its stream is being captured into a CUDA graph returns PHASTFT_ERR_INVALID_ARG. */
PHASTFT_API int32_t phastft_plan_any_f64_reserve(const phastft_plan_any_f64* plan, size_t batch);
PHASTFT_API int32_t phastft_plan_any_f32_reserve(const phastft_plan_any_f32* plan, size_t batch);
/* Device-resident, asynchronous on `stream`: `batch` transforms, transform b at d_re + b * batch_stride (batch_stride >= n
 * when batch > 1).  batch == 0 launches nothing.  NULL pointers and bad directions return PHASTFT_ERR_INVALID_ARG before any
 * launch.  Allocates only when the plan's workspace must grow (synchronising). */
PHASTFT_API int32_t phastft_fft_any_f64_dev(const phastft_plan_any_f64* plan, double* d_reals, double* d_imags, int direction,
                                            size_t batch, size_t batch_stride, void* stream);
PHASTFT_API int32_t phastft_fft_any_f32_dev(const phastft_plan_any_f32* plan, float* d_reals, float* d_imags, int direction,
                                            size_t batch, size_t batch_stride, void* stream);
/* Host slices, synchronous, in place: len_re != len_im -> PHASTFT_ERR_LEN_MISMATCH, length != n -> PHASTFT_ERR_PLAN_MISMATCH. */
PHASTFT_API int32_t phastft_fft_any_f64_host(const phastft_plan_any_f64* plan, double* reals, size_t len_re, double* imags,
                                             size_t len_im, int direction);
PHASTFT_API int32_t phastft_fft_any_f32_host(const phastft_plan_any_f32* plan, float* reals, size_t len_re, float* imags,
                                             size_t len_im, int direction);

/* ---- lib.rs:41-140 (feature complex-nums): fft_{64,32}_interleaved* --------------------------
 * signal = N interleaved (re, im) pairs (num_complex::Complex<T> layout), in place.  The
 * reference deinterleaves into two fresh Vecs, runs the planar FFT and re-interleaves
 * (complex_nums.rs:11-55); here the AoS<->planar conversion is fused into the first pass's
 * load and the last pass's store.  The *_dev form accesses d_signal as (re, im) pairs: it must be aligned to
 * 2 * sizeof(T) bytes (a Complex<T>'s own alignment), else PHASTFT_ERR_INVALID_ARG and nothing is launched. */
PHASTFT_API int32_t phastft_fft_interleaved_f64_host(const phastft_plan_dit_f64* plan, double* signal, size_t len_complex,
                                                     int direction);
PHASTFT_API int32_t phastft_fft_interleaved_f32_host(const phastft_plan_dit_f32* plan, float* signal, size_t len_complex,
                                                     int direction);
PHASTFT_API int32_t phastft_fft_interleaved_f64_dev(const phastft_plan_dit_f64* plan, double* d_signal, int direction,
                                                    size_t batch, size_t batch_stride_complex, void* stream);
PHASTFT_API int32_t phastft_fft_interleaved_f32_dev(const phastft_plan_dit_f32* plan, float* d_signal, int direction,
                                                    size_t batch, size_t batch_stride_complex, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PHASTFT_CUDA_H */
