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
 * kernels), CHIRP-PRE / CHIRP-MUL / CHIRP-POST (the any-length transform's elementwise kernels: R=<M>, C=<members>), CHIRP-PRE-R2C /
 * CHIRP-POST-R2C / CHIRP-PRE-C2R / CHIRP-POST-C2R (the same around the real any-length transforms), SMOOTH-PRE (the mixed-radix
 * path's de-interleave: R=<P>, C=<workspace members>) and ODD (its radix-3/5/7 passes: R=<rows>, C=<columns per CTA>, mode reg
 * for the register kernel or tile for the shared-memory one), SMOOTH-PRE-R2C / SMOOTH-PRE-C2R and ODD-R2C / ODD-C2R (the same with
 * the real any-length transforms' loads and last-pass stores), SMOOTH-POST-R2C (their halved r2c's untangle: R=<L>,
 * C=<members>) and CHIRP-PRE-IL / CHIRP-POST-IL / SMOOTH-PRE-IL / ODD-IL (the complex any-length transform's end kernels, the
 * last ODD pass only, in phastft_fft_interleaved_any_*: R, C and NT as in the planar call), R2C-UNTANGLE-IL / C2R-PRE-IL /
 * CHIRP-POST-R2C-IL / CHIRP-PRE-C2R-IL / SMOOTH-PRE-C2R-IL / ODD-R2C-IL / SMOOTH-POST-R2C-IL (the spectrum's end of
 * phastft_{r2c,c2r}_interleaved_any_*, whose halved mixed r2c's last pass is ODD-IL), DCT-PRE-<kind> / DCT-POST-<kind> (the ends of
 * phastft_dct_*, kind DCT2, DCT3, DST2 or DST3: R=<N>, C=<members>), CONV-PRE / CONV-MUL / CONV-POST (phastft_conv_*: R=<L>,
 * C=<members>), STFT-FRAME (phastft_stft_*: R=<n_fft>, C=<frames>) / ISTFT-OLA (phastft_istft_*: R=<n_fft>, C=<members>); mode plain, tma (tile input by TMA), bulk (tile input by bulk copies), row-bulk (one-CTA tile in and out by bulk
 * copies), c2r-in (c2r pre-processing on load), c2r-in-il (the same from interleaved bins), cluster, pipe or pipe-tma; " pdl" marks
 * programmatic dependent launch.
 * Reset at the start of every execution call; valid until the thread's next call. */
PHASTFT_API const char* phastft_last_launches(void);
/* Thread-local, like phastft_last_launches: the bytes of plan-owned scratch (workspaces, c2r scratch, host staging) that the
 * calling thread's most recent execution call filled with 0xFF bytes (a NaN in f32 and f64) before using them.  Nonzero only
 * for plans built while the environment variable PHASTFT_SCRIBBLE=1 was set: such plans poison their scratch when it is
 * allocated and, with cudaMemsetAsync on the call's stream, before each call's first use, so a kernel that reads scratch it has
 * not written in the same call produces NaN.  A testing aid; it never touches constant tables and changes no result.
 * A second testing aid, the environment variable PHASTFT_GRID_BLOCKS_MAX, is read on every call: the most blocks one launch of
 * a member-major elementwise kernel (R2C-UNTANGLE*, C2R-PRE*, SMOOTH-PRE*, SMOOTH-POST-R2C*, CHIRP-*, DCT-PRE-* / DCT-POST-*,
 * CONV-*, STFT-FRAME, ISTFT-OLA) may have.  A call whose grid would exceed it launches the kernel several times, each launch
 * on at most max(1, cap / blocks-per-member) members, with one launch record each.  Unset, not a number, <= 0 or above
 * 2^31 - 1 it is 2^31 - 1, gridDim.x's limit; a lower value makes those splits run at small sizes with the same results. */
PHASTFT_API uint64_t phastft_last_scribble_bytes(void);
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
/* The algorithm of a length that is not a power of two (a power of two takes the c2c plan under every value):
 *   PHASTFT_ANY_BLUESTEIN  Bluestein, as phastft_plan_any_*_create builds.
 *   PHASTFT_ANY_MIXED      the mixed-radix path for n = P * Q < 2^30, P = 2^a, Q = 3^b 5^c 7^d > 1: SMOOTH-PRE de-interleaves the
 *                          input by Q into a workspace of n complex values, the P-point plan transforms its Q * batch members,
 *                          and one ODD pass (Q <= 729) or two (Q = Q_a * Q_b, both <= 729, the most balanced split) run the
 *                          Q-point DFTs with the W_n twiddles and store in natural order.  No padding: about 8n values through
 *                          device memory where Bluestein moves 40n to 50n.  A length with another prime factor, or whose odd part
 *                          has no such split, returns PHASTFT_ERR_INVALID_ARG (the detail names the factor) before the device is
 *                          touched.  Smooth lengths between 2^29 and 2^30 run on this path only.
 *   PHASTFT_ANY_AUTO       mixed when n is eligible, Bluestein otherwise: decided from the factorisation of n alone.  The value
 *                          to pass unless one algorithm is wanted.
 * describe(): "n=1000000 f64 any: mixed 2^6 x 125 x 125 | inner: n=2^6 f64: ..." ("mixed 2^20 x 3" with one odd pass). */
#define PHASTFT_ANY_BLUESTEIN 0
#define PHASTFT_ANY_MIXED 1
#define PHASTFT_ANY_AUTO 2
PHASTFT_API int32_t phastft_plan_any_f64_create_with(size_t n, int device, int algo, phastft_plan_any_f64** out);
PHASTFT_API int32_t phastft_plan_any_f32_create_with(size_t n, int device, int algo, phastft_plan_any_f32** out);
/* Host-only: the split n = p * q_a * q_b of the mixed-radix path (q_b = 1: one odd pass; the same for both precisions), or
 * PHASTFT_ERR_INVALID_ARG with the reason when n is not eligible. */
PHASTFT_API int32_t phastft_any_mixed_factorization(size_t n, size_t* p, int* q_a, int* q_b);
/* Makes every allocation a call of `batch` transforms would make now: the inner plan's workspace and this plan's batch * M
 * (mixed: batch * n).
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
/* The same transforms on interleaved (re, im) pairs (torch.complex128 / complex64, std::complex<T>, num_complex::Complex<T>),
 * with any plan phastft_plan_any_*_create or _create_with built: member b starts at complex element b * batch_stride_complex
 * (>= n when batch > 1), in place, natural order, forward unscaled, reverse scaled by 1/n.  d_signal must be aligned to
 * 2 * sizeof(T) bytes.  Powers of two run phastft_fft_interleaved_*_dev on the plan's n-point plan; Bluestein and mixed-radix
 * plans run the kernels of phastft_fft_any_*_dev with the interleaved layout at both ends (CHIRP-PRE-IL / CHIRP-POST-IL,
 * SMOOTH-PRE-IL / ODD-IL) and give the planar call's results bit for bit.  Workspace, reserve() and batch == 0 as in
 * phastft_fft_any_*_dev; NULL or misaligned pointers, bad directions and short strides return PHASTFT_ERR_INVALID_ARG before any
 * launch.  The host form stages through a buffer of n complex values that its first call allocates; len_complex != n returns
 * PHASTFT_ERR_PLAN_MISMATCH. */
PHASTFT_API int32_t phastft_fft_interleaved_any_f64_dev(const phastft_plan_any_f64* plan, double* d_signal, int direction,
                                                        size_t batch, size_t batch_stride_complex, void* stream);
PHASTFT_API int32_t phastft_fft_interleaved_any_f32_dev(const phastft_plan_any_f32* plan, float* d_signal, int direction,
                                                        size_t batch, size_t batch_stride_complex, void* stream);
PHASTFT_API int32_t phastft_fft_interleaved_any_f64_host(const phastft_plan_any_f64* plan, double* signal, size_t len_complex,
                                                         int direction);
PHASTFT_API int32_t phastft_fft_interleaved_any_f32_host(const phastft_plan_any_f32* plan, float* signal, size_t len_complex,
                                                         int direction);

/* ---- real-input FFTs of any length (the reference's r2c / c2r accept powers of two >= 4 only) ---------------------------
 * r2c reads n reals and writes the n/2 + 1 bins X[0 .. floor(n/2)], planar, forward, unscaled.  c2r reads n/2 + 1 bins and
 * writes n reals scaled by 1/n, so c2r(r2c(x)) == x.  The path depends on n:
 *   a power of two, 4 .. 2^31   the r2c plan, exactly as phastft_{r2c,c2r}_*_batch_dev with plan-owned scratch (same results,
 *                               same launches);
 *   even, up to 2^30 - 2 ("halved")   Bluestein of L = n/2 over z[m] = x[2m] + i x[2m+1], then the r2c untangle with W_n^k,
 *                               M = 2^ceil(log2(n - 1)); c2r runs the library's c2r pre-processing with W_n^m into the inverse;
 *   odd, up to 2^29 - 1 ("direct")    Bluestein of L = n on the real input, M = 2^ceil(log2(2n - 1)); also n = 1 (and n = 2,
 *                               halved), with M = 4.
 * The Bluestein paths run CHIRP-PRE-R2C / CHIRP-POST-R2C (CHIRP-PRE-C2R / CHIRP-POST-C2R) around the two M-point transforms
 * and CHIRP-MUL of the complex any-length plan.  Any other n returns PHASTFT_ERR_INVALID_ARG at create, before the device is
 * touched.
 * phastft_plan_r2c_any_*_create_with(n, device, algo, out) selects the algorithm of the halved and direct paths with the
 * PHASTFT_ANY_* values of the complex plan (powers of two take the r2c plan under every value; _create builds Bluestein):
 *   PHASTFT_ANY_MIXED   the mixed-radix path of L = n/2 (halved, even n up to 2^31 - 2) or of L = n (direct, odd n = Q_a * Q_b
 *                       <= 729^2): SMOOTH-PRE-R2C loads the pairs (or the reals) into the workspace, the P-point plan and the ODD
 *                       passes transform it; the halved r2c stores Z = DFT_L(z) into the bins and SMOOTH-POST-R2C untangles them
 *                       in place with W_n^k, the direct r2c's last pass (ODD-R2C) stores bins 0 .. floor(n/2) only.  c2r loads
 *                       the c2r pre-processing with W_n^m (halved) or the Hermitian extension (direct) in SMOOTH-PRE-C2R, and the
 *                       last pass (ODD-C2R) stores the pairs (y[2k], y[2k+1]) or the real part.  No padding.  An n whose L is
 *                       not eligible for phastft_any_mixed_factorization returns PHASTFT_ERR_INVALID_ARG (the detail names L or
 *                       n and the reason) before the device is touched.
 *   PHASTFT_ANY_AUTO    mixed when L is eligible, Bluestein otherwise (an even n above 2^30 - 2 that is not eligible is refused).
 * describe(): "n=44100 f64 r2c any: halved, mixed 2^1 x 105 x 105 | inner: ..." or "n=1125 f64 r2c any: direct, mixed 2^0 x 25 x 45 |
 * inner: ...".
 * c2r of a spectrum that is not the half-spectrum of a real signal (non-real X[0], or for even n non-real X[n/2]): even n uses
 * the c2r pre-processing formula with W_n, as the power-of-two c2r does; odd n uses the Hermitian extension
 * Y[m] = conj X[n - m] (m > n/2) and keeps the real part of the inverse, so Im X[0] is dropped, as numpy.fft.irfft does.
 * For valid spectra both are the inverse real DFT. */
typedef struct phastft_plan_r2c_any_f64 phastft_plan_r2c_any_f64;
typedef struct phastft_plan_r2c_any_f32 phastft_plan_r2c_any_f32;
PHASTFT_API int32_t phastft_plan_r2c_any_f64_create(size_t n, int device, phastft_plan_r2c_any_f64** out);
PHASTFT_API int32_t phastft_plan_r2c_any_f32_create(size_t n, int device, phastft_plan_r2c_any_f32** out);
PHASTFT_API int32_t phastft_plan_r2c_any_f64_create_with(size_t n, int device, int algo, phastft_plan_r2c_any_f64** out);
PHASTFT_API int32_t phastft_plan_r2c_any_f32_create_with(size_t n, int device, int algo, phastft_plan_r2c_any_f32** out);
PHASTFT_API void phastft_plan_r2c_any_f64_destroy(phastft_plan_r2c_any_f64* plan);
PHASTFT_API void phastft_plan_r2c_any_f32_destroy(phastft_plan_r2c_any_f32* plan);
PHASTFT_API size_t phastft_plan_r2c_any_f64_size(const phastft_plan_r2c_any_f64* plan);
PHASTFT_API size_t phastft_plan_r2c_any_f32_size(const phastft_plan_r2c_any_f32* plan);
/* "n=44100 f64 r2c any: halved, Bluestein L=22050 M=2^16 | inner: ...", "n=1001 f64 r2c any: direct, Bluestein L=1001 M=2^11 |
 * inner: ..." or "n=2^20 f64 r2c any: power of two | <phastft_plan_r2c_f64_describe()>".  Valid until the thread's next call. */
PHASTFT_API const char* phastft_plan_r2c_any_f64_describe(const phastft_plan_r2c_any_f64* plan);
PHASTFT_API const char* phastft_plan_r2c_any_f32_describe(const phastft_plan_r2c_any_f32* plan);
/* Makes every allocation a call of `batch` members would make now, so such calls can be captured into a CUDA graph.  A call
 * that would allocate while its stream is being captured returns PHASTFT_ERR_INVALID_ARG. */
PHASTFT_API int32_t phastft_plan_r2c_any_f64_reserve(const phastft_plan_r2c_any_f64* plan, size_t batch);
PHASTFT_API int32_t phastft_plan_r2c_any_f32_reserve(const phastft_plan_r2c_any_f32* plan, size_t batch);
/* Device-resident, asynchronous on `stream`: member b reads n reals at d_input + b * in_stride and writes n/2 + 1 bins at
 * d_out_* + b * out_stride (c2r: the mirror).  in_stride >= n and out_stride >= n/2 + 1 (c2r: in_stride >= n/2 + 1, out_stride
 * >= n); for even n the real array's base must be aligned to 2 * sizeof(T) and its stride even (it is accessed as pairs).
 * NULL pointers and bad strides return PHASTFT_ERR_INVALID_ARG before any launch; batch == 0 launches nothing.  Allocates only
 * when the plan's workspace must grow (synchronising). */
PHASTFT_API int32_t phastft_r2c_any_f64_dev(const phastft_plan_r2c_any_f64* plan, const double* d_input, size_t in_stride,
                                            double* d_out_re, double* d_out_im, size_t out_stride, size_t batch, void* stream);
PHASTFT_API int32_t phastft_r2c_any_f32_dev(const phastft_plan_r2c_any_f32* plan, const float* d_input, size_t in_stride,
                                            float* d_out_re, float* d_out_im, size_t out_stride, size_t batch, void* stream);
PHASTFT_API int32_t phastft_c2r_any_f64_dev(const phastft_plan_r2c_any_f64* plan, const double* d_in_re, const double* d_in_im,
                                            size_t in_stride, double* d_output, size_t out_stride, size_t batch, void* stream);
PHASTFT_API int32_t phastft_c2r_any_f32_dev(const phastft_plan_r2c_any_f32* plan, const float* d_in_re, const float* d_in_im,
                                            size_t in_stride, float* d_output, size_t out_stride, size_t batch, void* stream);
/* Host slices, synchronous, with the length codes of phastft_{r2c,c2r}_*_host (N/2 + 1 meaning floor(n/2) + 1). */
PHASTFT_API int32_t phastft_r2c_any_f64_host(const phastft_plan_r2c_any_f64* plan, const double* input, size_t len_in,
                                             double* out_re, size_t len_ore, double* out_im, size_t len_oim);
PHASTFT_API int32_t phastft_r2c_any_f32_host(const phastft_plan_r2c_any_f32* plan, const float* input, size_t len_in,
                                             float* out_re, size_t len_ore, float* out_im, size_t len_oim);
PHASTFT_API int32_t phastft_c2r_any_f64_host(const phastft_plan_r2c_any_f64* plan, const double* in_re, size_t len_ire,
                                             const double* in_im, size_t len_iim, double* output, size_t len_out);
PHASTFT_API int32_t phastft_c2r_any_f32_host(const phastft_plan_r2c_any_f32* plan, const float* in_re, size_t len_ire,
                                             const float* in_im, size_t len_iim, float* output, size_t len_out);
/* The same transforms with the spectrum as floor(n/2) + 1 interleaved (re, im) values (torch.fft.rfft / irfft(n=n),
 * std::complex<T>, num_complex::Complex<T>): member b's bins start at complex element b * stride_complex of d_out / d_in
 * (>= floor(n/2) + 1), a pointer aligned to 2 * sizeof(T) (a member may start at an odd complex offset); the real side keeps the
 * rules above.  Forward unscaled, c2r scaled by 1/n, c2r never writes its input and drops Im X[0] for odd n, as the planar calls.
 * Every path runs the planar call's launches with the spectrum's end kernels in interleaved modes (the power of two's last pass
 * stores Z interleaved, then R2C-UNTANGLE-IL; its c2r reads the bins in the first pass (launch mode c2r-in-il) or in C2R-PRE-IL;
 * CHIRP-POST-R2C-IL / CHIRP-PRE-C2R-IL; ODD-IL + SMOOTH-POST-R2C-IL, ODD-R2C-IL, SMOOTH-PRE-C2R-IL) and gives the planar call's
 * results bit for bit.  NULL or misaligned pointers and short or odd strides return PHASTFT_ERR_INVALID_ARG before any launch;
 * batch == 0, workspace growth, reserve() and graph capture as in the planar calls.  The host forms use the planar host length
 * codes (r2c: input PHASTFT_ERR_INPUT_LEN, spectrum PHASTFT_ERR_OUTPUT_RE_LEN; c2r: spectrum PHASTFT_ERR_INPUT_RE_LEN, output
 * PHASTFT_ERR_OUTPUT_LEN, lengths of the spectrum in complex values) and stage through a plan-owned buffer their first call
 * allocates. */
PHASTFT_API int32_t phastft_r2c_interleaved_any_f64_dev(const phastft_plan_r2c_any_f64* plan, const double* d_input, size_t in_stride,
                                                        double* d_out, size_t out_stride_complex, size_t batch, void* stream);
PHASTFT_API int32_t phastft_r2c_interleaved_any_f32_dev(const phastft_plan_r2c_any_f32* plan, const float* d_input, size_t in_stride,
                                                        float* d_out, size_t out_stride_complex, size_t batch, void* stream);
PHASTFT_API int32_t phastft_c2r_interleaved_any_f64_dev(const phastft_plan_r2c_any_f64* plan, const double* d_in, size_t in_stride_complex,
                                                        double* d_output, size_t out_stride, size_t batch, void* stream);
PHASTFT_API int32_t phastft_c2r_interleaved_any_f32_dev(const phastft_plan_r2c_any_f32* plan, const float* d_in, size_t in_stride_complex,
                                                        float* d_output, size_t out_stride, size_t batch, void* stream);
PHASTFT_API int32_t phastft_r2c_interleaved_any_f64_host(const phastft_plan_r2c_any_f64* plan, const double* input, size_t len_in,
                                                         double* out, size_t len_out_complex);
PHASTFT_API int32_t phastft_r2c_interleaved_any_f32_host(const phastft_plan_r2c_any_f32* plan, const float* input, size_t len_in,
                                                         float* out, size_t len_out_complex);
PHASTFT_API int32_t phastft_c2r_interleaved_any_f64_host(const phastft_plan_r2c_any_f64* plan, const double* in, size_t len_in_complex,
                                                         double* output, size_t len_out);
PHASTFT_API int32_t phastft_c2r_interleaved_any_f32_host(const phastft_plan_r2c_any_f32* plan, const float* in, size_t len_in_complex,
                                                         float* output, size_t len_out);

/* ---- discrete cosine and sine transforms, types 2 and 3, of any length (scipy.fft.dct / dst) ----------------------------
 * kind, with N = n and scipy.fft's definitions (norm "backward"):
 *   PHASTFT_R2R_DCT2  y[k] = 2 sum_n x[n] cos(pi k (2n + 1) / 2N)
 *   PHASTFT_R2R_DCT3  y[k] = x[0] + 2 sum_{n >= 1} x[n] cos(pi n (2k + 1) / 2N)
 *   PHASTFT_R2R_DST2  y[k] = 2 sum_n x[n] sin(pi (k + 1)(2n + 1) / 2N)
 *   PHASTFT_R2R_DST3  y[k] = (-1)^k x[N-1] + 2 sum_{n < N-1} x[n] sin(pi (n + 1)(2k + 1) / 2N)
 * norm: PHASTFT_NORM_BACKWARD (as above), PHASTFT_NORM_ORTHO (scaled by 1/sqrt(2N), with scipy's orthogonalize=True: output 0
 * of DCT-II / input 0 of DCT-III scaled by 1/sqrt(2) / sqrt(2), element N-1 for the DSTs), PHASTFT_NORM_FORWARD (1/(2N)).
 * scipy's idct / idst of type t and norm m is kind t' = 5 - t with the inverse norm (backward <-> forward, ortho itself).
 * Each call runs DCT-PRE-<kind>, the inner real plan's interleaved r2c (types 2) or c2r (types 3) on the plan's workspace, and
 * DCT-POST-<kind>.  _create_with takes PHASTFT_ANY_* and has the limits and refusals of phastft_plan_r2c_any_*_create_with;
 * describe() is "n=<N> <prec> dct | " followed by the inner real plan's describe().
 * _dev: member b reads N reals at d_in + b * in_stride and writes N reals at d_out + b * out_stride; any strides >= N and any
 * element offsets (the caller's arrays are accessed one element at a time), d_out == d_in with equal strides transforms in
 * place.  A bad kind or norm, NULL pointers and short strides return PHASTFT_ERR_INVALID_ARG before any launch; batch == 0 does
 * nothing.  The workspace follows the any-length plans' protocol: it grows outside a stream capture only (a capture that would
 * need it to grow returns PHASTFT_ERR_INVALID_ARG; _reserve(batch) grows it and the inner plan's beforehand), and a call on
 * another stream waits for the previous one.
 * _host: synchronous, through a plan-owned staging buffer (allocated by the first host call); len_in != N is
 * PHASTFT_ERR_INPUT_LEN, len_out != N PHASTFT_ERR_OUTPUT_LEN; in may equal out. */
#define PHASTFT_R2R_DCT2 0
#define PHASTFT_R2R_DCT3 1
#define PHASTFT_R2R_DST2 2
#define PHASTFT_R2R_DST3 3
#define PHASTFT_NORM_BACKWARD 0
#define PHASTFT_NORM_ORTHO 1
#define PHASTFT_NORM_FORWARD 2
typedef struct phastft_plan_dct_f64 phastft_plan_dct_f64;
typedef struct phastft_plan_dct_f32 phastft_plan_dct_f32;
PHASTFT_API int32_t phastft_plan_dct_f64_create_with(size_t n, int device, int algo, phastft_plan_dct_f64** out);
PHASTFT_API int32_t phastft_plan_dct_f32_create_with(size_t n, int device, int algo, phastft_plan_dct_f32** out);
PHASTFT_API void phastft_plan_dct_f64_destroy(phastft_plan_dct_f64* plan);
PHASTFT_API void phastft_plan_dct_f32_destroy(phastft_plan_dct_f32* plan);
PHASTFT_API size_t phastft_plan_dct_f64_size(const phastft_plan_dct_f64* plan);
PHASTFT_API size_t phastft_plan_dct_f32_size(const phastft_plan_dct_f32* plan);
PHASTFT_API const char* phastft_plan_dct_f64_describe(const phastft_plan_dct_f64* plan);
PHASTFT_API const char* phastft_plan_dct_f32_describe(const phastft_plan_dct_f32* plan);
PHASTFT_API int32_t phastft_plan_dct_f64_reserve(const phastft_plan_dct_f64* plan, size_t batch);
PHASTFT_API int32_t phastft_plan_dct_f32_reserve(const phastft_plan_dct_f32* plan, size_t batch);
PHASTFT_API int32_t phastft_dct_f64_dev(const phastft_plan_dct_f64* plan, int kind, int norm, const double* d_in, size_t in_stride,
                                        double* d_out, size_t out_stride, size_t batch, void* stream);
PHASTFT_API int32_t phastft_dct_f32_dev(const phastft_plan_dct_f32* plan, int kind, int norm, const float* d_in, size_t in_stride,
                                        float* d_out, size_t out_stride, size_t batch, void* stream);
PHASTFT_API int32_t phastft_dct_f64_host(const phastft_plan_dct_f64* plan, int kind, int norm, const double* in, size_t len_in,
                                         double* out, size_t len_out);
PHASTFT_API int32_t phastft_dct_f32_host(const phastft_plan_dct_f32* plan, int kind, int norm, const float* in, size_t len_in,
                                         float* out, size_t len_out);

/* ---- linear convolution and cross-correlation of real or complex signals of any lengths (scipy.signal) --------------------
 * op PHASTFT_CONV_CONVOLVE: scipy.signal.fftconvolve(x, h, mode); PHASTFT_CONV_CORRELATE: scipy.signal.correlate(x, h, mode),
 * i.e. convolution with conj(h reversed).  Windows of the full convolution y[j] = sum_k x[k] h[j - k], 0 <= j < n_x + n_h - 1:
 *   PHASTFT_CONV_FULL   start 0,                    length n_x + n_h - 1
 *   PHASTFT_CONV_SAME   start (n_h - 1) / 2,        length n_x
 *   PHASTFT_CONV_VALID  start min(n_x, n_h) - 1,    length |n_x - n_h| + 1
 * phastft_conv_out_len gives that length (0 for a bad mode or a zero length).
 * _create: domain PHASTFT_CONV_REAL or PHASTFT_CONV_COMPLEX; the plan transforms at L = 2^ceil(log2(n_x + n_h - 1)), at least
 * 4 (_fft_len), on the real any-length plan (interleaved r2c / c2r) or the complex one (interleaved forward / reverse).  n_x or
 * n_h of 0, a bad domain, or L above 2^31 (real) / 2^30 (complex) return PHASTFT_ERR_INVALID_ARG before the device is touched.
 * describe() is "n_x=<n_x> n_h=<n_h> <prec> conv <real|complex> L=2^<k> | " followed by the inner plan's describe().
 * Each call runs CONV-PRE over the B signals and H filters (H = B, or 1 when h_stride == 0 or B == 1), the inner forward
 * transform of those B + H members, CONV-MUL and the inverse on the B signals, and CONV-POST; the inverse's 1/L is the only
 * scale.
 * _dev: member b reads n_x values at d_x + b * x_stride and n_h at d_h + b * h_stride (h_stride 0: one filter for every member)
 * and writes the window at d_y + b * y_stride.  Real values: any element offsets.  Complex values: interleaved (re, im) pairs,
 * strides in complex values, pointers aligned to 2 * sizeof(T).  d_y may equal d_x or d_h.  With batch > 1, x_stride < n_x,
 * y_stride < the output length, or h_stride neither 0 nor >= n_h; NULL or misaligned pointers; or a bad op or mode return
 * PHASTFT_ERR_INVALID_ARG before any launch; batch == 0 does nothing.  The workspace follows the any-length plans' protocol:
 * it grows outside a stream capture only (_reserve(batch) grows it and the inner plan's for `batch` pairwise members), and a
 * call on another stream waits for the previous one.
 * _host: synchronous, through a plan-owned staging buffer (allocated by the first host call); lengths in values (complex
 * ones for the complex domain): len_x != n_x or len_h != n_h is PHASTFT_ERR_INPUT_LEN, len_y != the output length
 * PHASTFT_ERR_OUTPUT_LEN. */
#define PHASTFT_CONV_REAL 0
#define PHASTFT_CONV_COMPLEX 1
#define PHASTFT_CONV_CONVOLVE 0
#define PHASTFT_CONV_CORRELATE 1
#define PHASTFT_CONV_FULL 0
#define PHASTFT_CONV_SAME 1
#define PHASTFT_CONV_VALID 2
typedef struct phastft_plan_conv_f64 phastft_plan_conv_f64;
typedef struct phastft_plan_conv_f32 phastft_plan_conv_f32;
PHASTFT_API size_t phastft_conv_out_len(size_t n_x, size_t n_h, int mode);
PHASTFT_API int32_t phastft_plan_conv_f64_create(size_t n_x, size_t n_h, int domain, int device, phastft_plan_conv_f64** out);
PHASTFT_API int32_t phastft_plan_conv_f32_create(size_t n_x, size_t n_h, int domain, int device, phastft_plan_conv_f32** out);
PHASTFT_API void phastft_plan_conv_f64_destroy(phastft_plan_conv_f64* plan);
PHASTFT_API void phastft_plan_conv_f32_destroy(phastft_plan_conv_f32* plan);
PHASTFT_API size_t phastft_plan_conv_f64_fft_len(const phastft_plan_conv_f64* plan);
PHASTFT_API size_t phastft_plan_conv_f32_fft_len(const phastft_plan_conv_f32* plan);
PHASTFT_API const char* phastft_plan_conv_f64_describe(const phastft_plan_conv_f64* plan);
PHASTFT_API const char* phastft_plan_conv_f32_describe(const phastft_plan_conv_f32* plan);
PHASTFT_API int32_t phastft_plan_conv_f64_reserve(const phastft_plan_conv_f64* plan, size_t batch);
PHASTFT_API int32_t phastft_plan_conv_f32_reserve(const phastft_plan_conv_f32* plan, size_t batch);
PHASTFT_API int32_t phastft_conv_f64_dev(const phastft_plan_conv_f64* plan, int op, int mode, const double* d_x, size_t x_stride,
                                         const double* d_h, size_t h_stride, double* d_y, size_t y_stride, size_t batch, void* stream);
PHASTFT_API int32_t phastft_conv_f32_dev(const phastft_plan_conv_f32* plan, int op, int mode, const float* d_x, size_t x_stride,
                                         const float* d_h, size_t h_stride, float* d_y, size_t y_stride, size_t batch, void* stream);
PHASTFT_API int32_t phastft_conv_f64_host(const phastft_plan_conv_f64* plan, int op, int mode, const double* x, size_t len_x,
                                          const double* h, size_t len_h, double* y, size_t len_y);
PHASTFT_API int32_t phastft_conv_f32_host(const phastft_plan_conv_f32* plan, int op, int mode, const float* x, size_t len_x,
                                          const float* h, size_t len_h, float* y, size_t len_y);

/* ---- short-time Fourier transform and its inverse of real or complex signals (torch.stft / torch.istft) -------------------
 * The semantics of torch.stft(x, n_fft, hop, win_length, window, center, pad_mode, normalized, return_complex=True) and
 * torch.istft(spec, n_fft, hop, win_length, window, center, normalized, length=n) for signals of n values.
 * _create: `window` is win_length host values (NULL: ones), zero-padded to n_fft from (n_fft - win_length) / 2 and kept on the
 * device in the plan's precision.  center pads n_fft / 2 values on each side, by reflection (PHASTFT_STFT_PAD_REFLECT) or
 * zeros (PHASTFT_STFT_PAD_CONSTANT).  F = 1 + (n + 2 pad - n_fft) / hop frames (_frames) of n_fft / 2 + 1 bins (domain
 * PHASTFT_STFT_REAL) or n_fft bins (PHASTFT_STFT_COMPLEX) (_bins), on the n_fft-point real or complex any-length plan
 * (PHASTFT_ANY_AUTO).  n or n_fft of 0, hop == 0, win_length of 0 or above n_fft, reflect padding with n_fft / 2 >= n, n <
 * n_fft without center, a bad pad mode or domain, and anything the inner plan refuses return PHASTFT_ERR_INVALID_ARG before the
 * device is touched.  _create also runs torch's NOLA check in long double (the window-squared overlap-add envelope >= 1e-11
 * over every retained sample some frame covers) and records the result: the STFT always runs; the istft of a failing plan
 * returns PHASTFT_ERR_INVALID_ARG naming the first failing sample.
 * describe() is "n=<n> n_fft=<n_fft> hop=<hop> <prec> stft <real|complex> F=<F> | " followed by the inner plan's describe().
 * _dev: member b's n values at d_x (d_y) + b * x_stride (y_stride); frame f of member b at d_spec + (b * F + f) * frame_stride
 * complex values (torch's layout; frame_stride >= the bin count).  Real signals: any element offsets; complex ones: interleaved
 * pairs, strides in complex values.  d_spec (and complex signals) aligned to 2 * sizeof(T).  normalized other than 0 / 1, NULL
 * or misaligned pointers, a short frame_stride, x_stride / y_stride < n with batch > 1, or d_spec's frames overlapping the
 * signals return PHASTFT_ERR_INVALID_ARG before any launch; batch == 0 does nothing.  The stft writes no value between frames;
 * the istft never writes d_spec and writes zero where no frame covers a sample (torch's tail).  Launches: STFT-FRAME, then the
 * inner forward launches over batch x F frames; the inner inverse launches, then ISTFT-OLA (complex: a strided device copy of
 * the frames into the workspace comes first).  The workspace follows the any-length plans' protocol (_reserve(batch) grows it
 * and the inner plan's for batch x F frames; capturing without it fails naming phastft_plan_stft_*_reserve).
 * _host: synchronous through a plan-owned staging buffer; dense frames (F x bins complex values); len_x / len_spec (stft) or
 * len_spec (istft) wrong is PHASTFT_ERR_INPUT_LEN, the output length wrong PHASTFT_ERR_OUTPUT_LEN. */
#define PHASTFT_STFT_REAL 0
#define PHASTFT_STFT_COMPLEX 1
#define PHASTFT_STFT_PAD_REFLECT 0
#define PHASTFT_STFT_PAD_CONSTANT 1
typedef struct phastft_plan_stft_f64 phastft_plan_stft_f64;
typedef struct phastft_plan_stft_f32 phastft_plan_stft_f32;
PHASTFT_API int32_t phastft_plan_stft_f64_create(size_t n, size_t n_fft, size_t hop, const double* window, size_t win_length, int center,
                                                 int pad_mode, int domain, int device, phastft_plan_stft_f64** out);
PHASTFT_API int32_t phastft_plan_stft_f32_create(size_t n, size_t n_fft, size_t hop, const float* window, size_t win_length, int center,
                                                 int pad_mode, int domain, int device, phastft_plan_stft_f32** out);
PHASTFT_API void phastft_plan_stft_f64_destroy(phastft_plan_stft_f64* plan);
PHASTFT_API void phastft_plan_stft_f32_destroy(phastft_plan_stft_f32* plan);
PHASTFT_API size_t phastft_plan_stft_f64_frames(const phastft_plan_stft_f64* plan);
PHASTFT_API size_t phastft_plan_stft_f32_frames(const phastft_plan_stft_f32* plan);
PHASTFT_API size_t phastft_plan_stft_f64_bins(const phastft_plan_stft_f64* plan);
PHASTFT_API size_t phastft_plan_stft_f32_bins(const phastft_plan_stft_f32* plan);
PHASTFT_API const char* phastft_plan_stft_f64_describe(const phastft_plan_stft_f64* plan);
PHASTFT_API const char* phastft_plan_stft_f32_describe(const phastft_plan_stft_f32* plan);
PHASTFT_API int32_t phastft_plan_stft_f64_reserve(const phastft_plan_stft_f64* plan, size_t batch);
PHASTFT_API int32_t phastft_plan_stft_f32_reserve(const phastft_plan_stft_f32* plan, size_t batch);
PHASTFT_API int32_t phastft_stft_f64_dev(const phastft_plan_stft_f64* plan, int normalized, const double* d_x, size_t x_stride, double* d_spec,
                                         size_t frame_stride, size_t batch, void* stream);
PHASTFT_API int32_t phastft_stft_f32_dev(const phastft_plan_stft_f32* plan, int normalized, const float* d_x, size_t x_stride, float* d_spec,
                                         size_t frame_stride, size_t batch, void* stream);
PHASTFT_API int32_t phastft_istft_f64_dev(const phastft_plan_stft_f64* plan, int normalized, const double* d_spec, size_t frame_stride,
                                          double* d_y, size_t y_stride, size_t batch, void* stream);
PHASTFT_API int32_t phastft_istft_f32_dev(const phastft_plan_stft_f32* plan, int normalized, const float* d_spec, size_t frame_stride,
                                          float* d_y, size_t y_stride, size_t batch, void* stream);
PHASTFT_API int32_t phastft_stft_f64_host(const phastft_plan_stft_f64* plan, int normalized, const double* x, size_t len_x, double* spec,
                                          size_t len_spec);
PHASTFT_API int32_t phastft_stft_f32_host(const phastft_plan_stft_f32* plan, int normalized, const float* x, size_t len_x, float* spec,
                                          size_t len_spec);
PHASTFT_API int32_t phastft_istft_f64_host(const phastft_plan_stft_f64* plan, int normalized, const double* spec, size_t len_spec,
                                           double* y, size_t len_y);
PHASTFT_API int32_t phastft_istft_f32_host(const phastft_plan_stft_f32* plan, int normalized, const float* spec, size_t len_spec,
                                           float* y, size_t len_y);

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
