// phastft_cuda.cu -- planner, launcher and C ABI of libphastft_cuda.so (see include/phastft_cuda.h).
//
// Reference items replaced (QuState/PhastFT @ 8cd3a39, paths under the reference's src/):
//   planner.rs:34-114   PlannerDit{64,32}: per-stage cos/sin tables, total 2(N-64) entries
//        -> Plan<T>: pass decomposition N = R_1*R_2[*R_3], a two-level W_N table (2*sqrt(N)
//           f64 entries) for the inter-pass twiddles and one W_R table per pass
//   planner.rs:164-212  PlannerR2c{64,32}                      -> PlanR2c<T>
//   algorithms/dit.rs:263-401 fft_*_dit_with_planner_and_opts  -> run_c2c(): 1-3 kernel launches
//   algorithms/r2c.rs:521-895 r2c / c2r entry points            -> r2c_dev() / c2r_dev()
//   options.rs:10-43    Options                                 -> accepted, no effect on the GPU
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <algorithm>
#include <functional>
#include <thread>
#include <type_traits>
#include <vector>

#include "../../include/phastft_cuda.h"
#include "registry.h"

using namespace phast;

// =================================================================================================
// errors
// =================================================================================================
namespace {

thread_local std::string g_last_error;
std::atomic<uint64_t> g_launches{0};

int32_t fail(int32_t code, const std::string& detail = std::string()) {
    g_last_error = phastft_status_message(code);
    if (!detail.empty()) { g_last_error += ": "; g_last_error += detail; }
    return code;
}

// The kernels the calling thread's most recent execution call launched (phastft_last_launches): one record per launch,
// appended where the launch is made and cleared at the start of every public execution entry point.
struct LaunchRec {
    const char* kind;    // COL / TRANS / ROW, CLUSTER, PIPE, or an elementwise r2c / c2r kernel
    int R, R2, C, NT, variant;   // R2: second pass size of the one-launch pairs (CLUSTER, PIPE), else 0
    const char* mode;    // plain / tma / bulk / row-bulk / c2r-in / cluster / pipe
    bool pdl;            // launched with programmatic dependent launch (PHASTFT_PDL=1)
};
thread_local std::vector<LaunchRec> g_launch_log;
thread_local std::string g_launch_text;
thread_local std::string g_r2c_desc_text;   // phastft_plan_r2c_*_describe: built per call (it reads the environment)

// PHASTFT_SCRIBBLE=1, read when a plan is built: the plan's scratch (workspaces, c2r scratch, host staging) is filled with 0xFF
// bytes, a NaN in f32 and f64, when it is allocated and, on the call's stream, before each call uses it.  A kernel that reads
// scratch before writing it in the same call then produces NaN instead of what the previous call left there.  Constant tables
// are never touched.  phastft_last_scribble_bytes() reports the bytes the calling thread's most recent call poisoned.
thread_local uint64_t g_scribble_bytes = 0;
bool scribble_env() {
    const char* e = getenv("PHASTFT_SCRIBBLE");
    return e && atoi(e) != 0;
}

// PHASTFT_GRID_BLOCKS_MAX, read on every call: the most blocks one launch of a member-major elementwise kernel may have before
// the call splits it into several launches (2^31 - 1, gridDim.x's limit, when unset, not a number, <= 0 or above that).  A
// lower value makes the splits that otherwise need more than 2^31 - 1 blocks run at small sizes, so tests can reach them.
size_t grid_blocks_max() {
    constexpr long long limit = 0x7fffffff;
    if (const char* e = getenv("PHASTFT_GRID_BLOCKS_MAX")) {
        char* end = nullptr;
        const long long v = strtoll(e, &end, 10);
        if (end != e && *end == '\0' && v > 0 && v <= limit) return (size_t)v;
    }
    return (size_t)limit;
}

// before a call's first use of [p, p + bytes), ordered on `stream` (a graph node while the stream is being captured)
cudaError_t scribble(bool on, void* p, size_t bytes, cudaStream_t stream) {
    if (!on || !p || !bytes) return cudaSuccess;
    g_scribble_bytes += bytes;
    return cudaMemsetAsync(p, 0xFF, bytes, stream);
}
// a buffer just allocated: done before any stream can use it
cudaError_t scribble_new(bool on, void* p, size_t bytes) {
    if (!on || !p || !bytes) return cudaSuccess;
    g_scribble_bytes += bytes;
    cudaError_t e = cudaMemset(p, 0xFF, bytes);
    return e == cudaSuccess ? cudaDeviceSynchronize() : e;
}

void launches_reset() { g_launch_log.clear(); g_scribble_bytes = 0; }
void note_launch(const LaunchRec& r) {
    g_launch_log.push_back(r);
    g_launches.fetch_add(1, std::memory_order_relaxed);
}
const char* mode_name(int mode) {
    switch (mode) {
        case MODE_TMA_IN: return "tma";
        case MODE_BULK_IN: return "bulk";
        case MODE_ROW_BULK: return "row-bulk";
        case MODE_C2R_IN: return "c2r-in";
        case MODE_C2R_IN_IL: return "c2r-in-il";
        default: return "plain";
    }
}

#define CUDA_TRY(expr)                                                                                  \
    do {                                                                                                \
        cudaError_t _e = (expr);                                                                        \
        if (_e != cudaSuccess) {                                                                        \
            int32_t _code = (_e == cudaErrorNoDevice || _e == cudaErrorInsufficientDriver ||            \
                             _e == cudaErrorInvalidDevice)                                              \
                                ? PHASTFT_ERR_NO_DEVICE                                                 \
                                : PHASTFT_ERR_CUDA;                                                     \
            (void)cudaGetLastError(); /* clear it: the next kernel-launch check must not see a stale error */ \
            return fail(_code, std::string(#expr) + " -> " + cudaGetErrorString(_e));                   \
        }                                                                                               \
    } while (0)

inline bool is_pow2(size_t n) { return n != 0 && (n & (n - 1)) == 0; }
inline int ilog2(size_t n) { int l = 0; while (n >>= 1) ++l; return l; }

struct DeviceGuard {
    int prev = -1;
    bool ok = false;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        ok = cudaSetDevice(dev) == cudaSuccess;
    }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};


// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda)
typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
encode_tiled_fn tensor_map_encoder() {
    static encode_tiled_fn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) p = nullptr;
        (void)cudaGetLastError();
        return reinterpret_cast<encode_tiled_fn>(p);
    }();
    return fn;
}
// {cols (contiguous), rows (stride row_stride elements), batch (stride bstride elements)} of T; box {box_cols, box_rows, 1}
template <typename T>
bool encode_tile_map(CUtensorMap* map, const T* base, size_t cols, size_t rows, size_t row_stride, size_t batch, size_t bstride,
                     unsigned box_cols, unsigned box_rows) {
    encode_tiled_fn enc = tensor_map_encoder();
    if (!enc) return false;
    if ((reinterpret_cast<uintptr_t>(base) & 15) || ((row_stride * sizeof(T)) & 15) || ((bstride * sizeof(T)) & 15)) return false;
    cuuint64_t dims[3] = {cols, rows, batch};
    cuuint64_t strides[2] = {row_stride * sizeof(T), bstride * sizeof(T)};
    if (batch == 1) strides[1] = strides[0] * rows;      // unused dimension: any legal stride
    cuuint32_t box[3] = {box_cols, box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    const CUtensorMapDataType dt = sizeof(T) == 8 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT64 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    return enc(map, dt, 3, const_cast<T*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// =================================================================================================
// kernel registry (the kernels themselves are instantiated in reg_strided.cu / reg_row.cu / reg_multi.cu)
// =================================================================================================
template <typename T>
const std::vector<KernelEntry<T>>& registry() {
    static const std::vector<KernelEntry<T>> reg = [] {
        std::vector<KernelEntry<T>> v;
        add_row_kernels<T>(v);                       // whole transform in one CTA (rows contiguous in and out)
        add_strided_kernels<T, KIND_COL>(v);         // first / middle passes
        add_strided_kernels<T, KIND_TRANS>(v);       // last pass
        add_c2r_il_kernels<T>(v);                    // the interleaved-spectrum twins of the first passes' c2r builds
        return v;
    }();
    return reg;
}

const char* kind_name(int k) { return k == KIND_COL ? "COL" : k == KIND_TRANS ? "TRANS" : "ROW"; }

// =================================================================================================
// twiddle generation (host, extended precision, octant-reduced so symmetric entries are exact)
// =================================================================================================
void root_of_unity(uint64_t k, uint64_t n, double& re, double& im) {
    // W_n^k = exp(-2*pi*i*k/n), n a power of two
    k &= (n - 1);
    if (n < 8) {
        // n in {1, 2, 4}
        static const double c4[4] = {1, 0, -1, 0}, s4[4] = {0, -1, 0, 1};
        uint64_t q = k * (4 / n);
        re = c4[q]; im = s4[q];
        return;
    }
    const uint64_t eighth = n / 8;
    const uint64_t oct = k / eighth, rem = k % eighth;
    auto cs = [&](uint64_t j, long double& c, long double& s) {
        if (j == 0) { c = 1.0L; s = 0.0L; return; }
        if (j == eighth) { c = s = 0.70710678118654752440084436210484903928L; return; }
        long double a = 2.0L * 3.14159265358979323846264338327950288L * (long double)j / (long double)n;
        c = cosl(a); s = sinl(a);
    };
    long double c, s, co, si;
    switch (oct) {
        case 0: cs(rem, c, s); co = c; si = s; break;
        case 1: cs(eighth - rem, c, s); co = s; si = c; break;
        case 2: cs(rem, c, s); co = -s; si = c; break;
        case 3: cs(eighth - rem, c, s); co = -c; si = s; break;
        case 4: cs(rem, c, s); co = -c; si = -s; break;
        case 5: cs(eighth - rem, c, s); co = -s; si = -c; break;
        case 6: cs(rem, c, s); co = s; si = -c; break;
        default: cs(eighth - rem, c, s); co = c; si = -s; break;
    }
    re = (double)co;
    im = (double)(-si);
    if (re == 0.0) re = 0.0;
    if (im == 0.0) im = 0.0;
}

// W_n^k = exp(-2*pi*i*k/n) for any n >= 1 (k * 8 < 2^64): root_of_unity's octant reduction, with the octant found in integers
// from 8k = oct * n + rem, so the angle left for cosl / sinl is (pi/4) * rem / n or (pi/4) * (n - rem) / n.
void root_of_unity_any(uint64_t k, uint64_t n, double& re, double& im) {
    k %= n;
    const uint64_t oct = 8 * k / n, rem = 8 * k % n;
    auto cs = [&](uint64_t j, long double& c, long double& s) {
        if (j == 0) { c = 1.0L; s = 0.0L; return; }
        if (j == n) { c = s = 0.70710678118654752440084436210484903928L; return; }
        long double a = 0.25L * 3.14159265358979323846264338327950288L * (long double)j / (long double)n;
        c = cosl(a); s = sinl(a);
    };
    long double c, s, co, si;
    switch (oct) {
        case 0: cs(rem, c, s); co = c; si = s; break;
        case 1: cs(n - rem, c, s); co = s; si = c; break;
        case 2: cs(rem, c, s); co = -s; si = c; break;
        case 3: cs(n - rem, c, s); co = -c; si = s; break;
        case 4: cs(rem, c, s); co = -c; si = -s; break;
        case 5: cs(n - rem, c, s); co = -s; si = -c; break;
        case 6: cs(rem, c, s); co = s; si = -c; break;
        default: cs(n - rem, c, s); co = c; si = -s; break;
    }
    re = (double)co;
    im = (double)(-si);
    if (re == 0.0) re = 0.0;
    if (im == 0.0) im = 0.0;
}

// =================================================================================================
// plans
// =================================================================================================
constexpr int MAX_PASSES = 3;

// First 256 bytes of a plan's table blob: what the rest of the blob was laid out for.  Offsets and the W_L^(c*m)
// tables depend on the pass decomposition and on each pass's kernel (tile width, first radix), which can differ
// between ranks (PlannerMode::Tune, PHASTFT_* overrides): import / broadcast compare headers first.
constexpr size_t BLOB_HEADER_BYTES = 256;
struct BlobHeader {
    uint64_t magic;        // "PASTHFT3" (3: blobs with radix-32 stage tables)
    uint64_t bytes;        // whole blob, header included
    uint64_t n;
    uint32_t precision_bits, num_passes;
    uint64_t layout_sig;   // FNV-1a of the plan description (factors, kernels, radices, variants)
    uint64_t tw_stage_off[MAX_PASSES];   // per pass: byte offset of its W_R table
    uint64_t tw32_off[MAX_PASSES];       // ... and of its radix-32 stage table (PassDesc::tw32_off), 0 if it has none
};
static_assert(sizeof(BlobHeader) <= BLOB_HEADER_BYTES, "header fits its slot");
constexpr uint64_t BLOB_MAGIC = 0x3354464854534150ull;
inline uint64_t fnv1a(const std::string& str) {
    uint64_t h = 1469598103934665603ull;
    for (unsigned char c : str) { h ^= c; h *= 1099511628211ull; }
    return h;
}
constexpr int ALT_ROW_PASS = -1;   // launch_pass(): use Plan::alt_row

// A batch is processed in chunks so the workspace stays bounded.  Keeping a chunk's intermediate L2-resident was
// measured SLOWER than few large launches (4096 x 2^16 f32: L2-sized chunks, larger chunks and no chunking, fastest
// last), so the default chunk is as large as the workspace cap allows (PHASTFT_L2_CHUNK_MB overrides).
constexpr size_t L2_CHUNK_BYTES_DEFAULT = size_t(4) << 30;
// The pipelined launch's ring (PHASTFT_PIPE_RING_MB): 16 MiB is about a third of the H100's 50 MB L2, so the ring can stay
// resident beside the input and output streaming through (not measured).
constexpr long PIPE_RING_MB_DEFAULT = 16;

template <typename T>
struct PassDesc {
    const KernelEntry<T>* k = nullptr;    // kernel for a lone transform
    const KernelEntry<T>* kb = nullptr;   // kernel when the call carries many transforms (multi-wave grids)
    const KernelEntry<T>* kt = nullptr;   // 2-pass plans of lone transforms: the pass with an asynchronous (TMA) tile input
    const KernelEntry<T>* kc = nullptr;   // first pass only: `k` with the c2r pre-processing folded into its loads (MODE_C2R_IN)
    const KernelEntry<T>* kcb = nullptr;  // first pass only: the same build of `kb` (batched c2r)
    const KernelEntry<T>* kci = nullptr;  // kc and kcb reading interleaved bins (MODE_C2R_IN_IL): present wherever those are
    const KernelEntry<T>* kcbi = nullptr;
    const KernelEntry<T>* kr = nullptr;   // one-CTA plans: `kb` with its tile moved in and out by cp.async.bulk (MODE_ROW_BULK)
    size_t tw_wc_off_t = (size_t)-1;      // W_L^(c*m) table for `kt`
    size_t tw_im_off = (size_t)-1;        // one-CTA kernels: the per-stage [i][m] stage-twiddle tables for `k` ...
    size_t tw_im_off_b = (size_t)-1;      // ... and for `kb`
    int log2R = 0, log2A = 0, log2B = 0, log2R1 = 0, log2Rprev = 0, has_tw = 0, tw_shift = 0;
    size_t tw_stage_off = 0;  // byte offsets into the table blob
    size_t tw32_off = (size_t)-1;         // strided passes whose kernels end in a radix-32 stage: that stage's [m][i] = W_R^(m*i)
                                          // table (R values, filled on the device by stage32_table_kernel from the W_R table)
    size_t tw_wc_off = (size_t)-1;
    size_t tw_wc_off_b = (size_t)-1;      // same table for `kb` (depends on its C and first radix)
};

template <typename T>
struct Plan {
    size_t n = 0;
    int log2n = 0;
    int device = 0;
    int num_passes = 0;
    PassDesc<T> pass[MAX_PASSES];
    PassDesc<T> alt_row;               // multi-pass N that one CTA can hold (<= 128 KB): the one-CTA kernel, used for batches
    size_t alt_row_min_batch = 4;
    bool tma_lone = false;             // 2-pass plans: lone transforms through the asynchronous-input pair pass[].kt (PHASTFT_TMA=1)
    bool tma_batch = false;            // ... and batched calls (batch * N >= 2^21): the default where the pair exists (PHASTFT_TMA_BATCH=0 disables)
    const ClusterEntry<T>* cl = nullptr;   // both passes in ONE launch by a thread-block cluster (exchange through DSMEM)
    PassDesc<T> cl_pass[2];
    size_t cl_min_batch = 0;           // calls with at least this many transforms use the cluster launch
    int cl_max_active = 0;             // cudaOccupancyMaxActiveClusters of that launch on this device
    // 2-pass plans: both passes in one persistent launch, intermediates in an L2-resident ring (fft_pipe2_kernel)
    const PipeEntry<T>* pipe_b = nullptr;   // for batched calls (pairs pass[0].kb / pass[1].kb)
    const PipeEntry<T>* pipe_1 = nullptr;   // for a lone transform (pairs pass[0].k / pass[1].k); off unless PHASTFT_PIPE_LONE=1
    int pipe_grid_b = 0, pipe_grid_1 = 0;   // co-resident CTAs of those launches on this device
    mutable unsigned char* pipe_state = nullptr;   // ticket + done1[batch] + done2[batch], zeroed per call
    mutable size_t pipe_state_batch = 0;
    // table blob: [header][tw2_hi][tw2_lo][per pass W_R, [i][m] / radix-32 stage tables, wc]
    std::vector<unsigned char> blob_host;
    unsigned char* blob_dev = nullptr;
    size_t hi_off = 0, lo_off = 0;
    int lo_bits = 0;
    // workspace (multi-pass only) and host-API staging, grown lazily under `mu`
    mutable std::mutex mu;
    mutable std::mutex host_mu;         // held for a whole *_host call: staging buffers + the plan's streams are per plan
    mutable T* ws_re = nullptr;
    mutable T* ws_im = nullptr;
    mutable size_t ws_elems = 0;        // per array; ONE allocation of 2*ws_elems, ws_im = ws_re + ws_elems
    int ws_il = -1;                     // layout of the intermediates between passes: 0 planar, 1 interleaved
                                        // complex, -1 = interleaved for 3-pass plans and large batches (run_c2c)
    T* ws2_re = nullptr;                // 3-pass plans: L2-resident scratch for one k1 group (see run_c2c)
    T* ws2_im = nullptr;
    long long l2_group = 0;             // k1 values per group
    mutable T* stage_re = nullptr;      // host-API staging (N each, or 2N for interleaved in stage_re)
    mutable T* stage_im = nullptr;
    mutable size_t stage_elems = 0;
    mutable cudaStream_t stream = nullptr;   // used by the *_host entry points
    mutable cudaStream_t stream_h2d = nullptr;   // copy streams of the pipelined batch host path (created lazily)
    mutable cudaStream_t stream_d2h = nullptr;
    mutable cudaEvent_t ws_free = nullptr;   // orders workspace reuse across streams
    mutable cudaStream_t ws_last_stream = nullptr;
    mutable bool ws_used = false;
    // launch knobs, read when the plan is built like every other PHASTFT_* setting
    bool pdl = false;                   // PHASTFT_PDL=1: programmatic dependent launch of the passes
    size_t l2_chunk_bytes = 0;          // PHASTFT_L2_CHUNK_MB: signal bytes per chunk of a batched multi-pass call
    size_t pipe_ring_bytes = 0;         // PHASTFT_PIPE_RING_MB: workspace ring of the pipelined launch
    bool pipe_discard = true;           // PHASTFT_PIPE_DISCARD=0 keeps the ring's lines in L2 after pass 2 reads them
    bool scribble_on = false;           // PHASTFT_SCRIBBLE=1: NaN-fill the workspace and staging before each use (scribble())
    std::string description;

    ~Plan() {
        DeviceGuard g(device);
        if (blob_dev) cudaFree(blob_dev);
        if (ws_re) cudaFree(ws_re);
        if (pipe_state) cudaFree(pipe_state);
        if (ws2_re) cudaFree(ws2_re);
        if (ws2_im) cudaFree(ws2_im);
        if (stage_re) cudaFree(stage_re);
        if (stage_im) cudaFree(stage_im);
        if (ws_free) cudaEventDestroy(ws_free);
        if (stream) cudaStreamDestroy(stream);
        if (stream_h2d) cudaStreamDestroy(stream_h2d);
        if (stream_d2h) cudaStreamDestroy(stream_d2h);
    }
};

// Layout of the intermediates between passes: planar (two halves of the workspace) or interleaved
// complex.  Interleaved makes every access a 16-byte (f64) element, so a 64-byte run needs half as many
// columns: the 1024-row middle tile of 2^25..2^26 shrinks from 128 KB to 64 KB and two CTAs share an SM
// (faster on the 2^25..2^26 middle pass); streaming passes gain a few per cent, single L2-resident transforms lose a few
// per cent, hence the automatic rule.  PHASTFT_WS_IL=0|1 forces a layout.
inline int ws_interleaved_mode() {
    const char* e = getenv("PHASTFT_WS_IL");
    return e ? (atoi(e) != 0 ? 1 : 0) : -1;
}

// An explicit plan choice (PlannerMode::Tune tries several and keeps the fastest); consulted by
// choose_factors / pick_kernel before the heuristics, like the PHASTFT_FACTORS / PHASTFT_PASS_C env overrides.
struct PlanChoice {
    std::vector<int> factors;   // log2 of each pass size
    std::vector<int> pass_c;    // tile columns per pass (0 = heuristic)
};
thread_local const PlanChoice* g_choice = nullptr;

// pass sizes (log2) for a transform of 2^n points -------------------------------------------------
template <typename T>
std::vector<int> choose_factors(int n) {
    if (g_choice && !g_choice->factors.empty()) return g_choice->factors;
    // override: PHASTFT_FACTORS="20:10,10;26:9,9,8"  (applies to both precisions; tuning aid)
    if (const char* env = getenv("PHASTFT_FACTORS")) {
        std::string s(env);
        size_t pos = 0;
        while (pos < s.size()) {
            size_t end = s.find(';', pos);
            if (end == std::string::npos) end = s.size();
            std::string item = s.substr(pos, end - pos);
            size_t colon = item.find(':');
            if (colon != std::string::npos && atoi(item.substr(0, colon).c_str()) == n) {
                std::vector<int> f;
                int sum = 0;
                size_t p = colon + 1;
                while (p < item.size()) {
                    size_t q = item.find(',', p);
                    if (q == std::string::npos) q = item.size();
                    f.push_back(atoi(item.substr(p, q - p).c_str()));
                    sum += f.back();
                    p = q + 1;
                }
                if (sum == n && !f.empty() && (int)f.size() <= MAX_PASSES) return f;
            }
            pos = end + 1;
        }
    }
    // A lone transform is one CTA only while that beats two many-CTA passes (measured once the stage twiddles of the one-CTA
    // kernels became contiguous loads + products: up to 2^11 f64 / 2^13 f32).  Batches of <= 2^13 (f64) / 2^14 (f32) points always use a one-CTA
    // kernel (Plan::alt_row): one launch, one HBM round trip.
    const int single_max = sizeof(T) == 8 ? 11 : 13;
    if (n <= single_max) return {n};
    // two passes while both tiles stay <= 1024 points long; the ends of a 3-pass plan are kept at
    // 2^8 so they can use 128-byte runs in a 64 KB tile, the middle pass takes the rest (<= 2^10)
    // (measured-best splits)
    if (n <= 16) { int a = n / 2; return {a, n - a}; }
    if (n <= 20) { int a = (n + 1) / 2; return {a, n - a}; }
    if (n <= 22) return {7, n - 14, 7};
    if (n <= 26) return {8, n - 16, 8};
    // beyond 2^26 an end pass has to grow too: the 1024-row pass goes in the middle (its tile arrives by TMA at 0.84 of the peak), the
    // smaller end first (256-row first pass with 128-byte runs): measured faster than {9,9,9} for 2^27 and than {9,10,9} / {10,9,9}
    // for 2^28, in both precisions
    if (n == 27) return {8, 10, 9};
    if (n == 28) return {8, 10, 10};
    if (n == 29) return {9, 10, 10};
    int a = (n + 2) / 3, b = (n - a + 1) / 2;
    return {a, n - a - b, b};
}

// `l2_resident`: the whole signal fits L2 (a few MiB .. 64 MiB).  There the passes are launch- and
// latency-bound single waves and the tile width is chosen by a wave model (narrower tiles win while the CTAs still
// fit one wave; 2^20 f64 stays at 8 columns because its 1024-row tile holds only one CTA per SM).
template <typename T>
const KernelEntry<T>* pick_kernel(int kind, int R, int max_c, int pass_index, bool hbm_strided, bool l2_resident = false,
                                  size_t rows_total = 0, int pref_c = 0, int pref_variant = 0) {
    int want_c = pref_c, want_variant = pref_variant;
    auto nth = [&](const char* name, int& out) {
        if (const char* env = getenv(name)) {
            std::string sv(env);
            size_t pos = 0;
            for (int i = 0; pos <= sv.size(); ++i) {
                size_t q = sv.find(',', pos);
                if (q == std::string::npos) q = sv.size();
                if (i == pass_index) out = atoi(sv.substr(pos, q - pos).c_str());
                pos = q + 1;
            }
        }
    };
    if (const char* env = getenv("PHASTFT_TILE_C")) want_c = atoi(env);
    if (const char* env = getenv("PHASTFT_VARIANT")) want_variant = atoi(env);
    nth("PHASTFT_PASS_C", want_c);                 // e.g. "16,8,16"
    if (g_choice && pass_index >= 0 && pass_index < (int)g_choice->pass_c.size() && g_choice->pass_c[pass_index] > 0)
        want_c = g_choice->pass_c[pass_index];
    nth("PHASTFT_PASS_VARIANT", want_variant);     // e.g. "0,5,0"
    const int CH = TileC<T>::CH, CN = TileC<T>::CN, CW = TileC<T>::CW;
    const size_t tile_limit = 72 * 1024;           // keep >= 3 CTAs/SM worth of shared memory
    const KernelEntry<T>* best = nullptr;
    int best_rank = 1 << 30;
    for (const auto& e : registry<T>()) {
        if (e.kind != kind || e.R != R || e.mode != MODE_PLAIN) continue;
        if (kind != KIND_ROW && e.C > max_c) continue;
        if (e.variant != want_variant) continue;
        int rank;
        if (kind == KIND_ROW) rank = 0;
        else if (want_c) rank = (e.C == want_c) ? 0 : 10 + abs(e.C - want_c);
        else if (l2_resident) {
            // cost ~ (waves of CTAs) x (points per tile): a pass over an L2-resident signal is one or two
            // latency-bound waves, so smaller tiles win until they no longer fit the chip in one wave
            if (e.C != CH && e.C != CN && e.C != CW) continue;
            int occ = 1, sms = 132, dev = 0;
            cudaGetDevice(&dev);
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
            cudaFuncSetAttribute(e.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e.smem);
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, e.fn, e.NT, e.smem) != cudaSuccess || occ < 1) occ = 1;
            const size_t ctas = std::max<size_t>(1, rows_total / (size_t)e.C);
            const size_t waves = (ctas + (size_t)sms * occ - 1) / ((size_t)sms * occ);
            rank = (int)std::min<size_t>(waves * (size_t)e.R * e.C, 1u << 24) * 4 - ilog2(e.C);   // tie -> wider tile
        }
        else if (hbm_strided) rank = (e.C == CW && e.smem <= tile_limit) ? 0 : (e.C == CN) ? 1 : (e.C == CW) ? 2 : (e.C == CH) ? 4 : 3;
        else rank = (e.C == CN) ? 0 : (e.C == CW && e.smem <= tile_limit) ? 1 : (e.C == CH) ? 2 : 3;
        if (rank < best_rank) { best = &e; best_rank = rank; }
    }
    if (!best && want_variant != 0) {   // requested variant does not exist for this tile: fall back to the default
        for (const auto& e : registry<T>())
            if (e.kind == kind && e.R == R && e.variant == 0 && e.mode == MODE_PLAIN && (kind == KIND_ROW || e.C <= max_c) && !best) best = &e;
    }
    return best;
}

// One-CTA kernels: for a batch the radix-16 builds win at some sizes (2^8, f32 2^11, f64 2^11 / 2^12) while a lone
// transform prefers the default.
template <typename T>
const KernelEntry<T>* pick_row_batch_kernel(int R, const KernelEntry<T>* dflt) {
    if (const char* env = getenv("PHASTFT_ROW_VARIANT")) {        // re-tuning override
        const int want = atoi(env);
        for (const auto& e : registry<T>())
            if (e.kind == KIND_ROW && e.R == R && e.variant == want) return &e;
    }
    // measured per size, batches of 2^24 points, after the stage twiddles of these kernels became contiguous loads + products;
    // 0 = the lone-transform kernel is also the best batch kernel
    const bool f64 = sizeof(T) == 8;
    int want = 0;
    switch (R) {
        case 4: case 8: want = 80; break;
        case 16: want = f64 ? 80 : 81; break;
        case 256: want = 70; break;
        case 512: want = f64 ? 0 : 81; break;
        case 1024: want = 0; break;
        case 2048: want = f64 ? 81 : 70; break;
        case 4096: want = 70; break;
        case 8192: want = f64 ? 90 : 0; break;
        case 16384: want = 91; break;
        default: break;
    }
    for (const auto& e : registry<T>())        // want == 0: the plain build (the lone-transform choice may be another variant)
        if (e.kind == KIND_ROW && e.R == R && e.variant == want && e.mode == MODE_PLAIN) return &e;
    return dflt;
}

// The MODE_ROW_BULK build of a one-CTA batch kernel (same radices, C and id; NT may differ), or NULL.  Opt-in (PHASTFT_ROW_BULK=1):
// bit-identical and measured equal or slower at every size (the doubled shared memory costs occupancy) -- these kernels are
// not bound by their per-lane global accesses.
template <typename T>
const KernelEntry<T>* find_row_bulk(const KernelEntry<T>* kb) {
    if (!kb || kb->kind != KIND_ROW) return nullptr;
    const char* env = getenv("PHASTFT_ROW_BULK");
    if (!env || atoi(env) == 0) return nullptr;
    for (const auto& e : registry<T>())
        if (e.mode == MODE_ROW_BULK && e.kind == KIND_ROW && e.R == kb->R && e.C == kb->C && e.variant == kb->variant && e.rl == kb->rl) return &e;
    return nullptr;
}

// Entries of the concatenated per-stage [i][m] stage-twiddle tables of a one-CTA kernel (stage q >= 1 owns Ns(q) * rad(q)).
template <typename T>
size_t tw_im_entries(const KernelEntry<T>* k) {
    size_t tot = 0, ns = (size_t)k->rads[0];
    for (int q = 1; q < k->stages; ++q) { tot += ns * (size_t)k->rads[q]; ns *= (size_t)k->rads[q]; }
    return tot;
}

template <typename T>
int32_t build_plan(size_t n, int device, Plan<T>** out) {
    if (!out) return fail(PHASTFT_ERR_INVALID_ARG, "out == NULL");
    *out = nullptr;
    if (!is_pow2(n)) return fail(PHASTFT_ERR_NOT_POW2);          // planner.rs:66
    if (n > (size_t(1) << 30)) return fail(PHASTFT_ERR_INVALID_ARG, "num_points > 2^30 not supported");
    int count = 0;
    cudaError_t ce = cudaGetDeviceCount(&count);
    if (ce != cudaSuccess || count == 0) return fail(PHASTFT_ERR_NO_DEVICE, ce != cudaSuccess ? cudaGetErrorString(ce) : "");
    if (device < 0 || device >= count) return fail(PHASTFT_ERR_NO_DEVICE, "device ordinal out of range");
    DeviceGuard guard(device);

    std::unique_ptr<Plan<T>> pl(new Plan<T>());
    pl->n = n;
    pl->log2n = ilog2(n);
    pl->device = device;
    const int ln = pl->log2n;

    std::vector<int> f = ln == 0 ? std::vector<int>{} : choose_factors<T>(ln);
    pl->num_passes = (int)f.size();
    pl->ws_il = ws_interleaved_mode();
    if (const char* e = getenv("PHASTFT_PDL")) pl->pdl = atoi(e) != 0;
    pl->l2_chunk_bytes = L2_CHUNK_BYTES_DEFAULT;
    if (const char* e = getenv("PHASTFT_L2_CHUNK_MB")) { const long mb = atol(e); if (mb > 0) pl->l2_chunk_bytes = (size_t)mb << 20; }
    {
        long mb = PIPE_RING_MB_DEFAULT;
        if (const char* e = getenv("PHASTFT_PIPE_RING_MB")) mb = atol(e);
        pl->pipe_ring_bytes = (size_t)std::max(1L, mb) << 20;
    }
    if (const char* e = getenv("PHASTFT_PIPE_DISCARD")) pl->pipe_discard = atoi(e) != 0;
    pl->scribble_on = scribble_env();
    const bool il3 = pl->num_passes == 3 && pl->ws_il != 0;   // the middle pass reads and writes interleaved data
    // two-level W_N table
    pl->lo_bits = (ln + 1) / 2;
    const size_t n_lo = size_t(1) << pl->lo_bits, n_hi = size_t(1) << (ln - pl->lo_bits);
    size_t off = BLOB_HEADER_BYTES;
    pl->hi_off = off; off += n_hi * sizeof(double2);
    pl->lo_off = off; off += n_lo * sizeof(double2);

    int acc = 0;
    for (int p = 0; p < pl->num_passes; ++p) {
        PassDesc<T>& d = pl->pass[p];
        d.log2R = f[p];
        d.log2A = acc;
        d.log2B = ln - acc - f[p];
        d.log2R1 = f[0];
        acc += f[p];
        const bool last = (p == pl->num_passes - 1);
        const int kind = pl->num_passes == 1 ? KIND_ROW : (last ? KIND_TRANS : KIND_COL);
        const int max_c = kind == KIND_COL ? (1 << d.log2B) : kind == KIND_TRANS ? (1 << f[0]) : (1 << 30);
        // wide (128-byte) runs pay off once the signal no longer lives in L2; below that more, smaller CTAs win
        const bool big = ln >= 21;     // above 2^20 the passes are multi-wave streams, below single latency-bound waves
        const bool wide = (p == 0 || last) && big;
        // interleaved 1024-row middle pass: half-width (64-byte-run) tile, two CTAs per SM
        const bool half_mid = il3 && p == 1 && f[p] == 10;
        // lone 2^11-point f32 transform in one CTA: 8x16x16 measured faster than 4x8x8x8
        const bool row2048_f32 = kind == KIND_ROW && f[p] == 11 && sizeof(T) == 4;
        // likewise f64 2^11 8x16x16 (against 4x8x8x8), f32 2^12 16x16x16 (8x8x8x8), f32 2^13 16x16x32 (16x8x8x8)
        const bool row_r16 = kind == KIND_ROW && ((f[p] == 11 && sizeof(T) == 8) || (f[p] == 12 && sizeof(T) == 4));
        const bool row8192_f32 = kind == KIND_ROW && f[p] == 13 && sizeof(T) == 4;
        const int pref_c = half_mid ? TileC<T>::CH : 0, pref_v = half_mid ? 62 : (row2048_f32 || row_r16) ? 70 : row8192_f32 ? 91 : 0;
        d.k = pick_kernel<T>(kind, 1 << f[p], max_c, p, /*hbm_strided=*/wide, /*l2_resident=*/!big, /*rows_total=*/n >> f[p], pref_c, pref_v);
        // batched calls are multi-wave streams whatever N is: wide runs only where the rows of a tile are
        // far apart in memory (>= 64 KiB: first-pass loads, last-pass stores of large N), else 64-byte runs
        const size_t far_stride = (kind == KIND_COL ? (size_t(1) << d.log2B) : (n >> f[p])) * sizeof(T);
        const bool wide_b = (p == 0 || last) && far_stride >= (size_t(64) << 10);
        // f32 batches of 2^17..2^20 points: 32-byte-run tiles (more CTAs per SM) measured faster than 64-byte runs; f64 measured the
        // other way round and keeps its 64-byte runs
        // (the opt-in pipelined launch is compiled for the 64-byte-run pairs: whenever PHASTFT_PIPE is set, to 0 or 1, the batch
        // kernels stay those, so that the two settings run the same pass kernels and can be compared bit for bit)
        const bool pipe_on = getenv("PHASTFT_PIPE") != nullptr;
        const int pref_c_b = (sizeof(T) == 4 && pl->num_passes == 2 && ln >= 17 && kind != KIND_ROW && !pipe_on) ? TileC<T>::CH : pref_c;
        d.kb = (kind == KIND_ROW) ? pick_row_batch_kernel<T>(1 << f[p], d.k) : pick_kernel<T>(kind, 1 << f[p], max_c, p, /*hbm_strided=*/wide_b, false, 0, pref_c_b, pref_v);
        if (!d.k) return fail(PHASTFT_ERR_INVALID_ARG, "no kernel for pass size 2^" + std::to_string(f[p]) + " kind " + kind_name(kind));
        if (kind == KIND_ROW) d.kr = find_row_bulk<T>(d.kb);
        if (p == 0 && kind == KIND_COL)         // the same tile with the c2r pre-processing in its loads, if compiled (c2r_dev uses it)
            for (const auto& e : registry<T>()) {
                const bool same = e.kind == kind && e.R == d.k->R && e.C == d.k->C && e.NT == d.k->NT && e.variant == d.k->variant &&
                                  e.rl == d.k->rl && !e.batch_only;
                if (same && e.mode == MODE_C2R_IN) d.kc = &e;
                if (same && e.mode == MODE_C2R_IN_IL) d.kci = &e;
            }
        if (p == 0 && kind == KIND_COL && d.kb)  // ... and of the batch tile (batched c2r)
            for (const auto& e : registry<T>()) {
                const bool same = e.kind == kind && e.R == d.kb->R && e.C == d.kb->C && e.NT == d.kb->NT && e.variant == d.kb->variant &&
                                  e.rl == d.kb->rl;
                if (same && e.mode == MODE_C2R_IN) d.kcb = &e;
                if (same && e.mode == MODE_C2R_IN_IL) d.kcbi = &e;
            }
        // the interleaved c2r takes the planar one's path, so every c2r build has its interleaved twin (one tile list, reg_strided.cu)
        if ((d.kc != nullptr) != (d.kci != nullptr) || (d.kcb != nullptr) != (d.kcbi != nullptr))
            return fail(PHASTFT_ERR_INVALID_ARG, "unreachable: a c2r build of the first pass has no interleaved twin");
        if (p > 0) {
            d.has_tw = 1;
            d.log2Rprev = f[p - 1];
            d.tw_shift = ln - (f[p - 1] + f[p] + d.log2B);
        }
        d.tw_stage_off = off; off += (size_t(1) << f[p]) * sizeof(cx<T>);
        if (kind == KIND_ROW) {
            off = (off + 255) & ~size_t(255);
            d.tw_im_off = off; off += std::max<size_t>(1, tw_im_entries<T>(d.k)) * sizeof(cx<T>);
            if (d.kb && d.kb != d.k) {
                off = (off + 255) & ~size_t(255);
                d.tw_im_off_b = off; off += std::max<size_t>(1, tw_im_entries<T>(d.kb)) * sizeof(cx<T>);
            } else {
                d.tw_im_off_b = d.tw_im_off;
            }
        }
        if (kind == KIND_TRANS && pl->num_passes == 2) {
            d.tw_wc_off = off;
            off += (size_t)d.k->C * ((size_t(1) << f[p]) / d.k->first_radix) * sizeof(cx<T>);
            if (d.kb && d.kb != d.k) {
                off = (off + 255) & ~size_t(255);
                d.tw_wc_off_b = off;
                off += (size_t)d.kb->C * ((size_t(1) << f[p]) / d.kb->first_radix) * sizeof(cx<T>);
            } else {
                d.tw_wc_off_b = d.tw_wc_off;
            }
        }
        off = (off + 255) & ~size_t(255);
    }
    // Two-pass plans with both tiles of 256 / 512 / 1024 rows (2^16..2^20 points): a pair of asynchronous-input kernels (TMA boxes
    // of the planar input into the first pass's tile, bulk copies of the interleaved workspace's rows into the second's).
    //   batched calls (batch * N >= 2^21, multi-wave grids): the default (faster in both precisions from 2^16 to 2^20 points);
    //   PHASTFT_TMA_BATCH=0 keeps the register-staged kernels
    //   lone transforms (single-wave grids): equal or slower, opt-in with PHASTFT_TMA=1
    // PHASTFT_TMA_VARIANT picks a build (300: 64 KB tiles, 301: 128 KB tiles).
    if (pl->num_passes == 2) {
        int lone = 0, batch = 1, want = 300;
        if (const char* env = getenv("PHASTFT_TMA")) lone = atoi(env);
        if (const char* env = getenv("PHASTFT_TMA_BATCH")) batch = atoi(env);
        else if (getenv("PHASTFT_PIPE")) batch = 0;    // A/B runs of the pipelined launch compare against the kernels it is built from
        if (getenv("PHASTFT_TMA_VARIANT") && !getenv("PHASTFT_TMA")) lone = 1;
        if (const char* env = getenv("PHASTFT_TMA_VARIANT")) want = atoi(env);
        const bool enabled = lone || batch;
        pl->tma_lone = lone != 0; pl->tma_batch = batch != 0;
        const KernelEntry<T>* t0 = nullptr; const KernelEntry<T>* t1 = nullptr;
        if (enabled && tensor_map_encoder())
            for (const auto& e : registry<T>()) {
                if (e.variant != want) continue;
                if (e.mode == MODE_TMA_IN && e.kind == KIND_COL && e.R == (1 << f[0]) && e.C <= (1 << f[1])) t0 = &e;
                if (e.mode == MODE_BULK_IN && e.kind == KIND_TRANS && e.R == (1 << f[1]) && e.C <= (1 << f[0])) t1 = &e;
            }
        if (t0 && t1) {
            pl->pass[0].kt = t0; pl->pass[1].kt = t1;
            PassDesc<T>& d = pl->pass[1];
            d.tw_wc_off_t = off;
            off += (size_t)t1->C * ((size_t(1) << f[1]) / t1->first_radix) * sizeof(cx<T>);
            off = (off + 255) & ~size_t(255);
        }
    }
    // 3-pass plans with interleaved intermediates: the 1024-row middle pass with its tile arriving by TMA (64 KB landing zone =
    // the tile, no register-staged loads: three CTAs per SM each with its whole tile in flight).  PHASTFT_TMA_MID=0|1.
    if (pl->num_passes == 3 && il3) {
        int enabled = 1, ends = 0;
        if (const char* env = getenv("PHASTFT_TMA_MID")) enabled = atoi(env);
        if (const char* env = getenv("PHASTFT_TMA_ENDS")) ends = atoi(env);
        if (tensor_map_encoder())
            for (const auto& e : registry<T>()) {
                if (enabled >= 2 && e.variant == 310 && e.mode == MODE_TMA_IN && e.kind == KIND_COL && e.R == (1 << f[1]) && e.C == TileC<T>::CH) pl->pass[1].kt = &e;
                if (e.variant != 300) continue;
                if (enabled && e.mode == MODE_TMA_IN && e.kind == KIND_COL && e.R == (1 << f[1]) && e.C == TileC<T>::CH) pl->pass[1].kt = &e;
                // the 128-byte-run end passes: planar boxes in (first pass), contiguous rows of the workspace in (last pass)
                if (ends && e.mode == MODE_TMA_IN && e.kind == KIND_COL && e.R == (1 << f[0]) && e.C == TileC<T>::CW) pl->pass[0].kt = &e;
                if (ends && e.mode == MODE_BULK_IN && e.kind == KIND_TRANS && e.R == (1 << f[2]) && e.C == TileC<T>::CW) pl->pass[2].kt = &e;
            }
    }
    // The radix-32 stage table of every strided pass that may launch a kernel ending in a radix-32 stage (any of k, kb, kt, kc, kcb)
    auto ends_in_32 = [](const KernelEntry<T>* k) { return k && k->kind != KIND_ROW && k->stages >= 2 && k->rads[k->stages - 1] == 32; };
    for (int p = 0; p < pl->num_passes; ++p) {
        PassDesc<T>& d = pl->pass[p];
        if (ends_in_32(d.k) || ends_in_32(d.kb) || ends_in_32(d.kt) || ends_in_32(d.kc) || ends_in_32(d.kcb)) {
            d.tw32_off = off;
            off += (size_t(1) << d.log2R) * sizeof(cx<T>);
            off = (off + 255) & ~size_t(255);
        }
    }
    // Batches of transforms that one CTA can hold (128 KB tile: 2^13 f64, 2^14 f32) use a one-CTA kernel: one launch,
    // one HBM round trip.  PHASTFT_ONE_CTA_MAX (log2) lowers the limit for re-tuning.
    // 2^13 f64 / 2^13-2^14 f32 in one CTA (64-128 KB tile): slower than two passes of small tiles while the stage twiddles were
    // gathers, faster since they are contiguous loads + products.
    int one_cta_max = sizeof(T) == 8 ? 13 : 14;
    if (const char* env = getenv("PHASTFT_ONE_CTA_MAX")) one_cta_max = std::min(atoi(env), sizeof(T) == 8 ? 13 : 14);
    if (pl->num_passes >= 2 && ln <= one_cta_max) {
        PassDesc<T>& d = pl->alt_row;
        d.log2R = ln; d.log2A = 0; d.log2B = 0; d.log2R1 = ln;
        d.k = pick_kernel<T>(KIND_ROW, 1 << ln, 1 << 30, 0, false);
        d.k = pick_row_batch_kernel<T>(1 << ln, d.k);            // alt_row is only ever used for batches
        d.kb = d.k;
        d.kr = find_row_bulk<T>(d.kb);
        if (d.k) {
            d.tw_stage_off = off; off += (size_t(1) << ln) * sizeof(cx<T>);
            off = (off + 255) & ~size_t(255);
            d.tw_im_off = d.tw_im_off_b = off; off += std::max<size_t>(1, tw_im_entries<T>(d.k)) * sizeof(cx<T>);
            off = (off + 255) & ~size_t(255);
            pl->alt_row_min_batch = ln <= 12 ? 4 : 32;
        }
    }
    // Larger transforms up to the shared memory of a cluster (2^14..2^16 f64, 2^15..2^16 f32): both passes in one
    // cluster launch.  PHASTFT_CLUSTER=0 disables, PHASTFT_CLUSTER_VARIANT=<id> picks a build, PHASTFT_CLUSTER_MIN_BATCH
    // sets the smallest call that uses it (a lone transform keeps K SMs busy, the two-launch plan the whole chip).
    {
        int want = 0, enabled = 0;        // measured slower than the two-launch plan at every size: opt-in
        if (const char* env = getenv("PHASTFT_CLUSTER")) enabled = atoi(env);
        if (const char* env = getenv("PHASTFT_CLUSTER_VARIANT")) { want = atoi(env); if (!getenv("PHASTFT_CLUSTER")) enabled = 1; }
        if (getenv("PHASTFT_CLUSTER_MIN_BATCH") && !getenv("PHASTFT_CLUSTER")) enabled = 1;
        if (enabled && !pl->alt_row.k)
            for (const auto& ce : cluster_registry<T>())
                if (ce.log2n == ln && ce.variant == want) { pl->cl = &ce; break; }
        if (pl->cl) {
            pl->cl_min_batch = 8;
            if (const char* env = getenv("PHASTFT_CLUSTER_MIN_BATCH")) pl->cl_min_batch = (size_t)std::max(1, atoi(env));
            const int l1 = ilog2((size_t)pl->cl->k1.R), l2 = ilog2((size_t)pl->cl->k2.R);
            PassDesc<T>& a = pl->cl_pass[0];
            a.k = a.kb = &pl->cl->k1;
            a.log2R = l1; a.log2A = 0; a.log2B = l2; a.log2R1 = l1;
            a.tw_stage_off = off; off += (size_t(1) << l1) * sizeof(cx<T>);
            off = (off + 255) & ~size_t(255);
            PassDesc<T>& b = pl->cl_pass[1];
            b.k = b.kb = &pl->cl->k2;
            b.log2R = l2; b.log2A = l1; b.log2B = 0; b.log2R1 = l1;
            b.has_tw = 1; b.log2Rprev = l1; b.tw_shift = 0;
            b.tw_stage_off = off; off += (size_t(1) << l2) * sizeof(cx<T>);
            b.tw_wc_off = b.tw_wc_off_b = off;
            off += (size_t)b.k->C * ((size_t(1) << l2) / b.k->first_radix) * sizeof(cx<T>);
            off = (off + 255) & ~size_t(255);
        }
    }
    // ---- fill the blob ------------------------------------------------------------------------------
    pl->blob_host.assign(off, 0);
    {
        double2* hi = reinterpret_cast<double2*>(pl->blob_host.data() + pl->hi_off);
        double2* lo = reinterpret_cast<double2*>(pl->blob_host.data() + pl->lo_off);
        for (size_t h = 0; h < n_hi; ++h) root_of_unity((uint64_t)h << pl->lo_bits, n, hi[h].x, hi[h].y);
        for (size_t l = 0; l < n_lo; ++l) root_of_unity(l, n, lo[l].x, lo[l].y);
    }
    auto fill_pass_tables = [&](PassDesc<T>& d) {
        const size_t R = size_t(1) << d.log2R;
        cx<T>* tw = reinterpret_cast<cx<T>*>(pl->blob_host.data() + d.tw_stage_off);
        for (size_t e = 0; e < R; ++e) {
            double re, im;
            root_of_unity(e, R, re, im);
            tw[e].x = (T)re; tw[e].y = (T)im;
        }
        for (int which = 0; which < 2; ++which) {      // one-CTA kernels: per-stage [i][m] tables, W_L^(m*i) with L = Ns * rad
            const KernelEntry<T>* kk = which ? d.kb : d.k;
            const size_t ioff = which ? d.tw_im_off_b : d.tw_im_off;
            if (!kk || kk->kind != KIND_ROW || ioff == (size_t)-1 || (which && ioff == d.tw_im_off)) continue;
            cx<T>* t = reinterpret_cast<cx<T>*>(pl->blob_host.data() + ioff);
            size_t ns = (size_t)kk->rads[0];
            for (int q = 1; q < kk->stages; ++q) {
                const size_t rad = (size_t)kk->rads[q], L = ns * rad;
                for (size_t i = 0; i < rad; ++i)
                    for (size_t m = 0; m < ns; ++m) {
                        double re, im;
                        root_of_unity((uint64_t)(m * i), L, re, im);
                        t[i * ns + m].x = (T)re; t[i * ns + m].y = (T)im;
                    }
                t += L; ns = L;
            }
        }
        for (int which = 0; which < 3; ++which) {
            const KernelEntry<T>* kk = which == 2 ? d.kt : which ? d.kb : d.k;
            const size_t woff = which == 2 ? d.tw_wc_off_t : which ? d.tw_wc_off_b : d.tw_wc_off;
            if (!kk || woff == (size_t)-1 || (which == 1 && woff == d.tw_wc_off)) continue;
            // W_L^(c*m), L = N (2-pass plan), [c][m] layout, m < M = R / first_radix
            const size_t M = R / kk->first_radix;
            cx<T>* wc = reinterpret_cast<cx<T>*>(pl->blob_host.data() + woff);
            for (int c = 0; c < kk->C; ++c)
                for (size_t m = 0; m < M; ++m) {
                    double re, im;
                    root_of_unity((uint64_t)c * m, n, re, im);
                    wc[(size_t)c * M + m].x = (T)re; wc[(size_t)c * M + m].y = (T)im;
                }
        }
    };
    for (int p = 0; p < pl->num_passes; ++p) fill_pass_tables(pl->pass[p]);
    if (pl->alt_row.k) fill_pass_tables(pl->alt_row);
    if (pl->cl) { fill_pass_tables(pl->cl_pass[0]); fill_pass_tables(pl->cl_pass[1]); }
    CUDA_TRY(cudaMalloc(&pl->blob_dev, pl->blob_host.size()));
    CUDA_TRY(cudaMemcpy(pl->blob_dev, pl->blob_host.data(), pl->blob_host.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaStreamCreateWithFlags(&pl->stream, cudaStreamNonBlocking));
    CUDA_TRY(cudaEventCreateWithFlags(&pl->ws_free, cudaEventDisableTiming));
    // The radix-32 stage tables, from the W_R tables just copied.  On the default stream: a cudaMemcpy from pageable memory may
    // return before its data has landed, and only work on that stream is ordered after it.
    for (int p = 0; p < pl->num_passes; ++p) {
        const PassDesc<T>& d = pl->pass[p];
        if (d.tw32_off == (size_t)-1) continue;
        const int ns = 1 << (d.log2R - 5);
        stage32_table_kernel<T><<<(ns + 255) / 256, 256>>>(reinterpret_cast<const cx<T>*>(pl->blob_dev + d.tw_stage_off),
                                                           reinterpret_cast<cx<T>*>(pl->blob_dev + d.tw32_off), ns);
        CUDA_TRY(cudaGetLastError());
    }
    CUDA_TRY(cudaStreamSynchronize(0));
    for (int p = 0; p < pl->num_passes; ++p) {
        CUDA_TRY(cudaFuncSetAttribute(pl->pass[p].k->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl->pass[p].k->smem));
        if (pl->pass[p].kb)
            CUDA_TRY(cudaFuncSetAttribute(pl->pass[p].kb->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl->pass[p].kb->smem));
        if (pl->pass[p].kt)
            CUDA_TRY(cudaFuncSetAttribute(pl->pass[p].kt->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl->pass[p].kt->smem));
        if (pl->pass[p].kc)
            CUDA_TRY(cudaFuncSetAttribute(pl->pass[p].kc->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl->pass[p].kc->smem));
        if (pl->pass[p].kcb)
            CUDA_TRY(cudaFuncSetAttribute(pl->pass[p].kcb->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl->pass[p].kcb->smem));
        if (pl->pass[p].kci)
            CUDA_TRY(cudaFuncSetAttribute(pl->pass[p].kci->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl->pass[p].kci->smem));
        if (pl->pass[p].kcbi)
            CUDA_TRY(cudaFuncSetAttribute(pl->pass[p].kcbi->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl->pass[p].kcbi->smem));
        if (pl->pass[p].kr)
            CUDA_TRY(cudaFuncSetAttribute(pl->pass[p].kr->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl->pass[p].kr->smem));
    }
    if (pl->alt_row.k)
        CUDA_TRY(cudaFuncSetAttribute(pl->alt_row.k->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl->alt_row.k->smem));
    if (pl->alt_row.kr)
        CUDA_TRY(cudaFuncSetAttribute(pl->alt_row.kr->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl->alt_row.kr->smem));
    if (pl->cl) {
        // usable only if the device can co-schedule at least one cluster of this shape
        cudaError_t ce = cudaFuncSetAttribute(pl->cl->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl->cl->smem);
        if (ce == cudaSuccess && pl->cl->K > 8) ce = cudaFuncSetAttribute(pl->cl->fn, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
        int nclusters = 0;
        if (ce == cudaSuccess) {
            cudaLaunchConfig_t cfg;
            memset(&cfg, 0, sizeof(cfg));
            cfg.gridDim = dim3((unsigned)pl->cl->K); cfg.blockDim = dim3((unsigned)pl->cl->NT); cfg.dynamicSmemBytes = pl->cl->smem;
            cudaLaunchAttribute attr[1];
            attr[0].id = cudaLaunchAttributeClusterDimension;
            attr[0].val.clusterDim.x = (unsigned)pl->cl->K; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
            cfg.attrs = attr; cfg.numAttrs = 1;
            ce = cudaOccupancyMaxActiveClusters(&nclusters, pl->cl->fn, &cfg);
        }
        if (ce != cudaSuccess || nclusters < 1) { (void)cudaGetLastError(); pl->cl = nullptr; }
        pl->cl_max_active = nclusters;
    }
    if (pl->num_passes >= 2) {
        CUDA_TRY(cudaMalloc(&pl->ws_re, 2 * n * sizeof(T)));
        pl->ws_im = pl->ws_re + n;
        pl->ws_elems = n;
        CUDA_TRY(scribble_new(pl->scribble_on, pl->ws_re, 2 * n * sizeof(T)));
    }
    if (pl->num_passes == 3) {
        // L2 blocking of passes 2+3: group size in bytes from PHASTFT_L2_GROUP_MB (default 32; 0 disables)
        size_t group_mb = 0;   // measured slower than three full-size passes (launch ramp/tail per group), off by default
        if (const char* env = getenv("PHASTFT_L2_GROUP_MB")) group_mb = (size_t)atoi(env);
        const size_t sub_bytes = (n >> f[0]) * 2 * sizeof(T);
        const long long R1 = 1LL << f[0];
        const long long ctrans = pl->pass[2].k->C;
        long long G = ctrans;
        while (G * 2 <= R1 && (size_t)(G * 2) * sub_bytes <= (group_mb << 20)) G *= 2;
        if (group_mb > 0 && (size_t)G * sub_bytes * 2 <= n * 2 * sizeof(T)) {
            pl->l2_group = G;
            CUDA_TRY(cudaMalloc(&pl->ws2_re, (size_t)G * (n >> f[0]) * sizeof(T)));
            CUDA_TRY(cudaMalloc(&pl->ws2_im, (size_t)G * (n >> f[0]) * sizeof(T)));
            CUDA_TRY(scribble_new(pl->scribble_on, pl->ws2_re, (size_t)G * (n >> f[0]) * sizeof(T)));
            CUDA_TRY(scribble_new(pl->scribble_on, pl->ws2_im, (size_t)G * (n >> f[0]) * sizeof(T)));
        }
    }
    if (pl->num_passes == 2) {
        // PHASTFT_PIPE=0 disables the pipelined launch; PHASTFT_PIPE_LONE=1 also sends lone transforms through it
        int enabled = 0, lone = 0;        // opt-in until it beats two launches
        if (const char* e = getenv("PHASTFT_PIPE")) enabled = atoi(e);
        if (const char* e = getenv("PHASTFT_PIPE_LONE")) lone = atoi(e);
        int want_mode = 0;                 // PHASTFT_PIPE_TMA=1: the pair with asynchronous tile input, where one exists
        if (const char* e = getenv("PHASTFT_PIPE_TMA")) want_mode = atoi(e) != 0;
        auto find = [&](const KernelEntry<T>* a, const KernelEntry<T>* b) -> const PipeEntry<T>* {
            if (!a || !b) return nullptr;
            const PipeEntry<T>* plain = nullptr;
            for (const auto& pe : pipe_registry<T>())
                if (pe.R1 == a->R && pe.C1 == a->C && pe.NT1 == a->NT && pe.rad1 == a->radices && pe.R2 == b->R && pe.C2 == b->C &&
                    pe.NT2 == b->NT && pe.rad2 == b->radices) {
                    if (pe.mode == want_mode && tensor_map_encoder()) return &pe;
                    if (pe.mode == 0) plain = &pe;
                }
            return plain;
        };
        auto resident = [&](const PipeEntry<T>* pe) -> int {
            int occ = 0, sms = 0;
            if (cudaFuncSetAttribute(pe->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pe->smem) != cudaSuccess ||
                cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess ||
                cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, pe->fn, pe->NT, pe->smem) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
            return sms * std::max(occ, 0);
        };
        if (enabled) {
            pl->pipe_b = find(pl->pass[0].kb, pl->pass[1].kb);
            if (pl->pipe_b && (pl->pipe_grid_b = resident(pl->pipe_b)) < 2) pl->pipe_b = nullptr;
            if (lone) {
                pl->pipe_1 = find(pl->pass[0].k, pl->pass[1].k);
                if (pl->pipe_1 && (pl->pipe_grid_1 = resident(pl->pipe_1)) < 2) pl->pipe_1 = nullptr;
            }
        }
    }
    // description
    {
        std::string s = "n=2^" + std::to_string(ln) + (sizeof(T) == 8 ? " f64:" : " f32:");
        if (pl->num_passes == 0) s += " identity";
        for (int p = 0; p < pl->num_passes; ++p) {
            const auto* k = pl->pass[p].k;
            s += std::string(p ? " |" : "") + " " + kind_name(k->kind) + " R=" + std::to_string(k->R) + "(" + k->radices + ") C=" +
                 std::to_string(k->C) + " NT=" + std::to_string(k->NT) + " smem=" + std::to_string(k->smem);
        }
        if (pl->num_passes == 2 && pl->pass[0].kt) {
            s += pl->tma_lone && pl->tma_batch ? " || planar input: " : pl->tma_lone ? " || lone planar: " : " || batches, planar input: ";
            for (int p = 0; p < 2; ++p) {
                const auto* k = pl->pass[p].kt;
                s += std::string(p ? " | " : "") + kind_name(k->kind) + " R=" + std::to_string(k->R) + "(" + k->radices + ") C=" + std::to_string(k->C) +
                     " NT=" + std::to_string(k->NT) + " smem=" + std::to_string(k->smem);
            }
        }
        if (pl->num_passes == 3 && pl->pass[1].kt) {
            const auto* k = pl->pass[1].kt;
            s += " [middle pass by TMA: COL R=" + std::to_string(k->R) + "(" + k->radices + ") C=" + std::to_string(k->C) + " NT=" + std::to_string(k->NT) + "]";
        }
        if (pl->num_passes == 3 && pl->pass[0].kt && pl->pass[2].kt) s += " [end passes by TMA / bulk copies, C=" + std::to_string(pl->pass[0].kt->C) + "]";
        if (pl->l2_group) s += " | L2-blocked tail: " + std::to_string(pl->l2_group) + " k1/group";
        bool differs = false;
        for (int p = 0; p < pl->num_passes; ++p) differs |= pl->pass[p].kb && pl->pass[p].kb != pl->pass[p].k;
        if (differs) {
            s += " || batches:";
            for (int p = 0; p < pl->num_passes; ++p) {
                const auto* k = pl->pass[p].kb;
                s += std::string(p ? " |" : "") + " " + kind_name(k->kind) + " R=" + std::to_string(k->R) + "(" + k->radices + ") C=" +
                     std::to_string(k->C) + " NT=" + std::to_string(k->NT);
            }
        }
        if (pl->num_passes >= 2) s += pl->ws_il == 1 ? " [interleaved intermediates]" : pl->ws_il == 0 ? " [planar intermediates]" : "";
        const std::string ring = "L2 ring of " + std::to_string(pl->pipe_ring_bytes >> 20) + " MiB";
        if (pl->pipe_b) s += std::string(" [batches: one pipelined launch, ") + (pl->pipe_b->mode ? "TMA / bulk tile input, " : "") + std::to_string(pl->pipe_grid_b) + " resident CTAs, " + ring + "]";
        if (pl->pipe_1) s += " [lone: one pipelined launch, " + std::to_string(pl->pipe_grid_1) + " resident CTAs, " + ring + "]";
        if (pl->alt_row.k) s += " || batches: ROW R=" + std::to_string(pl->alt_row.k->R) + "(" + pl->alt_row.k->radices + ")";
        if ((pl->num_passes == 1 && pl->pass[0].kr) || pl->alt_row.kr) s += " [contiguous planar batches: tile in / out by cp.async.bulk]";
        if (pl->cl)
            s += " || batches >= " + std::to_string(pl->cl_min_batch) + ": CLUSTER K=" + std::to_string(pl->cl->K) + " NT=" + std::to_string(pl->cl->NT) +
                 " " + std::to_string(pl->cl->k1.R) + "(" + pl->cl->k1.radices + ") x " + std::to_string(pl->cl->k2.R) + "(" + pl->cl->k2.radices +
                 ") smem=" + std::to_string(pl->cl->smem) + (pl->cl->variant ? ",v" + std::to_string(pl->cl->variant) : std::string()) +
                 " resident clusters=" + std::to_string(pl->cl_max_active);
        pl->description = s;
    }
    {
        BlobHeader h;
        memset(&h, 0, sizeof(h));
        h.magic = BLOB_MAGIC; h.bytes = pl->blob_host.size(); h.n = n;
        h.precision_bits = 8 * sizeof(T); h.num_passes = (uint32_t)pl->num_passes;
        h.layout_sig = fnv1a(pl->description);
        for (int p = 0; p < pl->num_passes; ++p) {
            h.tw_stage_off[p] = pl->pass[p].tw_stage_off;
            h.tw32_off[p] = pl->pass[p].tw32_off == (size_t)-1 ? 0 : pl->pass[p].tw32_off;
        }
        memcpy(pl->blob_host.data(), &h, sizeof(h));
        CUDA_TRY(cudaMemcpy(pl->blob_dev, pl->blob_host.data(), BLOB_HEADER_BYTES, cudaMemcpyHostToDevice));
    }
    *out = pl.release();
    return PHASTFT_OK;
}

// =================================================================================================
// execution
// =================================================================================================

template <typename T>
struct Io {
    const T* in_re; const T* in_im;
    T* out_re; T* out_im;
    long long in_bstride, out_bstride;
    int in_il, out_il;   // 0 planar, 1 interleaved, 2 interleaved with re/im swapped
    // c2r: in_re / in_im are the half-spectrum's N/2 + 1 bins and the first pass builds its input from them while loading
    // (PassDesc::kc; in_il = 1: the bins interleaved at in_re, PassDesc::kci); pre_log2half = log2(N/2), 0 = off
    Tw2 pre_tw2 = {nullptr, nullptr, 0};
    int pre_log2half = 0;
    const double2* pre_wc = nullptr;     // host: W_(2 R1)^i, i < 32 (PlanR2c::pre_wc)
    const double2* pre_wc_b = nullptr;   // the same for the first radix of PassDesc::kcb (PlanR2c::pre_wc_b)
};

// Whether a launch of `batch` transforms of this pass runs the batch kernel PassDesc::kb (multi-wave grids).
template <typename T>
bool pass_takes_kb(const Plan<T>& pl, const PassDesc<T>& d, size_t batch) {
    return d.kb != nullptr && batch > 1 && (batch << pl.log2n) >= (size_t(1) << 21);
}

// k1_lo / k1_cnt (multi-pass plans, batch == 1): restrict a pass AFTER the first to the sub-transforms
// whose first-pass output digit k1 lies in [k1_lo, k1_lo + k1_cnt) -- the unit of L2 blocking.
template <typename T>
int32_t prepare_pass(const Plan<T>& pl, int p, const PassParams<T>& base, size_t batch, long long k1_lo, long long k1_cnt,
                     PassParams<T>& prm_out, const KernelEntry<T>*& k_out, unsigned long long& blocks_out, bool use_kt = false);

// use_kt: launch the pass's asynchronous-input kernel (PassDesc::kt); the caller has checked its preconditions
// (pass 0: planar 16-byte-aligned input; last pass: interleaved workspace).
template <typename T>
int32_t launch_pass(const Plan<T>& pl, int p, const PassParams<T>& base, size_t batch, cudaStream_t stream,
                    long long k1_lo = 0, long long k1_cnt = -1, bool use_kt = false) {
    PassParams<T> prm;
    const KernelEntry<T>* k = nullptr;
    unsigned long long blocks = 0;
    int32_t st = prepare_pass(pl, p, base, batch, k1_lo, k1_cnt, prm, k, blocks, use_kt);
    if (st) return st;
    if (k->mode == MODE_TMA_IN) {
        const size_t B = size_t(1) << prm.log2B, A = size_t(1) << prm.log2A;
        const unsigned box_rows = (unsigned)std::min(k->R, 256);
        bool ok;
        if (prm.in_interleaved) {
            // the interleaved workspace as an array of T: rows of 2B values, A * batch blocks of R rows (batch stride = A * R * B pairs)
            if (batch > 1 && (size_t)prm.in_bstride != A * (size_t)k->R * B) return fail(PHASTFT_ERR_INVALID_ARG, "TMA middle pass: the workspace must be dense");
            ok = encode_tile_map<T>(&prm.tmap_re, prm.in_re, 2 * B, (size_t)k->R, 2 * B, A * batch, (size_t)k->R * 2 * B, 2u * (unsigned)k->C, box_rows);
        } else {
            if (A != 1) return fail(PHASTFT_ERR_INVALID_ARG, "TMA planar input: first pass only");
            ok = encode_tile_map<T>(&prm.tmap_re, prm.in_re, B, (size_t)k->R, B, batch, (size_t)prm.in_bstride, (unsigned)k->C, box_rows) &&
                 encode_tile_map<T>(&prm.tmap_im, prm.in_im, B, (size_t)k->R, B, batch, (size_t)prm.in_bstride, (unsigned)k->C, box_rows);
        }
        if (!ok) return fail(PHASTFT_ERR_CUDA, "cuTensorMapEncodeTiled failed");
    }
    void* args[] = {&prm};
    // Programmatic dependent launch: measured no gain with 128 KB tiles (the next grid cannot become resident early), -10%
    // at 2^24+, and slower too with the 64 KB asynchronous-input tiles.  PHASTFT_PDL=1 enables it (Plan::pdl).
    if (pl.pdl) {                          // off by default: measured slower with and without the asynchronous-input kernels
        // Programmatic dependent launch: back-to-back passes overlap the next grid's launch and prologue
        // with the previous grid's tail (the kernel waits with griddepcontrol.wait before its first access).
        prm.pdl = 1;
        cudaLaunchConfig_t cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.gridDim = dim3((unsigned)blocks); cfg.blockDim = dim3(k->NT); cfg.dynamicSmemBytes = k->smem; cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
        CUDA_TRY(cudaLaunchKernelExC(&cfg, k->fn, args));
    } else {
        CUDA_TRY(cudaLaunchKernel(k->fn, dim3((unsigned)blocks), dim3(k->NT), args, k->smem, stream));
    }
    note_launch({kind_name(k->kind), k->R, 0, k->C, k->NT, k->variant, mode_name(k->mode), pl.pdl});
    return PHASTFT_OK;
}

template <typename T>
int32_t prepare_pass_desc(const Plan<T>& pl, const PassDesc<T>& d, int p, const PassParams<T>& base, size_t batch, long long k1_lo,
                          long long k1_cnt, PassParams<T>& prm_out, const KernelEntry<T>*& k_out, unsigned long long& blocks_out,
                          bool use_kt = false);

template <typename T>
int32_t prepare_pass(const Plan<T>& pl, int p, const PassParams<T>& base, size_t batch, long long k1_lo, long long k1_cnt,
                     PassParams<T>& prm_out, const KernelEntry<T>*& k_out, unsigned long long& blocks_out, bool use_kt) {
    const PassDesc<T>& d = (p == ALT_ROW_PASS) ? pl.alt_row : pl.pass[p];
    return prepare_pass_desc(pl, d, p, base, batch, k1_lo, k1_cnt, prm_out, k_out, blocks_out, use_kt);
}

template <typename T>
int32_t prepare_pass_desc(const Plan<T>& pl, const PassDesc<T>& d, int p, const PassParams<T>& base, size_t batch, long long k1_lo,
                          long long k1_cnt, PassParams<T>& prm_out, const KernelEntry<T>*& k_out, unsigned long long& blocks_out,
                          bool use_kt) {
    const bool many = !use_kt && pass_takes_kb(pl, d, batch);
    const KernelEntry<T>* k = use_kt ? d.kt : many ? d.kb : d.k;
    // one-CTA batch kernel with bulk tile input / output: planar arrays, transforms back to back, 16-byte-aligned planes
    if (many && d.kr && k == d.kb && base.in_interleaved == 0 && base.out_interleaved == 0 && base.in_bstride == (long long)pl.n &&
        base.out_bstride == (long long)pl.n &&
        ((reinterpret_cast<uintptr_t>(base.in_re) | reinterpret_cast<uintptr_t>(base.in_im) | reinterpret_cast<uintptr_t>(base.out_re) |
          reinterpret_cast<uintptr_t>(base.out_im)) & 15) == 0)
        k = d.kr;
    if (base.pre_log2half) {
        // interleaved bins (in_interleaved = 1): the MODE_C2R_IN_IL twin of the same tile
        const KernelEntry<T>* kc = base.in_interleaved ? (many ? d.kcbi : d.kci) : many ? d.kcb : d.kc;
        if (p != 0 || use_kt || !kc) return fail(PHASTFT_ERR_INVALID_ARG, "c2r pre-processing on load: first pass with a MODE_C2R_IN kernel only");
        k = kc;
    }
    PassParams<T> prm = base;
    prm.batch = (int)batch;
    prm.log2A = d.log2A; prm.log2B = d.log2B; prm.log2R1 = d.log2R1; prm.log2Rprev = d.log2Rprev;
    prm.has_tw = d.has_tw; prm.tw_shift = d.tw_shift;
    prm.tw2.hi = reinterpret_cast<const double2*>(pl.blob_dev + pl.hi_off);
    prm.tw2.lo = reinterpret_cast<const double2*>(pl.blob_dev + pl.lo_off);
    prm.tw2.lo_bits = pl.lo_bits;
    prm.tw_stage = reinterpret_cast<const cx<T>*>(pl.blob_dev + d.tw_stage_off);
    const size_t wc_off = use_kt ? d.tw_wc_off_t : many ? d.tw_wc_off_b : d.tw_wc_off;
    const size_t im_off = d.tw32_off != (size_t)-1 ? d.tw32_off : many ? d.tw_im_off_b : d.tw_im_off;
    prm.tw_stage_im = im_off == (size_t)-1 ? nullptr : reinterpret_cast<const cx<T>*>(pl.blob_dev + im_off);
    prm.tw_wc = wc_off == (size_t)-1 ? nullptr : reinterpret_cast<const cx<T>*>(pl.blob_dev + wc_off);
    unsigned long long blocks;
    prm.blk_offset = 0; prm.kt_base = 0; prm.log2_ktn = d.log2R1 - ilog2(k->C);
    if (k->kind == KIND_ROW) blocks = (batch + k->C - 1) / k->C;
    else blocks = (unsigned long long)batch * (pl.n >> d.log2R) / k->C;
    if (k1_cnt >= 0 && p > 0) {
        const unsigned long long tiles_per_k1 = ((pl.n >> d.log2R) / k->C) >> d.log2R1;   // COL: (A/R1) * B/C
        if (k->kind == KIND_COL) {
            prm.blk_offset = (int)(k1_lo * tiles_per_k1);
            blocks = k1_cnt * tiles_per_k1;
        } else {
            prm.kt_base = (int)(k1_lo / k->C);
            prm.log2_ktn = ilog2((size_t)(k1_cnt / k->C));
            blocks = ((pl.n >> d.log2R) >> d.log2R1) * (k1_cnt / k->C);                     // rest_n * chunk tiles
        }
    }
    if (blocks == 0 || blocks > 0x7fffffffULL) return fail(PHASTFT_ERR_INVALID_ARG, "grid too large");
    prm_out = prm; k_out = k; blocks_out = blocks;
    return PHASTFT_OK;
}

// Ring of workspace slots of the pipelined two-pass launch: the largest power-of-two number of transforms whose
// intermediates fit Plan::pipe_ring_bytes, at least 1.
template <typename T>
size_t pipe_ring_transforms(const Plan<T>& pl, size_t batch) {
    const size_t bytes_per = pl.n * 2 * sizeof(T);
    size_t ring = 1;
    while (ring * 2 * bytes_per <= pl.pipe_ring_bytes && ring * 2 <= batch) ring *= 2;
    if (ring < 2 && batch > 1) ring = 2;            // two slots at least: pass 1 of b+1 beside pass 2 of b
    return ring;
}
// Transforms per chunk of a batched multi-pass call (run_c2c).
template <typename T>
size_t chunk_transforms(const Plan<T>& pl, size_t batch) {
    const size_t bytes_per = pl.n * 2 * sizeof(T);
    size_t chunk = std::max<size_t>(1, pl.l2_chunk_bytes / bytes_per);
    chunk = std::min(chunk, batch);
    if (pl.num_passes == 3 && pl.ws2_re != nullptr) chunk = 1;
    return chunk;
}
// caller holds pl.mu
template <typename T>
int32_t grow_workspace(const Plan<T>& pl, size_t transforms, cudaStream_t stream) {
    if (pl.ws_elems >= transforms * pl.n) return PHASTFT_OK;
    if (stream) CUDA_TRY(cudaStreamSynchronize(stream));
    CUDA_TRY(cudaDeviceSynchronize());
    if (pl.ws_re) cudaFree(pl.ws_re);
    pl.ws_re = pl.ws_im = nullptr; pl.ws_elems = 0;
    CUDA_TRY(cudaMalloc(&pl.ws_re, 2 * transforms * pl.n * sizeof(T)));
    pl.ws_im = pl.ws_re + transforms * pl.n;
    pl.ws_elems = transforms * pl.n;
    CUDA_TRY(scribble_new(pl.scribble_on, pl.ws_re, 2 * transforms * pl.n * sizeof(T)));
    return PHASTFT_OK;
}

template <typename T>
int32_t plan_reserve(const Plan<T>* pl, size_t batch) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (pl->num_passes < 2 || batch <= 1) return PHASTFT_OK;       // one-CTA plans have no workspace
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> lock(pl->mu);
    const size_t bytes_per = pl->n * 2 * sizeof(T);
    size_t chunk = std::max<size_t>(1, pl->l2_chunk_bytes / bytes_per);
    chunk = std::min(chunk, batch);
    if (pl->pipe_b && (batch << pl->log2n) >= (size_t(1) << 21)) chunk = pipe_ring_transforms(*pl, batch);
    return grow_workspace(*pl, chunk, nullptr);
}

// `pass_events` (profiling aid, bench.py roofline): if non-NULL, num_passes+1 events are recorded
// around the passes of the FIRST chunk.
template <typename T>
int32_t run_c2c(const Plan<T>& pl, const Io<T>& io, size_t batch, T scale, cudaStream_t stream,
                cudaEvent_t* pass_events = nullptr) {
    if (batch == 0) return PHASTFT_OK;
    PassParams<T> prm;
    memset(&prm, 0, sizeof(prm));
    if (pl.num_passes == 0) {
        // N == 1: the transform is the identity (the reference runs zero stages, dit.rs:44-65).
        if (io.in_re != io.out_re || io.in_il != io.out_il || scale != T(1))
            return fail(PHASTFT_ERR_INVALID_ARG, "N == 1 supports only the in-place unscaled form");
        return PHASTFT_OK;
    }
    const bool use_alt_row = pl.alt_row.k != nullptr && batch >= pl.alt_row_min_batch;
    if (pl.num_passes == 1 || use_alt_row) {
        const int which = use_alt_row ? ALT_ROW_PASS : 0;
        size_t done = 0;
        const size_t max_chunk = (size_t)1 << 24;
        while (done < batch) {
            size_t nb = std::min(batch - done, max_chunk);
            prm.in_re = io.in_re + (io.in_il ? 2 : 1) * done * io.in_bstride;
            prm.in_im = io.in_im ? io.in_im + done * io.in_bstride : nullptr;
            prm.out_re = io.out_re + (io.out_il ? 2 : 1) * done * io.out_bstride;
            prm.out_im = io.out_im ? io.out_im + done * io.out_bstride : nullptr;
            prm.in_bstride = io.in_bstride; prm.out_bstride = io.out_bstride;
            prm.in_interleaved = io.in_il; prm.out_interleaved = io.out_il;
            prm.scale = scale;
            if (pass_events && done == 0) CUDA_TRY(cudaEventRecord(pass_events[0], stream));
            int32_t st = launch_pass(pl, which, prm, nb, stream);
            if (st) return st;
            if (pass_events && done == 0) {
                CUDA_TRY(cudaEventRecord(pass_events[1], stream));
                for (int q = 2; q <= pl.num_passes; ++q) CUDA_TRY(cudaEventRecord(pass_events[q], stream));
            }
            done += nb;
        }
        return PHASTFT_OK;
    }
    // ---- both passes in one cluster launch: no workspace, HBM sees the batch once in and once out ----------------
    if (pl.cl && batch >= pl.cl_min_batch) {
        const size_t max_chunk = (size_t(1) << 30) / (size_t)pl.cl->K;        // grid = transforms x K CTAs
        for (size_t done = 0; done < batch; done += max_chunk) {
            const size_t nb = std::min(batch - done, max_chunk);
            PassParams<T> b1, b2, p1, p2;
            memset(&b1, 0, sizeof(b1)); memset(&b2, 0, sizeof(b2));
            b1.scale = T(1);
            b1.in_re = io.in_re + (io.in_il ? 2 : 1) * done * io.in_bstride;
            b1.in_im = io.in_im ? io.in_im + done * io.in_bstride : nullptr;
            b1.in_bstride = io.in_bstride; b1.in_interleaved = io.in_il;
            b1.xch_log2P2 = pl.cl_pass[1].log2R;
            b1.xch_log2CB = ilog2((size_t)pl.cl->k2.C);
            b2.out_re = io.out_re + (io.out_il ? 2 : 1) * done * io.out_bstride;
            b2.out_im = io.out_im ? io.out_im + done * io.out_bstride : nullptr;
            b2.out_bstride = io.out_bstride; b2.out_interleaved = io.out_il;
            b2.scale = scale;
            const KernelEntry<T>* k1 = nullptr; const KernelEntry<T>* k2 = nullptr;
            unsigned long long t1 = 0, t2 = 0;
            int32_t st = prepare_pass_desc(pl, pl.cl_pass[0], 0, b1, nb, 0, -1, p1, k1, t1);
            if (!st) st = prepare_pass_desc(pl, pl.cl_pass[1], 1, b2, nb, 0, -1, p2, k2, t2);
            if (st) return st;
            if (t1 != t2 || t1 != (unsigned long long)nb * pl.cl->K) return fail(PHASTFT_ERR_INVALID_ARG, "cluster plan: tile count mismatch");
            void* args[] = {&p1, &p2};
            cudaLaunchConfig_t cfg;
            memset(&cfg, 0, sizeof(cfg));
            cfg.gridDim = dim3((unsigned)t1); cfg.blockDim = dim3((unsigned)pl.cl->NT); cfg.dynamicSmemBytes = pl.cl->smem; cfg.stream = stream;
            cudaLaunchAttribute attr[1];
            attr[0].id = cudaLaunchAttributeClusterDimension;
            attr[0].val.clusterDim.x = (unsigned)pl.cl->K; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
            cfg.attrs = attr; cfg.numAttrs = 1;
            if (pass_events && done == 0) CUDA_TRY(cudaEventRecord(pass_events[0], stream));
            CUDA_TRY(cudaLaunchKernelExC(&cfg, pl.cl->fn, args));
            note_launch({"CLUSTER", pl.cl->k1.R, pl.cl->k2.R, pl.cl->K, pl.cl->NT, pl.cl->variant, "cluster", false});
            if (pass_events && done == 0)
                for (int q = 1; q <= pl.num_passes; ++q) CUDA_TRY(cudaEventRecord(pass_events[q], stream));
        }
        return PHASTFT_OK;
    }
    // multi-pass: in -> ws (COL) [-> ws (COL)] -> out (TRANS), batch processed in L2-sized chunks
    std::lock_guard<std::mutex> lock(pl.mu);
    const size_t chunk = chunk_transforms(pl, batch);
    // pipelined two-pass launch (see fft_pipe2_kernel): the workspace is a ring of transforms instead of the whole chunk
    const PipeEntry<T>* pipe = nullptr;
    if (pl.num_passes == 2 && !pass_events) {
        if (batch > 1 && (batch << pl.log2n) >= (size_t(1) << 21)) pipe = pl.pipe_b;
        else if (batch == 1 && io.in_il == 0 && io.out_il == 0 && !io.pre_log2half) pipe = pl.pipe_1;
    }
    size_t ws_need = chunk;
    const size_t ring = pipe ? pipe_ring_transforms(pl, batch) : 0;
    if (pipe) ws_need = ring;
    // Workspace reuse is ordered by the stream itself when consecutive calls use the same stream;
    // a call on a different stream first waits for the previous user.  While `stream` is being
    // captured into a CUDA graph the cross-stream bookkeeping is skipped (the graph's owner orders
    // replays against other users of the plan).
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    CUDA_TRY(cudaStreamIsCapturing(stream, &cap));
    const bool capturing = cap != cudaStreamCaptureStatusNone;
    if (pl.ws_elems < ws_need * pl.n || (pipe && pl.pipe_state_batch < batch)) {
        // The plan is created with room for one transform; the first batched call grows it (synchronising).
        // phastft_plan_dit_*_reserve(batch) does this ahead of time; inside a graph capture growing is an error.
        if (capturing)
            return fail(PHASTFT_ERR_INVALID_ARG, "the plan's workspace is too small for this batch and the stream is being captured: "
                                                 "call phastft_plan_dit_*_reserve(batch) before capturing");
        int32_t st = grow_workspace(pl, ws_need, stream);
        if (st) return st;
        if (pipe && pl.pipe_state_batch < batch) {
            CUDA_TRY(cudaStreamSynchronize(stream));
            if (pl.pipe_state) cudaFree(pl.pipe_state);
            pl.pipe_state = nullptr; pl.pipe_state_batch = 0;
            const size_t cap = std::max<size_t>(batch, 4096);
            CUDA_TRY(cudaMalloc(&pl.pipe_state, 64 + 2 * cap * sizeof(unsigned)));
            pl.pipe_state_batch = cap;
            CUDA_TRY(scribble_new(pl.scribble_on, pl.pipe_state, 64 + 2 * cap * sizeof(unsigned)));
        }
    }
    if (!capturing && pl.ws_last_stream != stream && pl.ws_used) CUDA_TRY(cudaStreamWaitEvent(stream, pl.ws_free, 0));
    // the part of the workspace this call uses: the pipelined launch's ring (both arrays in one run), else one chunk per array;
    // the pipelined launch's state is zeroed below, the 3-pass group scratch is used whole
    if (pipe) CUDA_TRY(scribble(pl.scribble_on, pl.ws_re, 2 * ring * pl.n * sizeof(T), stream));
    else {
        CUDA_TRY(scribble(pl.scribble_on, pl.ws_re, chunk * pl.n * sizeof(T), stream));
        CUDA_TRY(scribble(pl.scribble_on, pl.ws_im, chunk * pl.n * sizeof(T), stream));
    }
    if (pl.num_passes == 3 && pl.ws2_re) {
        const size_t g2 = (size_t)pl.l2_group * (pl.n >> pl.pass[0].log2R) * sizeof(T);
        CUDA_TRY(scribble(pl.scribble_on, pl.ws2_re, g2, stream));
        CUDA_TRY(scribble(pl.scribble_on, pl.ws2_im, g2, stream));
    }
    const int P = pl.num_passes;
    if (pipe) {
        const bool lone = batch == 1;
        const int il_p = lone ? (pl.ws_il >= 0 ? pl.ws_il : 0) : (pl.ws_il >= 0 ? pl.ws_il : 1);
        PassParams<T> b1, b2, p1, p2;
        memset(&b1, 0, sizeof(b1)); memset(&b2, 0, sizeof(b2));
        b1.scale = T(1);
        b1.in_re = io.in_re; b1.in_im = io.in_im; b1.in_bstride = io.in_bstride; b1.in_interleaved = io.in_il;
        b1.out_re = pl.ws_re; b1.out_im = pl.ws_re + ring * pl.n; b1.out_bstride = (long long)pl.n; b1.out_interleaved = il_p;
        b1.out_ring = (int)ring;
        b2.in_re = pl.ws_re; b2.in_im = pl.ws_re + ring * pl.n; b2.in_bstride = (long long)pl.n; b2.in_interleaved = il_p;
        b2.in_ring = (int)ring;
        b2.out_re = io.out_re; b2.out_im = io.out_im; b2.out_bstride = io.out_bstride; b2.out_interleaved = io.out_il;
        b2.scale = scale;
        const KernelEntry<T>* k1 = nullptr; const KernelEntry<T>* k2 = nullptr;
        unsigned long long t1 = 0, t2 = 0;
        // descriptors with the batch flavour of each pass's kernel (prepare_pass picks kb for many-transform calls)
        int32_t st = prepare_pass(pl, 0, b1, batch, 0, -1, p1, k1, t1);
        if (!st) st = prepare_pass(pl, 1, b2, batch, 0, -1, p2, k2, t2);
        if (st) return st;
        if (k1->R != pipe->R1 || k1->C != pipe->C1 || k2->R != pipe->R2 || k2->C != pipe->C2)
            return fail(PHASTFT_ERR_INVALID_ARG, "pipelined launch: kernel pair does not match the plan");
        if (pipe->mode == 1) {
            const size_t B = size_t(1) << p1.log2B;
            const bool ok_align = io.in_il == 0 && il_p == 1 && ((reinterpret_cast<uintptr_t>(io.in_re) | reinterpret_cast<uintptr_t>(io.in_im)) & 15) == 0 &&
                                  ((size_t)io.in_bstride * sizeof(T)) % 16 == 0;
            if (!ok_align) return fail(PHASTFT_ERR_INVALID_ARG, "pipelined launch with TMA input needs planar 16-byte-aligned input (unset PHASTFT_PIPE_TMA)");
            const unsigned box_rows = (unsigned)std::min(k1->R, 256);
            if (!encode_tile_map<T>(&p1.tmap_re, p1.in_re, B, (size_t)k1->R, B, batch, (size_t)p1.in_bstride, (unsigned)k1->C, box_rows) ||
                !encode_tile_map<T>(&p1.tmap_im, p1.in_im, B, (size_t)k1->R, B, batch, (size_t)p1.in_bstride, (unsigned)k1->C, box_rows))
                return fail(PHASTFT_ERR_CUDA, "cuTensorMapEncodeTiled failed");
        }
        PipeCtl ctl;
        ctl.ticket = reinterpret_cast<unsigned*>(pl.pipe_state);
        ctl.done1 = reinterpret_cast<unsigned*>(pl.pipe_state + 64);
        ctl.done2 = ctl.done1 + pl.pipe_state_batch;
        ctl.tiles1 = (unsigned)(t1 / batch); ctl.tiles2 = (unsigned)(t2 / batch);
        ctl.batch = (unsigned)batch; ctl.ring = (unsigned)ring;
        ctl.delay = lone ? 1u : (unsigned)std::max<size_t>(1, ring / 2);
        ctl.discard = (pl.pipe_discard && il_p == 1 && !lone) ? 1 : 0;
        CUDA_TRY(cudaMemsetAsync(pl.pipe_state, 0, 64 + 2 * pl.pipe_state_batch * sizeof(unsigned), stream));
        const unsigned long long items = (unsigned long long)(batch + ctl.delay) * (ctl.tiles1 + ctl.tiles2);
        if (items > 0x7fffffffULL) return fail(PHASTFT_ERR_INVALID_ARG, "grid too large");
        const unsigned grid = (unsigned)items;                               // one CTA per work item (a ticket decides which)
        void* args[] = {&p1, &p2, &ctl};
        CUDA_TRY(cudaLaunchKernel(pipe->fn, dim3(grid), dim3(pipe->NT), args, pipe->smem, stream));
        note_launch({"PIPE", pipe->R1, pipe->R2, pipe->C1, pipe->NT, 0, pipe->mode ? "pipe-tma" : "pipe", false});
        if (!capturing) {
            CUDA_TRY(cudaEventRecord(pl.ws_free, stream));
            pl.ws_last_stream = stream;
            pl.ws_used = true;
        }
        return PHASTFT_OK;
    }
    // ---- 3-pass plans: pass 1 streams the whole signal HBM -> HBM; passes 2+3 then run per group of
    // G consecutive k1 values (G * N/R1 elements ~ tens of MiB): pass 2 writes its result into a small
    // reused scratch that stays L2-resident and pass 3 reads it back from L2, so the tail costs one
    // HBM read + one HBM write instead of two of each.
    if (P == 3 && pl.ws2_re != nullptr) {
        const long long R1 = 1LL << pl.pass[0].log2R;
        const long long sub = (long long)(pl.n >> pl.pass[0].log2R);    // elements per k1
        const long long G = pl.l2_group;
        for (size_t b = 0; b < batch; ++b) {
            memset(&prm, 0, sizeof(prm));
            prm.scale = T(1);
            prm.in_re = io.in_re + (io.in_il ? 2 : 1) * b * io.in_bstride;
            prm.in_im = io.in_im ? io.in_im + b * io.in_bstride : nullptr;
            prm.in_bstride = io.in_bstride; prm.in_interleaved = io.in_il;
            prm.pre_tw2 = io.pre_tw2; prm.pre_log2half = io.pre_log2half;
                if (io.pre_wc) memcpy(prm.pre_wc, io.pre_wc, sizeof(prm.pre_wc));
            prm.out_re = pl.ws_re; prm.out_im = pl.ws_im; prm.out_bstride = (long long)pl.n;
            if (pass_events && b == 0) CUDA_TRY(cudaEventRecord(pass_events[0], stream));
            int32_t st = launch_pass(pl, 0, prm, 1, stream);
            if (st) return st;
            if (pass_events && b == 0) CUDA_TRY(cudaEventRecord(pass_events[1], stream));
            for (long long k1 = 0; k1 < R1; k1 += G) {
                memset(&prm, 0, sizeof(prm));
                prm.scale = T(1);
                prm.in_re = pl.ws_re; prm.in_im = pl.ws_im; prm.in_bstride = (long long)pl.n;
                prm.out_re = pl.ws2_re - k1 * sub; prm.out_im = pl.ws2_im - k1 * sub; prm.out_bstride = (long long)pl.n;
                st = launch_pass(pl, 1, prm, 1, stream, k1, G);
                if (st) return st;
                memset(&prm, 0, sizeof(prm));
                prm.in_re = pl.ws2_re - k1 * sub; prm.in_im = pl.ws2_im - k1 * sub; prm.in_bstride = (long long)pl.n;
                prm.out_re = io.out_re + (io.out_il ? 2 : 1) * b * io.out_bstride;
                prm.out_im = io.out_im ? io.out_im + b * io.out_bstride : nullptr;
                prm.out_bstride = io.out_bstride; prm.out_interleaved = io.out_il;
                prm.scale = scale;
                st = launch_pass(pl, 2, prm, 1, stream, k1, G);
                if (st) return st;
            }
            if (pass_events && b == 0) { CUDA_TRY(cudaEventRecord(pass_events[2], stream)); CUDA_TRY(cudaEventRecord(pass_events[3], stream)); }
        }
        if (!capturing) {
            CUDA_TRY(cudaEventRecord(pl.ws_free, stream));
            pl.ws_last_stream = stream;
            pl.ws_used = true;
        }
        return PHASTFT_OK;
    }
    const bool many_call = batch > 1 && (batch << pl.log2n) >= (size_t(1) << 21);
    // asynchronous-input kernels: planar 16-byte-aligned input whose batch stride keeps the alignment, interleaved intermediates
    // batches: from 32 MiB of signal per array (2^22 f64 / 2^23 f32 points) -- below that the grid is about one wave and the pair
    // measured equal or a few per cent slower
    const bool tma_many = many_call && pl.tma_batch && (batch << pl.log2n) * sizeof(T) >= (size_t(32) << 20);
    const bool tma = P == 2 && pl.pass[0].kt && pl.pass[1].kt && (many_call ? tma_many : pl.tma_lone) && io.in_il == 0 && pl.ws_il != 0 && !io.pre_log2half &&
                     ((reinterpret_cast<uintptr_t>(io.in_re) | reinterpret_cast<uintptr_t>(io.in_im)) & 15) == 0 &&
                     (batch == 1 || ((size_t)io.in_bstride * sizeof(T)) % 16 == 0);
    const int il = tma ? 1 : pl.ws_il >= 0 ? pl.ws_il : ((P == 3 || many_call) ? 1 : 0);
    for (size_t done = 0; done < batch; done += chunk) {
        const size_t nb = std::min(chunk, batch - done);
        for (int p = 0; p < P; ++p) {
            memset(&prm, 0, sizeof(prm));
            prm.scale = T(1);
            if (p == 0) {
                prm.in_re = io.in_re + (io.in_il ? 2 : 1) * done * io.in_bstride;
                prm.in_im = io.in_im ? io.in_im + done * io.in_bstride : nullptr;
                prm.in_bstride = io.in_bstride;
                prm.in_interleaved = io.in_il;
                prm.pre_tw2 = io.pre_tw2; prm.pre_log2half = io.pre_log2half;
                // the W_(2 R1) factors for the first radix of the build that runs: kcb on a multi-wave chunk, else kc
                const double2* wc = (io.pre_wc_b && pass_takes_kb(pl, pl.pass[0], nb)) ? io.pre_wc_b : io.pre_wc;
                if (wc) memcpy(prm.pre_wc, wc, sizeof(prm.pre_wc));
            } else {
                prm.in_re = pl.ws_re; prm.in_im = pl.ws_im; prm.in_bstride = (long long)pl.n;
                prm.in_interleaved = il;
            }
            if (p == P - 1) {
                prm.out_re = io.out_re + (io.out_il ? 2 : 1) * done * io.out_bstride;
                prm.out_im = io.out_im ? io.out_im + done * io.out_bstride : nullptr;
                prm.out_bstride = io.out_bstride;
                prm.out_interleaved = io.out_il;
                prm.scale = scale;
            } else {
                prm.out_re = pl.ws_re; prm.out_im = pl.ws_im; prm.out_bstride = (long long)pl.n;
                prm.out_interleaved = il;
            }
            if (pass_events && done == 0 && p == 0) CUDA_TRY(cudaEventRecord(pass_events[0], stream));
            bool tma3 = false;
            if (P == 3 && pl.pass[p].kt != nullptr && il == 1 && nb == 1) {
                if (p == 0) tma3 = io.in_il == 0 && !io.pre_log2half && ((reinterpret_cast<uintptr_t>(prm.in_re) | reinterpret_cast<uintptr_t>(prm.in_im)) & 15) == 0;
                else tma3 = true;
            }
            int32_t st = launch_pass(pl, p, prm, nb, stream, 0, -1, tma || tma3);
            if (st) return st;
            if (pass_events && done == 0) CUDA_TRY(cudaEventRecord(pass_events[p + 1], stream));
        }
    }
    if (!capturing) {
        CUDA_TRY(cudaEventRecord(pl.ws_free, stream));
        pl.ws_last_stream = stream;
        pl.ws_used = true;
    }
    return PHASTFT_OK;
}

// The kernels move interleaved data as (re, im) pairs: one 2 * sizeof(T)-byte access per complex value.  A pointer the
// device entry points read or write that way must be aligned to it (the host-slice entry points stage through aligned
// plan buffers).
template <typename T>
int32_t check_pair_alignment(const T* p, const char* what) {
    if (reinterpret_cast<uintptr_t>(p) % (2 * sizeof(T)) == 0) return PHASTFT_OK;
    return fail(PHASTFT_ERR_INVALID_ARG, std::string(what) + " must be aligned to " + std::to_string(2 * sizeof(T)) +
                                             " bytes (it is accessed as interleaved (re, im) pairs)");
}

template <typename T>
int32_t check_c2c_args(const Plan<T>* pl, size_t len_re, size_t len_im, int direction) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (len_re != len_im) return fail(PHASTFT_ERR_LEN_MISMATCH);                      // dit.rs:284
    if (!is_pow2(len_re)) return fail(PHASTFT_ERR_NOT_POW2);                          // dit.rs:285
    if (ilog2(len_re) != pl->log2n) return fail(PHASTFT_ERR_PLAN_MISMATCH);           // dit.rs:289
    if (direction != PHASTFT_FORWARD && direction != PHASTFT_REVERSE) return fail(PHASTFT_ERR_INVALID_ARG, "direction must be 1 or -1");
    return PHASTFT_OK;
}

// planar, in place, device pointers ------------------------------------------------------------------
template <typename T>
int32_t fft_dev(const Plan<T>* pl, T* d_re, T* d_im, int direction, size_t batch, size_t bstride, cudaStream_t stream,
                cudaEvent_t* pass_events = nullptr) {
    if (!pl || !d_re || !d_im) return fail(PHASTFT_ERR_INVALID_ARG, "NULL argument");
    if (direction != PHASTFT_FORWARD && direction != PHASTFT_REVERSE) return fail(PHASTFT_ERR_INVALID_ARG, "direction must be 1 or -1");
    if (batch > 1 && bstride < pl->n) return fail(PHASTFT_ERR_INVALID_ARG, "batch_stride < N");
    DeviceGuard g(pl->device);
    Io<T> io;
    // inverse via the swap trick (algorithms/dit.rs:297-300): forward transform of (imags, reals), then 1/N
    if (direction == PHASTFT_FORWARD) { io.in_re = d_re; io.in_im = d_im; io.out_re = d_re; io.out_im = d_im; }
    else { io.in_re = d_im; io.in_im = d_re; io.out_re = d_im; io.out_im = d_re; }
    io.in_bstride = io.out_bstride = (long long)bstride;
    io.in_il = io.out_il = 0;
    const T scale = direction == PHASTFT_REVERSE ? T(1) / (T)pl->n : T(1);   // dit.rs:326
    if (pl->num_passes == 0) return PHASTFT_OK;
    return run_c2c(*pl, io, batch, scale, stream, pass_events);
}

// One profiled call: per-pass device time from CUDA events on the launching stream (synchronises).
template <typename T>
int32_t fft_dev_profile(const Plan<T>* pl, T* d_re, T* d_im, int direction, size_t batch, size_t bstride,
                        cudaStream_t stream, float* pass_ms, int* num_passes) {
    if (!pl || !pass_ms || !num_passes) return fail(PHASTFT_ERR_INVALID_ARG, "NULL argument");
    DeviceGuard g(pl->device);
    *num_passes = pl->num_passes;
    cudaEvent_t ev[MAX_PASSES + 1];
    for (int i = 0; i <= pl->num_passes; ++i) CUDA_TRY(cudaEventCreate(&ev[i]));
    int32_t st = fft_dev(pl, d_re, d_im, direction, batch, bstride, stream, ev);
    if (st == PHASTFT_OK && pl->num_passes > 0) {
        cudaError_t e = cudaEventSynchronize(ev[pl->num_passes]);
        if (e != cudaSuccess) st = fail(PHASTFT_ERR_CUDA, cudaGetErrorString(e));
        for (int i = 0; i < pl->num_passes && st == PHASTFT_OK; ++i) cudaEventElapsedTime(&pass_ms[i], ev[i], ev[i + 1]);
    }
    for (int i = 0; i <= pl->num_passes; ++i) cudaEventDestroy(ev[i]);
    return st;
}

template <typename T>
int32_t fft_interleaved_dev(const Plan<T>* pl, T* d_sig, int direction, size_t batch, size_t bstride, cudaStream_t stream) {
    if (!pl || !d_sig) return fail(PHASTFT_ERR_INVALID_ARG, "NULL argument");
    if (direction != PHASTFT_FORWARD && direction != PHASTFT_REVERSE) return fail(PHASTFT_ERR_INVALID_ARG, "direction must be 1 or -1");
    if (batch > 1 && bstride < pl->n) return fail(PHASTFT_ERR_INVALID_ARG, "batch_stride < N");
    if (int32_t st = check_pair_alignment(d_sig, "d_signal")) return st;
    DeviceGuard g(pl->device);
    if (pl->num_passes == 0) return PHASTFT_OK;
    Io<T> io;
    io.in_re = d_sig; io.in_im = nullptr; io.out_re = d_sig; io.out_im = nullptr;
    io.in_bstride = io.out_bstride = (long long)bstride;
    io.in_il = io.out_il = direction == PHASTFT_FORWARD ? 1 : 2;
    const T scale = direction == PHASTFT_REVERSE ? T(1) / (T)pl->n : T(1);
    return run_c2c(*pl, io, batch, scale, stream);
}

template <typename T>
int32_t ensure_staging(const Plan<T>* pl, size_t elems) {
    if (pl->stage_elems >= elems) return PHASTFT_OK;
    if (pl->stage_re) cudaFree(pl->stage_re);
    if (pl->stage_im) cudaFree(pl->stage_im);
    pl->stage_re = pl->stage_im = nullptr; pl->stage_elems = 0;
    CUDA_TRY(cudaMalloc(&pl->stage_re, elems * sizeof(T)));
    CUDA_TRY(cudaMalloc(&pl->stage_im, elems * sizeof(T)));
    pl->stage_elems = elems;
    return PHASTFT_OK;
}

// host slices: H2D, run, D2H, synchronous (lib.rs:143-150 semantics) ----------------------------------
template <typename T>
int32_t fft_host(const Plan<T>* pl, T* re, size_t len_re, T* im, size_t len_im, int direction) {
    int32_t st = check_c2c_args(pl, len_re, len_im, direction);
    if (st) return st;
    if (!re || !im) return fail(PHASTFT_ERR_INVALID_ARG, "NULL slice");
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> host_lock(pl->host_mu);   // planners are shared by reference between threads
    {
        std::lock_guard<std::mutex> lock(pl->mu);
        st = ensure_staging(pl, pl->n);
        if (st) return st;
    }
    const size_t bytes = pl->n * sizeof(T);
    CUDA_TRY(scribble(pl->scribble_on, pl->stage_re, bytes, pl->stream));
    CUDA_TRY(scribble(pl->scribble_on, pl->stage_im, bytes, pl->stream));
    CUDA_TRY(cudaMemcpyAsync(pl->stage_re, re, bytes, cudaMemcpyHostToDevice, pl->stream));
    CUDA_TRY(cudaMemcpyAsync(pl->stage_im, im, bytes, cudaMemcpyHostToDevice, pl->stream));
    st = fft_dev(pl, pl->stage_re, pl->stage_im, direction, 1, pl->n, pl->stream);
    if (st) return st;
    CUDA_TRY(cudaMemcpyAsync(re, pl->stage_re, bytes, cudaMemcpyDeviceToHost, pl->stream));
    CUDA_TRY(cudaMemcpyAsync(im, pl->stage_im, bytes, cudaMemcpyDeviceToHost, pl->stream));
    CUDA_TRY(cudaStreamSynchronize(pl->stream));
    return PHASTFT_OK;
}

template <typename T>
int32_t fft_interleaved_host(const Plan<T>* pl, T* sig, size_t len_complex, int direction) {
    int32_t st = check_c2c_args(pl, len_complex, len_complex, direction);
    if (st) return st;
    if (!sig) return fail(PHASTFT_ERR_INVALID_ARG, "NULL slice");
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> host_lock(pl->host_mu);
    {
        std::lock_guard<std::mutex> lock(pl->mu);
        st = ensure_staging(pl, 2 * pl->n);
        if (st) return st;
    }
    const size_t bytes = 2 * pl->n * sizeof(T);
    CUDA_TRY(scribble(pl->scribble_on, pl->stage_re, bytes, pl->stream));
    CUDA_TRY(cudaMemcpyAsync(pl->stage_re, sig, bytes, cudaMemcpyHostToDevice, pl->stream));
    st = fft_interleaved_dev(pl, pl->stage_re, direction, 1, pl->n, pl->stream);
    if (st) return st;
    CUDA_TRY(cudaMemcpyAsync(sig, pl->stage_re, bytes, cudaMemcpyDeviceToHost, pl->stream));
    CUDA_TRY(cudaStreamSynchronize(pl->stream));
    return PHASTFT_OK;
}

// One-shot calls build their planner per call, like the reference (lib.rs:180-183).  Building is cheap, but
// allocating and releasing the workspace and staging buffers is not (130 ms per 2^24 f64 call), so the most
// recent one-shot plan per precision is kept and reused when the next call has the same size and device;
// phastft_oneshot_cache_clear() releases it.  The cache entry is held under its lock for the whole call.
template <class P>
struct OneShotCache {
    std::mutex mu;
    P* plan = nullptr;          // intentionally not freed at process exit (the CUDA context may be gone by then)
    size_t n = 0;
    int device = -1;
    void clear() {
        std::lock_guard<std::mutex> lock(mu);
        delete plan;
        plan = nullptr; n = 0; device = -1;
    }
};
template <typename T> OneShotCache<Plan<T>>& oneshot_c2c_cache() { static auto* c = new OneShotCache<Plan<T>>(); return *c; }

template <typename T>
int32_t fft_oneshot(T* re, size_t len_re, T* im, size_t len_im, int direction, int device) {
    if (!is_pow2(len_re)) return fail(PHASTFT_ERR_NOT_POW2);
    auto& c = oneshot_c2c_cache<T>();
    std::lock_guard<std::mutex> lock(c.mu);
    if (!c.plan || c.n != len_re || c.device != device) {
        delete c.plan;
        c.plan = nullptr; c.n = 0; c.device = -1;
        int32_t st = build_plan<T>(len_re, device, &c.plan);
        if (st) return st;
        c.n = len_re; c.device = device;
    }
    return fft_host(c.plan, re, len_re, im, len_im, direction);
}

// Host-resident batch, sharded over the plans' devices (contiguous ranges, SURVEY.md 8e; no collective on
// the data path).  Per device the shard moves through a three-slot pipeline -- H2D of chunk j+1, the FFTs of
// chunk j and D2H of chunk j-1 run on three streams -- so both PCIe directions are busy at once; a chunk is
// ~16 MiB per array (PHASTFT_HOST_CHUNK_MB).  Overlap needs page-locked host memory; pageable memory is
// still correct, the copies just serialise.
template <typename T>
int32_t batch_sharded_host(Plan<T>* const* plans, int num_plans, T* re, T* im, size_t batch, size_t bstride, int direction) {
    if (!plans || num_plans <= 0 || !re || !im) return fail(PHASTFT_ERR_INVALID_ARG, "NULL argument");
    if (direction != PHASTFT_FORWARD && direction != PHASTFT_REVERSE) return fail(PHASTFT_ERR_INVALID_ARG, "direction must be 1 or -1");
    for (int g = 0; g < num_plans; ++g)
        if (!plans[g]) return fail(PHASTFT_ERR_INVALID_ARG, "NULL plan in the plan list");
    const size_t n = plans[0]->n;
    for (int g = 0; g < num_plans; ++g)
        if (plans[g]->n != n) return fail(PHASTFT_ERR_PLAN_MISMATCH);
    if (bstride < n) return fail(PHASTFT_ERR_INVALID_ARG, "batch_stride < N");
    if (batch == 0) return PHASTFT_OK;
    std::vector<std::mutex*> locks;
    for (int g = 0; g < num_plans; ++g) locks.push_back(&plans[g]->host_mu);
    std::sort(locks.begin(), locks.end(), std::less<std::mutex*>());
    locks.erase(std::unique(locks.begin(), locks.end()), locks.end());
    if (locks.size() != (size_t)num_plans) return fail(PHASTFT_ERR_INVALID_ARG, "the same plan passed twice");
    struct Unlock { std::vector<std::mutex*>& l; ~Unlock() { for (auto* m : l) m->unlock(); } };
    for (auto* m : locks) m->lock();                         // address order: no deadlock between overlapping calls
    Unlock unlock_all{locks};
    constexpr int NSLOT = 3;
    size_t chunk_mb = 16;
    if (const char* e = getenv("PHASTFT_HOST_CHUNK_MB")) { long v = atol(e); if (v > 0) chunk_mb = (size_t)v; }
    const size_t per_chunk = std::max<size_t>(1, (chunk_mb << 20) / (n * sizeof(T)));   // transforms per chunk
    struct Shard {
        const Plan<T>* pl; size_t lo, nb, chunks; size_t slot_elems;
        cudaEvent_t h2d_done[NSLOT], fft_done[NSLOT], d2h_done[NSLOT];
        bool ev = false;
    };
    std::vector<Shard> sh(num_plans);
    auto cleanup = [&]() {
        for (auto& s : sh)
            if (s.ev) {
                DeviceGuard guard(s.pl->device);
                for (int k = 0; k < NSLOT; ++k)
                    for (cudaEvent_t e : {s.h2d_done[k], s.fft_done[k], s.d2h_done[k]}) if (e) cudaEventDestroy(e);
                s.ev = false;
            }
    };
    size_t max_chunks = 0;
    for (int g = 0; g < num_plans; ++g) {
        Shard& s = sh[g];
        s.pl = plans[g];
        s.lo = batch * g / num_plans;
        s.nb = batch * (g + 1) / num_plans - s.lo;
        const size_t pc = std::min(per_chunk, std::max<size_t>(1, s.nb));
        s.chunks = (s.nb + pc - 1) / pc;
        s.slot_elems = pc * n;
        max_chunks = std::max(max_chunks, s.chunks);
        if (!s.nb) continue;
        DeviceGuard guard(s.pl->device);
        {
            std::lock_guard<std::mutex> lock(s.pl->mu);
            int32_t st = ensure_staging(s.pl, std::min<size_t>(NSLOT, s.chunks) * s.slot_elems);
            if (st) { cleanup(); return st; }
            if (!s.pl->stream_h2d) {
                if (cudaStreamCreateWithFlags(&s.pl->stream_h2d, cudaStreamNonBlocking) != cudaSuccess ||
                    cudaStreamCreateWithFlags(&s.pl->stream_d2h, cudaStreamNonBlocking) != cudaSuccess) { cleanup(); return fail(PHASTFT_ERR_CUDA, "stream create"); }
            }
        }
        bool ev_ok = true;
        for (int k = 0; k < NSLOT; ++k) { s.h2d_done[k] = s.fft_done[k] = s.d2h_done[k] = nullptr; }
        for (int k = 0; k < NSLOT; ++k) {
            ev_ok &= cudaEventCreateWithFlags(&s.h2d_done[k], cudaEventDisableTiming) == cudaSuccess;
            ev_ok &= cudaEventCreateWithFlags(&s.fft_done[k], cudaEventDisableTiming) == cudaSuccess;
            ev_ok &= cudaEventCreateWithFlags(&s.d2h_done[k], cudaEventDisableTiming) == cudaSuccess;
        }
        s.ev = true;
        if (!ev_ok) { (void)cudaGetLastError(); cleanup(); return fail(PHASTFT_ERR_CUDA, "cudaEventCreate"); }
        const size_t staged = std::min<size_t>(NSLOT, s.chunks) * s.slot_elems * sizeof(T);
        if (scribble(s.pl->scribble_on, s.pl->stage_re, staged, s.pl->stream_h2d) != cudaSuccess ||
            scribble(s.pl->scribble_on, s.pl->stage_im, staged, s.pl->stream_h2d) != cudaSuccess) { (void)cudaGetLastError(); cleanup(); return fail(PHASTFT_ERR_CUDA, "cudaMemsetAsync"); }
    }
    // issue chunk j of every device before chunk j+1 of any, so all devices stream concurrently
    int32_t st = PHASTFT_OK;
    for (size_t j = 0; j < max_chunks && !st; ++j) {
        for (int g = 0; g < num_plans && !st; ++g) {
            Shard& s = sh[g];
            if (j >= s.chunks) continue;
            const Plan<T>* pl = s.pl;
            DeviceGuard guard(pl->device);
            const size_t pc = s.slot_elems / n;
            const size_t first = s.lo + j * pc;
            const size_t cnt = std::min(pc, s.lo + s.nb - first);
            const int slot = (int)(j % NSLOT);
            T* d_re = pl->stage_re + (size_t)slot * s.slot_elems;
            T* d_im = pl->stage_im + (size_t)slot * s.slot_elems;
            T* h_re = re + first * bstride;
            T* h_im = im + first * bstride;
            auto ok = [&](cudaError_t e) { if (e != cudaSuccess && !st) st = fail(PHASTFT_ERR_CUDA, cudaGetErrorString(e)); return e == cudaSuccess; };
            if (j >= NSLOT) ok(cudaStreamWaitEvent(pl->stream_h2d, s.d2h_done[slot], 0));     // the slot's previous result has left
            ok(cudaMemcpy2DAsync(d_re, n * sizeof(T), h_re, bstride * sizeof(T), n * sizeof(T), cnt, cudaMemcpyHostToDevice, pl->stream_h2d));
            ok(cudaMemcpy2DAsync(d_im, n * sizeof(T), h_im, bstride * sizeof(T), n * sizeof(T), cnt, cudaMemcpyHostToDevice, pl->stream_h2d));
            ok(cudaEventRecord(s.h2d_done[slot], pl->stream_h2d));
            ok(cudaStreamWaitEvent(pl->stream, s.h2d_done[slot], 0));
            if (!st) st = fft_dev(pl, d_re, d_im, direction, cnt, n, pl->stream);
            ok(cudaEventRecord(s.fft_done[slot], pl->stream));
            ok(cudaStreamWaitEvent(pl->stream_d2h, s.fft_done[slot], 0));
            ok(cudaMemcpy2DAsync(h_re, bstride * sizeof(T), d_re, n * sizeof(T), n * sizeof(T), cnt, cudaMemcpyDeviceToHost, pl->stream_d2h));
            ok(cudaMemcpy2DAsync(h_im, bstride * sizeof(T), d_im, n * sizeof(T), n * sizeof(T), cnt, cudaMemcpyDeviceToHost, pl->stream_d2h));
            ok(cudaEventRecord(s.d2h_done[slot], pl->stream_d2h));
        }
    }
    for (int g = 0; g < num_plans; ++g) {
        if (!sh[g].nb) continue;
        DeviceGuard guard(plans[g]->device);
        cudaError_t e1 = cudaStreamSynchronize(plans[g]->stream_h2d);
        cudaError_t e2 = cudaStreamSynchronize(plans[g]->stream);
        cudaError_t e3 = cudaStreamSynchronize(plans[g]->stream_d2h);
        for (cudaError_t e : {e1, e2, e3})
            if (e != cudaSuccess && !st) st = fail(PHASTFT_ERR_CUDA, cudaGetErrorString(e));
    }
    cleanup();
    return st;
}

// ---- PlannerMode::Tune (planner.rs:25-32: "benchmarks both paths at plan time, picks whichever is faster";
// the reference accepts the mode and ignores it, planner.rs:65).  Here it is real: a handful of pass
// decompositions / tile widths around the heuristic choice are built, timed on a scratch signal with CUDA
// events, and the fastest is kept.
//
// The candidates, host-only (phastft_plan_tune_candidates exposes the same list, so tests can force every plan the
// tuner may pick).  Each entry is stated as it builds: strided tiles exist for 32..1024 rows, a 1024-row tile has no
// CW build (CN is the widest), and the 1024-row middle pass of a 3-pass plan is the half-width CH tile (id 62).
template <typename T>
std::vector<PlanChoice> tune_candidates(int ln) {
    std::vector<PlanChoice> cands;
    if (ln == 0 || choose_factors<T>(ln).size() < 2) return cands;    // one-CTA sizes: nothing to choose
    const int CH = TileC<T>::CH, CN = TileC<T>::CN, CW = TileC<T>::CW;
    auto width = [&](int log2r, int c) { return log2r == 10 ? std::min(c, CN) : c; };
    auto add = [&](std::vector<int> f, std::vector<int> c) {
        for (size_t p = 0; p < f.size(); ++p) c[p] = width(f[p], c[p]);
        if (f.size() == 3 && f[1] == 10) c[1] = CH;
        for (const PlanChoice& q : cands)
            if (q.factors == f && q.pass_c == c) return;
        PlanChoice pc; pc.factors = std::move(f); pc.pass_c = std::move(c); cands.push_back(std::move(pc));
    };
    if (ln <= 20) {
        for (int a : {ln / 2, (ln + 1) / 2})
            for (int c : {CH, CN, CW}) {
                if (a > 10 || ln - a > 10 || a < 5 || ln - a < 5) continue;
                add({a, ln - a}, {c, c});
            }
        if (ln >= 18) add({6, ln - 12, 6}, {CN, CN, CN});
        if (ln >= 19) add({7, ln - 14, 7}, {CN, CN, CN});
    } else {
        for (int e : {7, 8, 9}) {
            const int m = ln - 2 * e;
            if (m < 5 || m > 10) continue;
            add({e, m, e}, {CW, CN, CW});
            add({e, m, e}, {CN, CN, CN});
        }
        if (ln - 18 >= 5 && ln - 18 <= 10) { add({10, ln - 18, 8}, {CN, CN, CW}); add({8, ln - 18, 10}, {CW, CN, CN}); }
    }
    return cands;
}

template <typename T>
int32_t build_plan_tuned(size_t n, int device, Plan<T>** out) {
    if (!out) return fail(PHASTFT_ERR_INVALID_ARG, "out == NULL");
    *out = nullptr;
    int32_t st = build_plan<T>(n, device, out);             // the heuristic plan (also validates n / device)
    if (st) return st;
    Plan<T>* best = *out;
    const int ln = best->log2n;
    if (best->num_passes < 2) return PHASTFT_OK;            // one-CTA sizes: nothing to choose
    DeviceGuard guard(device);
    const std::vector<PlanChoice> cands = tune_candidates<T>(ln);
    T *re = nullptr, *im = nullptr;
    if (cudaMalloc(&re, n * sizeof(T)) != cudaSuccess || cudaMalloc(&im, n * sizeof(T)) != cudaSuccess) {
        cudaGetLastError();
        if (re) cudaFree(re);
        return PHASTFT_OK;                                   // no room to tune: keep the heuristic plan
    }
    cudaMemset(re, 0, n * sizeof(T)); cudaMemset(im, 0, n * sizeof(T));
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    auto time_plan = [&](Plan<T>* pl) -> float {
        const int reps = ln <= 20 ? 20 : (ln <= 24 ? 5 : 2);
        for (int w = 0; w < 2; ++w) if (fft_dev(pl, re, im, PHASTFT_FORWARD, 1, n, pl->stream) != PHASTFT_OK) return 1e30f;
        cudaEventRecord(e0, pl->stream);
        for (int r = 0; r < reps; ++r) fft_dev(pl, re, im, PHASTFT_FORWARD, 1, n, pl->stream);
        cudaEventRecord(e1, pl->stream);
        if (cudaEventSynchronize(e1) != cudaSuccess) return 1e30f;
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        return ms / reps;
    };
    float best_ms = time_plan(best);
    for (const PlanChoice& pc : cands) {
        Plan<T>* cand = nullptr;
        g_choice = &pc;
        int32_t cst = build_plan<T>(n, device, &cand);
        g_choice = nullptr;
        if (cst != PHASTFT_OK || !cand) { delete cand; continue; }
        if (cand->description == best->description) { delete cand; continue; }
        const float ms = time_plan(cand);
        if (ms < best_ms * 0.98f) { delete best; best = cand; best_ms = ms; } else delete cand;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    cudaFree(re); cudaFree(im);
    best->description += " [tuned]";
    g_last_error.clear();
    *out = best;
    return PHASTFT_OK;
}

// ---- table blob export / import / broadcast ------------------------------------------------------------
template <typename T>
int32_t tables_export(const Plan<T>* pl, void* dst, cudaStream_t s) {
    if (!pl || !dst) return fail(PHASTFT_ERR_INVALID_ARG, "NULL argument");
    DeviceGuard g(pl->device);
    CUDA_TRY(cudaMemcpyAsync(dst, pl->blob_dev, pl->blob_host.size(), cudaMemcpyDeviceToDevice, s));
    return PHASTFT_OK;
}
// Compares a blob header (already on the host) with the plan's own.
template <typename T>
int32_t check_blob_header(const Plan<T>* pl, const BlobHeader& h) {
    BlobHeader mine;
    memcpy(&mine, pl->blob_host.data(), sizeof(mine));
    if (h.magic != BLOB_MAGIC) return fail(PHASTFT_ERR_PLAN_MISMATCH, "table blob: bad magic (not a phastft table blob)");
    if (h.n != mine.n || h.precision_bits != mine.precision_bits) return fail(PHASTFT_ERR_PLAN_MISMATCH, "table blob is for another size / precision");
    if (h.bytes != mine.bytes || h.num_passes != mine.num_passes || h.layout_sig != mine.layout_sig ||
        memcmp(h.tw_stage_off, mine.tw_stage_off, sizeof(h.tw_stage_off)) || memcmp(h.tw32_off, mine.tw32_off, sizeof(h.tw32_off)))
        return fail(PHASTFT_ERR_PLAN_MISMATCH, "table blob was laid out for a different pass decomposition / kernel choice "
                                               "(PlannerMode::Tune or a PHASTFT_* override on one rank only?)");
    return PHASTFT_OK;
}

template <typename T>
int32_t tables_import(Plan<T>* pl, const void* src, cudaStream_t s) {
    if (!pl || !src) return fail(PHASTFT_ERR_INVALID_ARG, "NULL argument");
    DeviceGuard g(pl->device);
    BlobHeader h;
    CUDA_TRY(cudaMemcpyAsync(&h, src, sizeof(h), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    int32_t st = check_blob_header(pl, h);
    if (st) return st;
    CUDA_TRY(cudaMemcpyAsync(pl->blob_dev, src, pl->blob_host.size(), cudaMemcpyDeviceToDevice, s));
    return PHASTFT_OK;
}

typedef int (*nccl_bcast_fn)(const void*, void*, size_t, int, int, void*, cudaStream_t);
// Two collectives, both joined by every rank whatever it finds (so a mismatching rank cannot leave the others hanging):
// the root's 256-byte header first, then the root's blob at the size the header states -- into the plan's tables when the
// layouts agree, into a throw-away buffer (and PHASTFT_ERR_PLAN_MISMATCH) when they do not.
template <typename T>
int32_t tables_broadcast(Plan<T>* pl, void* comm, int root, cudaStream_t s) {
    if (!pl || !comm) return fail(PHASTFT_ERR_INVALID_ARG, "NULL argument");
    static nccl_bcast_fn bcast = [] {
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        return h ? reinterpret_cast<nccl_bcast_fn>(dlsym(h, "ncclBroadcast")) : nullptr;
    }();
    if (!bcast) return fail(PHASTFT_ERR_NCCL, "libnccl.so.2 / ncclBroadcast not found");
    DeviceGuard g(pl->device);
    unsigned char* d_hdr = nullptr;
    CUDA_TRY(cudaMalloc(&d_hdr, BLOB_HEADER_BYTES));
    int rc = bcast(pl->blob_dev, d_hdr, BLOB_HEADER_BYTES, /*ncclChar*/ 0, root, comm, s);
    BlobHeader h;
    memset(&h, 0, sizeof(h));
    cudaError_t ce = rc == 0 ? cudaMemcpyAsync(&h, d_hdr, sizeof(h), cudaMemcpyDeviceToHost, s) : cudaSuccess;
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
    cudaFree(d_hdr);
    if (rc != 0) return fail(PHASTFT_ERR_NCCL, "ncclBroadcast (header) returned " + std::to_string(rc));
    if (ce != cudaSuccess) return fail(PHASTFT_ERR_CUDA, cudaGetErrorString(ce));
    const int32_t st = check_blob_header(pl, h);
    if (h.magic != BLOB_MAGIC || h.bytes == 0 || h.bytes > (uint64_t(1) << 34)) return st ? st : fail(PHASTFT_ERR_PLAN_MISMATCH, "bad header from root");
    unsigned char* target = pl->blob_dev;
    unsigned char* scratch = nullptr;
    if (st) {   // join the second collective anyway, at the root's size
        if (cudaMalloc(&scratch, h.bytes) != cudaSuccess) { (void)cudaGetLastError(); return st; }
        target = scratch;
    }
    rc = bcast(pl->blob_dev, target, h.bytes, /*ncclChar*/ 0, root, comm, s);
    if (scratch) { cudaStreamSynchronize(s); cudaFree(scratch); }
    if (st) { const std::string keep = g_last_error; (void)keep; return check_blob_header(pl, h); }
    if (rc != 0) return fail(PHASTFT_ERR_NCCL, "ncclBroadcast returned " + std::to_string(rc));
    return PHASTFT_OK;
}

// =================================================================================================
// r2c / c2r
// =================================================================================================
template <typename T>
struct PlanR2c {
    size_t n = 0;
    int device = 0;
    Plan<T>* inner = nullptr;          // half-length c2c (planner.rs:203)
    unsigned char* tw_dev = nullptr;   // two-level W_n table for the untangle / preprocess twiddles
    size_t hi_elems = 0, lo_elems = 0;
    int lo_bits = 0;
    double2 pre_wc[32];                // W_(2 R1)^i for the fused c2r first pass (R1 = first radix of inner->pass[0].kc)
    double2 pre_wc_b[32];              // ... and of a batched one (R1 = first radix of inner->pass[0].kcb)
    mutable std::mutex mu;
    mutable std::mutex host_mu;        // held for a whole *_host call (lock order: host_mu, then mu)
    mutable T* d_real = nullptr;       // host-API staging: N reals
    mutable T* d_spec_re = nullptr;    // N/2+1
    mutable T* d_spec_im = nullptr;
    mutable T* d_scr_re = nullptr;     // N/2 (c2r scratch when the caller passes none); grown under `mu` by batched sweeps
    mutable T* d_scr_im = nullptr;
    mutable size_t scr_elems = 0;      // per array
    mutable cudaEvent_t scr_free = nullptr;        // orders reuse of the plan-owned scratch across streams (like Plan::ws_free)
    mutable cudaStream_t scr_last_stream = nullptr;
    mutable bool scr_used = false;
    ~PlanR2c() {
        DeviceGuard g(device);
        if (scr_free) cudaEventDestroy(scr_free);
        for (void* p : {(void*)tw_dev, (void*)d_real, (void*)d_spec_re, (void*)d_spec_im, (void*)d_scr_re, (void*)d_scr_im})
            if (p) cudaFree(p);
        delete inner;
    }
};

template <typename T>
int32_t build_plan_r2c(size_t n, int device, PlanR2c<T>** out) {
    if (!out) return fail(PHASTFT_ERR_INVALID_ARG, "out == NULL");
    *out = nullptr;
    if (!(n >= 4 && is_pow2(n))) return fail(PHASTFT_ERR_R2C_N);   // planner.rs:195
    if (n > (size_t(1) << 31)) return fail(PHASTFT_ERR_INVALID_ARG, "n > 2^31 not supported");
    std::unique_ptr<PlanR2c<T>> pl(new PlanR2c<T>());
    pl->n = n; pl->device = device;
    int32_t st = build_plan<T>(n / 2, device, &pl->inner);
    if (st) return st;
    DeviceGuard g(device);
    const int ln = ilog2(n);
    pl->lo_bits = (ln + 1) / 2;
    pl->lo_elems = size_t(1) << pl->lo_bits;
    pl->hi_elems = size_t(1) << (ln - pl->lo_bits);
    std::vector<double2> tab(pl->hi_elems + pl->lo_elems);
    for (size_t h = 0; h < pl->hi_elems; ++h) root_of_unity((uint64_t)h << pl->lo_bits, n, tab[h].x, tab[h].y);
    for (size_t l = 0; l < pl->lo_elems; ++l) root_of_unity(l, n, tab[pl->hi_elems + l].x, tab[pl->hi_elems + l].y);
    CUDA_TRY(cudaMalloc(&pl->tw_dev, tab.size() * sizeof(double2)));
    CUDA_TRY(cudaMemcpy(pl->tw_dev, tab.data(), tab.size() * sizeof(double2), cudaMemcpyHostToDevice));
    memset(pl->pre_wc, 0, sizeof(pl->pre_wc));
    memset(pl->pre_wc_b, 0, sizeof(pl->pre_wc_b));
    if (pl->inner->num_passes >= 2 && pl->inner->pass[0].kc) {
        const uint64_t r1 = (uint64_t)pl->inner->pass[0].kc->first_radix;
        for (uint64_t i = 0; i < r1 && i < 32; ++i) root_of_unity(i, 2 * r1, pl->pre_wc[i].x, pl->pre_wc[i].y);
    }
    if (pl->inner->num_passes >= 2 && pl->inner->pass[0].kcb) {
        const uint64_t r1 = (uint64_t)pl->inner->pass[0].kcb->first_radix;
        for (uint64_t i = 0; i < r1 && i < 32; ++i) root_of_unity(i, 2 * r1, pl->pre_wc_b[i].x, pl->pre_wc_b[i].y);
    }
    // c2r scratch for the allocating variants lives in the plan (r2c.rs:716-718 allocates per call)
    CUDA_TRY(cudaMalloc(&pl->d_scr_re, (n / 2) * sizeof(T)));
    CUDA_TRY(cudaMalloc(&pl->d_scr_im, (n / 2) * sizeof(T)));
    pl->scr_elems = n / 2;
    CUDA_TRY(scribble_new(pl->inner->scribble_on, pl->d_scr_re, (n / 2) * sizeof(T)));
    CUDA_TRY(scribble_new(pl->inner->scribble_on, pl->d_scr_im, (n / 2) * sizeof(T)));
    CUDA_TRY(cudaEventCreateWithFlags(&pl->scr_free, cudaEventDisableTiming));
    *out = pl.release();
    return PHASTFT_OK;
}

template <typename T>
Tw2 r2c_tw2(const PlanR2c<T>* pl) {
    Tw2 t;
    t.hi = reinterpret_cast<const double2*>(pl->tw_dev);
    t.lo = t.hi + pl->hi_elems;
    t.lo_bits = pl->lo_bits;
    return t;
}

// The elementwise r2c untangle / c2r pre-processing of `members` batch members, `per` threads each: a member-major grid of
// 256-thread blocks, so a batch is not capped by gridDim.y; a batch of more than 2^31 - 1 blocks takes several launches.
// Launch record: R = N/2, C = the members of that launch.  `il`: the spectrum's bins are interleaved (the untangle's re, the
// pre-processing's in_re; im / in_im unused, strides in complex values): R2C-UNTANGLE-IL / C2R-PRE-IL.
template <typename T>
int32_t launch_real(bool untangle, const RealParams<T>& rp, size_t per, size_t members, cudaStream_t stream, bool il = false) {
    const size_t bpm = (per + 255) / 256;
    const size_t max_members = std::max<size_t>(1, grid_blocks_max() / bpm);
    const size_t out_w = il && untangle ? 2 : 1, in_w = il && !untangle ? 2 : 1;   // T per bin of the interleaved side
    for (size_t done = 0; done < members; done += max_members) {
        const size_t nb = std::min(members - done, max_members);
        RealParams<T> q = rp;
        q.re += out_w * done * rp.bstride;
        if (q.im) q.im += done * rp.bstride;
        if (q.in_re) {
            q.in_re += in_w * done * rp.in_bstride;
            if (q.in_im) q.in_im += done * rp.in_bstride;
        }
        q.blocks_per_member = (unsigned)bpm;
        const dim3 grid((unsigned)(nb * bpm));
        if (il) launch_real_il<T>(untangle, q, grid.x, stream);
        else if (untangle) r2c_untangle_kernel<T><<<grid, 256, 0, stream>>>(q);
        else c2r_preprocess_kernel<T><<<grid, 256, 0, stream>>>(q);
        CUDA_TRY(cudaGetLastError());
        note_launch({untangle ? (il ? "R2C-UNTANGLE-IL" : "R2C-UNTANGLE") : il ? "C2R-PRE-IL" : "C2R-PRE", 1 << rp.log2half, 0, (int)nb, 256, 0,
                     "plain", false});
    }
    return PHASTFT_OK;
}

template <typename T>
int32_t r2c_dev(const PlanR2c<T>* pl, const T* d_in, T* d_ore, T* d_oim, cudaStream_t stream) {
    if (!pl || !d_in || !d_ore || !d_oim) return fail(PHASTFT_ERR_INVALID_ARG, "NULL argument");
    if (int32_t st = check_pair_alignment(d_in, "d_input")) return st;     // read as (x[2k], x[2k+1]) pairs
    DeviceGuard g(pl->device);
    const size_t half = pl->n / 2;
    // (1)+(2) deinterleave fused into the first pass load: z[k] = x[2k] + i x[2k+1] (r2c.rs:557-569),
    //         half-length forward c2c into output[..half] (r2c.rs:575)
    Io<T> io;
    io.in_re = d_in; io.in_im = nullptr; io.in_il = 1; io.in_bstride = (long long)half;
    io.out_re = d_ore; io.out_im = d_oim; io.out_il = 0; io.out_bstride = (long long)half;
    int32_t st;
    if (pl->inner->num_passes == 0) return fail(PHASTFT_ERR_INVALID_ARG, "unreachable: half >= 2");
    st = run_c2c(*pl->inner, io, 1, T(1), stream);
    if (st) return st;
    // (3) untangle in place over all half+1 slots (r2c.rs:584-592)
    RealParams<T> rp;
    memset(&rp, 0, sizeof(rp));
    rp.re = d_ore; rp.im = d_oim; rp.log2half = ilog2(half); rp.tw2 = r2c_tw2(pl);
    return launch_real(true, rp, half / 2 + 1, 1, stream);
}

// The c2r build of the first pass a batched call of `batch` > 1 transforms runs on the inner plan, or NULL when that call
// takes a path without one (`why` says which).  The paths follow run_c2c: the one-CTA kernel, the cluster and pipelined
// launches and the TMA pair have no c2r build; otherwise every chunk's first pass needs one (kcb on a multi-wave chunk,
// kc on a chunk of one transform or below 2^21 points).
template <typename T>
const KernelEntry<T>* c2r_batch_first_pass(const Plan<T>& in, size_t batch, const char** why) {
    const bool many_call = (batch << in.log2n) >= (size_t(1) << 21);
    if (in.num_passes < 2) { *why = "one-CTA inner plan"; return nullptr; }
    if (in.alt_row.k && batch >= in.alt_row_min_batch) { *why = "batches of this size take the one-CTA kernel"; return nullptr; }
    if (in.cl && batch >= in.cl_min_batch) { *why = "batches of this size take the cluster launch"; return nullptr; }
    if (in.num_passes == 2 && many_call && in.pipe_b) { *why = "batches of this size take the pipelined launch"; return nullptr; }
    if (in.num_passes == 2 && in.pass[0].kt && in.pass[1].kt && many_call && in.tma_batch && in.ws_il != 0 &&
        (batch << in.log2n) * sizeof(T) >= (size_t(32) << 20)) {
        *why = "batches of this size take the TMA pair";
        return nullptr;
    }
    const size_t chunk = chunk_transforms(in, batch);
    const KernelEntry<T>* k = pass_takes_kb(in, in.pass[0], chunk) ? in.pass[0].kcb : in.pass[0].kc;
    if (!k) { *why = "the batched first pass tile has no c2r build"; return nullptr; }
    const size_t rest = batch % chunk;
    if (rest && !(pass_takes_kb(in, in.pass[0], rest) ? in.pass[0].kcb : in.pass[0].kc)) {
        *why = "the last chunk's first pass tile has no c2r build";
        return nullptr;
    }
    *why = "the batched first pass loads the half-spectra";
    return k;
}

// Whether c2r of `batch` transforms folds the pre-processing (r2c.rs:764-780) into the loads of the inverse transform's first
// pass under the current environment, and why (`why`: the rule that decided).  Fused: no scratch, one HBM round trip of N/2
// complex values less.  PHASTFT_C2R_FUSE=0 keeps the separate sweep.  c2r_dev, the batched call and both describe functions
// decide here, so they cannot disagree.
template <typename T>
bool c2r_fuses(const PlanR2c<T>* pl, size_t batch, const char** why) {
    const char* fuse_e = getenv("PHASTFT_C2R_FUSE");
    const Plan<T>& in = *pl->inner;
    const char* r = "the first pass loads the half-spectrum";
    bool fuse = false;
    if (batch > 1) {
        if (fuse_e && atoi(fuse_e) == 0) r = "PHASTFT_C2R_FUSE=0";
        else fuse = c2r_batch_first_pass(in, batch, &r) != nullptr;
        if (why) *why = r;
        return fuse;
    }
    if (fuse_e && atoi(fuse_e) == 0) r = "PHASTFT_C2R_FUSE=0";
    else if (in.num_passes < 2) r = "one-CTA inner plan";
    else if (!in.pass[0].kc) r = "the first pass tile has no c2r build";
    else if (in.cl && in.cl_min_batch <= 1) r = "lone transforms take the cluster launch";
    else if (in.pipe_1) r = "lone transforms take the pipelined launch";
    // Measured faster for f64 up to N = 2^20 and from 2^24 and for every f32 size; f64 2^21..2^23 (the sweep's scratch round
    // trip is cheap there, and the 1024-row tile of 2^21 keeps only 8 of its 32 loads per thread in flight) measured slightly
    // slower: those keep the separate sweep unless PHASTFT_C2R_FUSE=1 is set.
    else if (!(sizeof(T) == 4 || in.log2n < 20 || in.log2n > 22 || fuse_e != nullptr))
        r = "f64 inner 2^20..2^22 measured faster with the sweep (PHASTFT_C2R_FUSE=1 fuses)";
    else fuse = true;
    if (why) *why = r;
    return fuse;
}

// describe() (batch 1) and describe_batch(batch): the c2r path, the rule that decided and the c2r build of the first pass a call
// of `batch` transforms runs.
template <typename T>
std::string r2c_description(const PlanR2c<T>* pl, size_t batch) {
    const char* why = nullptr;
    const bool fuse = c2r_fuses(pl, batch, &why);
    const Plan<T>& in = *pl->inner;
    std::string s = "n=2^" + std::to_string(ilog2(pl->n)) + (sizeof(T) == 8 ? " f64" : " f32") + " r2c/c2r: c2r " +
                    (fuse ? "fused on load" : "separate sweep") + " (" + why + ") | c2r-in build: ";
    const char* unused = nullptr;
    const KernelEntry<T>* kc = batch > 1 ? c2r_batch_first_pass(in, batch, &unused) : in.num_passes >= 2 ? in.pass[0].kc : nullptr;
    if (kc)
        s += std::string(kind_name(kc->kind)) + " R=" + std::to_string(kc->R) + " C=" + std::to_string(kc->C) + " NT=" +
             std::to_string(kc->NT) + " R1=" + std::to_string(kc->first_radix);
    else
        s += "none";
    return s + " | inner: " + in.description;
}

template <typename T>
int32_t c2r_dev(const PlanR2c<T>* pl, const T* d_ire, const T* d_iim, T* d_out, T* d_sre, T* d_sim, cudaStream_t stream) {
    if (!pl || !d_ire || !d_iim || !d_out) return fail(PHASTFT_ERR_INVALID_ARG, "NULL argument");
    if ((d_sre == nullptr) != (d_sim == nullptr)) return fail(PHASTFT_ERR_INVALID_ARG, "pass both scratch arrays or neither");
    if (int32_t st = check_pair_alignment(d_out, "d_output")) return st;   // written as (y[2k], y[2k+1]) pairs, fused or not
    DeviceGuard g(pl->device);
    const size_t half = pl->n / 2;
    const Plan<T>& in = *pl->inner;
    if (c2r_fuses(pl, 1, nullptr)) {
        Io<T> io;
        io.in_re = d_ire; io.in_im = d_iim; io.in_il = 0; io.in_bstride = (long long)half;
        io.pre_tw2 = r2c_tw2(pl); io.pre_log2half = ilog2(half); io.pre_wc = pl->pre_wc;
        io.out_re = d_out; io.out_im = nullptr; io.out_il = 2; io.out_bstride = (long long)half;
        return run_c2c(in, io, 1, T(1) / (T)half, stream);
    }
    std::unique_lock<std::mutex> lock(pl->mu, std::defer_lock);
    bool own_scratch = false, capturing = false;
    if (!d_sre) {
        // The plan-owned scratch is used by kernels that run after this call returns: a caller on another stream
        // first waits for the previous user (the same protocol as the c2c workspace, run_c2c).
        lock.lock();
        d_sre = pl->d_scr_re; d_sim = pl->d_scr_im;
        own_scratch = true;
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        CUDA_TRY(cudaStreamIsCapturing(stream, &cap));
        capturing = cap != cudaStreamCaptureStatusNone;
        if (!capturing && pl->scr_used && pl->scr_last_stream != stream) CUDA_TRY(cudaStreamWaitEvent(stream, pl->scr_free, 0));
        CUDA_TRY(scribble(in.scribble_on, d_sre, half * sizeof(T), stream));
        CUDA_TRY(scribble(in.scribble_on, d_sim, half * sizeof(T), stream));
    }
    // (1) pre-process into scratch (r2c.rs:764-780)
    RealParams<T> rp;
    memset(&rp, 0, sizeof(rp));
    rp.re = d_sre; rp.im = d_sim; rp.in_re = d_ire; rp.in_im = d_iim; rp.log2half = ilog2(half); rp.tw2 = r2c_tw2(pl);
    if (int32_t st = launch_real(false, rp, half, 1, stream)) return st;
    // (2) inverse half-length c2c on the scratch (swap trick + 1/half, r2c.rs:782) with
    // (3) the re-interleave into the real output (r2c.rs:790-798) fused into the last store
    Io<T> io;
    io.in_re = d_sim; io.in_im = d_sre; io.in_il = 0; io.in_bstride = (long long)half;
    io.out_re = d_out; io.out_im = nullptr; io.out_il = 2; io.out_bstride = (long long)half;
    int32_t st = run_c2c(*pl->inner, io, 1, T(1) / (T)half, stream);
    if (st == PHASTFT_OK && own_scratch && !capturing) {
        CUDA_TRY(cudaEventRecord(pl->scr_free, stream));
        pl->scr_last_stream = stream;
        pl->scr_used = true;
    }
    return st;
}

// Grows the plan-owned c2r scratch to `elems` per array (batched sweeps).  Caller holds pl->mu.  The new arrays are allocated
// before the old ones are released, so a failed allocation leaves the plan as it was.
template <typename T>
int32_t grow_r2c_scratch(const PlanR2c<T>* pl, size_t elems) {
    if (pl->scr_elems >= elems) return PHASTFT_OK;
    T* re = nullptr;
    T* im = nullptr;
    if (cudaMalloc(&re, elems * sizeof(T)) != cudaSuccess || cudaMalloc(&im, elems * sizeof(T)) != cudaSuccess) {
        (void)cudaGetLastError();
        if (re) cudaFree(re);
        return fail(PHASTFT_ERR_CUDA, "cudaMalloc of the plan's c2r scratch for " + std::to_string(elems) + " elements failed");
    }
    CUDA_TRY(cudaDeviceSynchronize());   // every earlier user of the old scratch, on any stream, is done
    cudaFree(pl->d_scr_re);
    cudaFree(pl->d_scr_im);
    pl->d_scr_re = re; pl->d_scr_im = im; pl->scr_elems = elems;
    CUDA_TRY(scribble_new(pl->inner->scribble_on, re, elems * sizeof(T)));
    CUDA_TRY(scribble_new(pl->inner->scribble_on, im, elems * sizeof(T)));
    return PHASTFT_OK;
}

// Batched r2c: member b reads in_stride * b .. + N reals and writes N/2 + 1 bins at out_stride * b.  Batch 1 is r2c_dev.
template <typename T>
int32_t r2c_batch_dev(const PlanR2c<T>* pl, const T* d_in, size_t in_stride, T* d_ore, T* d_oim, size_t out_stride, size_t batch,
                      cudaStream_t stream) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (!d_in) return fail(PHASTFT_ERR_INVALID_ARG, "d_input == NULL");
    if (!d_ore) return fail(PHASTFT_ERR_INVALID_ARG, "d_out_re == NULL");
    if (!d_oim) return fail(PHASTFT_ERR_INVALID_ARG, "d_out_im == NULL");
    const size_t n = pl->n, half = n / 2;
    if (in_stride < n || in_stride % 2)
        return fail(PHASTFT_ERR_INVALID_ARG, "in_stride must be even and >= N = " + std::to_string(n) + " (got " + std::to_string(in_stride) + ")");
    if (out_stride < half + 1)
        return fail(PHASTFT_ERR_INVALID_ARG, "out_stride must be >= N/2 + 1 = " + std::to_string(half + 1) + " (got " + std::to_string(out_stride) + ")");
    if (int32_t st = check_pair_alignment(d_in, "d_input")) return st;
    if (batch == 0) return PHASTFT_OK;
    if (batch == 1) return r2c_dev(pl, d_in, d_ore, d_oim, stream);
    DeviceGuard g(pl->device);
    Io<T> io;
    io.in_re = d_in; io.in_im = nullptr; io.in_il = 1; io.in_bstride = (long long)(in_stride / 2);
    io.out_re = d_ore; io.out_im = d_oim; io.out_il = 0; io.out_bstride = (long long)out_stride;
    if (int32_t st = run_c2c(*pl->inner, io, batch, T(1), stream)) return st;
    RealParams<T> rp;
    memset(&rp, 0, sizeof(rp));
    rp.re = d_ore; rp.im = d_oim; rp.bstride = (long long)out_stride; rp.log2half = ilog2(half); rp.tw2 = r2c_tw2(pl);
    return launch_real(true, rp, half / 2 + 1, batch, stream);
}

// Batched c2r: member b reads N/2 + 1 bins at in_stride * b and writes N reals at out_stride * b.  Caller scratch holds
// batch * N/2 elements per array, dense.  Batch 1 is c2r_dev.
template <typename T>
int32_t c2r_batch_dev(const PlanR2c<T>* pl, const T* d_ire, const T* d_iim, size_t in_stride, T* d_out, size_t out_stride, T* d_sre,
                      T* d_sim, size_t batch, cudaStream_t stream) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (!d_ire) return fail(PHASTFT_ERR_INVALID_ARG, "d_in_re == NULL");
    if (!d_iim) return fail(PHASTFT_ERR_INVALID_ARG, "d_in_im == NULL");
    if (!d_out) return fail(PHASTFT_ERR_INVALID_ARG, "d_output == NULL");
    if ((d_sre == nullptr) != (d_sim == nullptr)) return fail(PHASTFT_ERR_INVALID_ARG, "pass both scratch arrays (d_scratch_re, d_scratch_im) or neither");
    const size_t n = pl->n, half = n / 2;
    if (in_stride < half + 1)
        return fail(PHASTFT_ERR_INVALID_ARG, "in_stride must be >= N/2 + 1 = " + std::to_string(half + 1) + " (got " + std::to_string(in_stride) + ")");
    if (out_stride < n || out_stride % 2)
        return fail(PHASTFT_ERR_INVALID_ARG, "out_stride must be even and >= N = " + std::to_string(n) + " (got " + std::to_string(out_stride) + ")");
    if (int32_t st = check_pair_alignment(d_out, "d_output")) return st;
    if (batch == 0) return PHASTFT_OK;
    if (batch == 1) return c2r_dev(pl, d_ire, d_iim, d_out, d_sre, d_sim, stream);
    DeviceGuard g(pl->device);
    Io<T> io;
    io.out_re = d_out; io.out_im = nullptr; io.out_il = 2; io.out_bstride = (long long)(out_stride / 2);
    if (c2r_fuses(pl, batch, nullptr)) {
        io.in_re = d_ire; io.in_im = d_iim; io.in_il = 0; io.in_bstride = (long long)in_stride;
        io.pre_tw2 = r2c_tw2(pl); io.pre_log2half = ilog2(half); io.pre_wc = pl->pre_wc; io.pre_wc_b = pl->pre_wc_b;
        return run_c2c(*pl->inner, io, batch, T(1) / (T)half, stream);
    }
    std::unique_lock<std::mutex> lock(pl->mu, std::defer_lock);
    bool own_scratch = false, capturing = false;
    if (!d_sre) {
        // the plan-owned scratch, grown to batch * N/2 (synchronising; an error while the stream is being captured)
        lock.lock();
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        CUDA_TRY(cudaStreamIsCapturing(stream, &cap));
        capturing = cap != cudaStreamCaptureStatusNone;
        if (pl->scr_elems < batch * half) {
            if (capturing)
                return fail(PHASTFT_ERR_INVALID_ARG, "the plan's c2r scratch is too small for this batch and the stream is being captured: "
                                                     "call phastft_plan_r2c_*_reserve(batch) before capturing");
            if (int32_t st = grow_r2c_scratch(pl, batch * half)) return st;
        }
        d_sre = pl->d_scr_re; d_sim = pl->d_scr_im;
        own_scratch = true;
        if (!capturing && pl->scr_used && pl->scr_last_stream != stream) CUDA_TRY(cudaStreamWaitEvent(stream, pl->scr_free, 0));
        CUDA_TRY(scribble(pl->inner->scribble_on, d_sre, batch * half * sizeof(T), stream));
        CUDA_TRY(scribble(pl->inner->scribble_on, d_sim, batch * half * sizeof(T), stream));
    }
    RealParams<T> rp;
    memset(&rp, 0, sizeof(rp));
    rp.re = d_sre; rp.im = d_sim; rp.bstride = (long long)half;
    rp.in_re = d_ire; rp.in_im = d_iim; rp.in_bstride = (long long)in_stride;
    rp.log2half = ilog2(half); rp.tw2 = r2c_tw2(pl);
    if (int32_t st = launch_real(false, rp, half, batch, stream)) return st;
    io.in_re = d_sim; io.in_im = d_sre; io.in_il = 0; io.in_bstride = (long long)half;
    int32_t st = run_c2c(*pl->inner, io, batch, T(1) / (T)half, stream);
    if (st == PHASTFT_OK && own_scratch && !capturing) {
        CUDA_TRY(cudaEventRecord(pl->scr_free, stream));
        pl->scr_last_stream = stream;
        pl->scr_used = true;
    }
    return st;
}

// Every allocation a batched call of `batch` would make: the inner plan's workspace, and the plan-owned c2r scratch when that
// batch's c2r takes the sweep.
template <typename T>
int32_t r2c_reserve(const PlanR2c<T>* pl, size_t batch) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (int32_t st = plan_reserve(pl->inner, batch)) return st;
    if (batch <= 1 || c2r_fuses(pl, batch, nullptr)) return PHASTFT_OK;
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> lock(pl->mu);
    return grow_r2c_scratch(pl, batch * (pl->n / 2));
}

// Interleaved spectra (phastft_{r2c,c2r}_interleaved_any_* on a power of two): member b's N/2 + 1 bins are Complex<T> values at
// complex element b * stride of d_spec.  The calls run the launches of r2c_batch_dev / c2r_batch_dev (c2r_dev for one member,
// with the plan's scratch) with the interleaved layout at the spectrum's end: the last pass stores Z as Complex<T>
// (out_interleaved = 1) and R2C-UNTANGLE-IL untangles it in place; c2r reads the bins in the MODE_C2R_IN_IL first pass or in
// C2R-PRE-IL.  Same arithmetic, so the planar call's results bit for bit.  The caller checked the arguments.
template <typename T>
int32_t r2c_il_dev(const PlanR2c<T>* pl, const T* d_in, size_t in_stride, T* d_spec, size_t spec_stride, size_t batch, cudaStream_t stream) {
    DeviceGuard g(pl->device);
    const size_t half = pl->n / 2;
    Io<T> io;
    io.in_re = d_in; io.in_im = nullptr; io.in_il = 1; io.in_bstride = (long long)(batch > 1 ? in_stride / 2 : half);
    io.out_re = d_spec; io.out_im = nullptr; io.out_il = 1; io.out_bstride = (long long)(batch > 1 ? spec_stride : half);
    if (int32_t st = run_c2c(*pl->inner, io, batch, T(1), stream)) return st;
    RealParams<T> rp;
    memset(&rp, 0, sizeof(rp));
    rp.re = d_spec; rp.im = nullptr; rp.bstride = (long long)(batch > 1 ? spec_stride : 0); rp.log2half = ilog2(half); rp.tw2 = r2c_tw2(pl);
    return launch_real(true, rp, half / 2 + 1, batch, stream, true);
}

template <typename T>
int32_t c2r_il_dev(const PlanR2c<T>* pl, const T* d_spec, size_t spec_stride, T* d_out, size_t out_stride, size_t batch, cudaStream_t stream) {
    DeviceGuard g(pl->device);
    const size_t half = pl->n / 2;
    Io<T> io;
    io.out_re = d_out; io.out_im = nullptr; io.out_il = 2; io.out_bstride = (long long)(batch > 1 ? out_stride / 2 : half);
    if (c2r_fuses(pl, batch, nullptr)) {
        io.in_re = d_spec; io.in_im = nullptr; io.in_il = 1; io.in_bstride = (long long)(batch > 1 ? spec_stride : half);
        io.pre_tw2 = r2c_tw2(pl); io.pre_log2half = ilog2(half); io.pre_wc = pl->pre_wc;
        if (batch > 1) io.pre_wc_b = pl->pre_wc_b;
        return run_c2c(*pl->inner, io, batch, T(1) / (T)half, stream);
    }
    // the separate sweep into the plan-owned scratch, under c2r_batch_dev's protocol (c2r_dev's for one member)
    std::lock_guard<std::mutex> lock(pl->mu);
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    CUDA_TRY(cudaStreamIsCapturing(stream, &cap));
    const bool capturing = cap != cudaStreamCaptureStatusNone;
    if (pl->scr_elems < batch * half) {
        if (capturing)
            return fail(PHASTFT_ERR_INVALID_ARG, "the plan's c2r scratch is too small for this batch and the stream is being captured: "
                                                 "call phastft_plan_r2c_any_*_reserve(batch) before capturing");
        if (int32_t st = grow_r2c_scratch(pl, batch * half)) return st;
    }
    T* sre = pl->d_scr_re;
    T* sim = pl->d_scr_im;
    if (!capturing && pl->scr_used && pl->scr_last_stream != stream) CUDA_TRY(cudaStreamWaitEvent(stream, pl->scr_free, 0));
    CUDA_TRY(scribble(pl->inner->scribble_on, sre, batch * half * sizeof(T), stream));
    CUDA_TRY(scribble(pl->inner->scribble_on, sim, batch * half * sizeof(T), stream));
    RealParams<T> rp;
    memset(&rp, 0, sizeof(rp));
    rp.re = sre; rp.im = sim; rp.bstride = (long long)(batch > 1 ? half : 0);
    rp.in_re = d_spec; rp.in_im = nullptr; rp.in_bstride = (long long)(batch > 1 ? spec_stride : 0);
    rp.log2half = ilog2(half); rp.tw2 = r2c_tw2(pl);
    if (int32_t st = launch_real(false, rp, half, batch, stream, true)) return st;
    io.in_re = sim; io.in_im = sre; io.in_il = 0; io.in_bstride = (long long)half;
    int32_t st = run_c2c(*pl->inner, io, batch, T(1) / (T)half, stream);
    if (st == PHASTFT_OK && !capturing) {
        CUDA_TRY(cudaEventRecord(pl->scr_free, stream));
        pl->scr_last_stream = stream;
        pl->scr_used = true;
    }
    return st;
}

template <typename T>
int32_t ensure_r2c_staging(const PlanR2c<T>* pl) {
    const size_t half = pl->n / 2;
    if (!pl->d_real) CUDA_TRY(cudaMalloc(&pl->d_real, pl->n * sizeof(T)));
    if (!pl->d_spec_re) CUDA_TRY(cudaMalloc(&pl->d_spec_re, (half + 1) * sizeof(T)));
    if (!pl->d_spec_im) CUDA_TRY(cudaMalloc(&pl->d_spec_im, (half + 1) * sizeof(T)));
    return PHASTFT_OK;
}

template <typename T>
int32_t r2c_host(const PlanR2c<T>* pl, const T* in, size_t len_in, T* ore, size_t len_ore, T* oim, size_t len_oim) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    const size_t n = pl->n, half = n / 2;
    if (len_in != n) return fail(PHASTFT_ERR_INPUT_LEN);              // r2c.rs:543
    if (len_ore != half + 1) return fail(PHASTFT_ERR_OUTPUT_RE_LEN);  // r2c.rs:544
    if (len_oim != half + 1) return fail(PHASTFT_ERR_OUTPUT_IM_LEN);  // r2c.rs:549
    if (!in || !ore || !oim) return fail(PHASTFT_ERR_INVALID_ARG, "NULL slice");
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> host_lock(pl->host_mu);     // same lock as c2r_host: both use the plan's staging buffers
    std::lock_guard<std::mutex> lock(pl->mu);
    int32_t st = ensure_r2c_staging(pl);
    if (st) return st;
    cudaStream_t s = pl->inner->stream;
    CUDA_TRY(scribble(pl->inner->scribble_on, pl->d_real, n * sizeof(T), s));
    CUDA_TRY(scribble(pl->inner->scribble_on, pl->d_spec_re, (half + 1) * sizeof(T), s));
    CUDA_TRY(scribble(pl->inner->scribble_on, pl->d_spec_im, (half + 1) * sizeof(T), s));
    CUDA_TRY(cudaMemcpyAsync(pl->d_real, in, n * sizeof(T), cudaMemcpyHostToDevice, s));
    st = r2c_dev(pl, pl->d_real, pl->d_spec_re, pl->d_spec_im, s);
    if (st) return st;
    CUDA_TRY(cudaMemcpyAsync(ore, pl->d_spec_re, (half + 1) * sizeof(T), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(oim, pl->d_spec_im, (half + 1) * sizeof(T), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return PHASTFT_OK;
}

template <typename T>
int32_t c2r_host(const PlanR2c<T>* pl, const T* ire, size_t len_ire, const T* iim, size_t len_iim, T* out, size_t len_out,
                 T* sre, size_t len_sre, T* sim, size_t len_sim) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    const size_t n = pl->n, half = n / 2;
    if (len_out != n) return fail(PHASTFT_ERR_OUTPUT_LEN);            // r2c.rs:750
    if (len_ire != half + 1) return fail(PHASTFT_ERR_INPUT_RE_LEN);   // r2c.rs:751
    if (len_iim != half + 1) return fail(PHASTFT_ERR_INPUT_IM_LEN);   // r2c.rs:756
    const bool has_scratch = sre || sim || len_sre || len_sim;
    if (has_scratch) {
        if (len_sre != half) return fail(PHASTFT_ERR_SCRATCH_RE_LEN);  // r2c.rs:761
        if (len_sim != half) return fail(PHASTFT_ERR_SCRATCH_IM_LEN);  // r2c.rs:762
    }
    if (!ire || !iim || !out) return fail(PHASTFT_ERR_INVALID_ARG, "NULL slice");
    DeviceGuard g(pl->device);
    cudaStream_t s = pl->inner->stream;
    std::lock_guard<std::mutex> host_lock(pl->host_mu);     // whole call: the staging buffers and the stream are per plan
    {
        std::lock_guard<std::mutex> lock(pl->mu);           // released before c2r_dev, which takes it for the plan-owned scratch
        int32_t st = ensure_r2c_staging(pl);
        if (st) return st;
    }
    CUDA_TRY(scribble(pl->inner->scribble_on, pl->d_real, n * sizeof(T), s));
    CUDA_TRY(scribble(pl->inner->scribble_on, pl->d_spec_re, (half + 1) * sizeof(T), s));
    CUDA_TRY(scribble(pl->inner->scribble_on, pl->d_spec_im, (half + 1) * sizeof(T), s));
    CUDA_TRY(cudaMemcpyAsync(pl->d_spec_re, ire, (half + 1) * sizeof(T), cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(pl->d_spec_im, iim, (half + 1) * sizeof(T), cudaMemcpyHostToDevice, s));
    int32_t st = c2r_dev<T>(pl, pl->d_spec_re, pl->d_spec_im, pl->d_real, nullptr, nullptr, s);
    if (st) return st;
    CUDA_TRY(cudaMemcpyAsync(out, pl->d_real, n * sizeof(T), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return PHASTFT_OK;
}

template <typename T> OneShotCache<PlanR2c<T>>& oneshot_r2c_cache() { static auto* c = new OneShotCache<PlanR2c<T>>(); return *c; }
// caller holds c.mu
template <typename T>
int32_t oneshot_r2c_plan(OneShotCache<PlanR2c<T>>& c, size_t n, int device, PlanR2c<T>** out) {
    if (!c.plan || c.n != n || c.device != device) {
        delete c.plan;
        c.plan = nullptr; c.n = 0; c.device = -1;
        int32_t st = build_plan_r2c<T>(n, device, &c.plan);
        if (st) return st;
        c.n = n; c.device = device;
    }
    *out = c.plan;
    return PHASTFT_OK;
}

// =================================================================================================
// any length: Bluestein's chirp-z algorithm over the power-of-two plans (the CHIRP-* kernels, fft_kernels.cuh)
// =================================================================================================
// The largest length that is not a power of two: its convolution length M = 2^ceil(log2(2N - 1)) is 2^30, the largest
// power-of-two plan.
constexpr size_t ANY_MAX_N = (size_t(1) << 29) - 1;

// The interleaved workspace of an any-length plan (Bluestein's batch x M, the mixed-radix path's batch x N) and its protocol,
// the one of run_c2c: grown (synchronising) outside a stream capture only; a caller on another stream first waits for the
// previous user.  `mu` also guards the owner's host staging.
template <typename T>
struct AnyWorkspace {
    std::mutex mu;
    cx<T>* ws = nullptr;
    size_t elems = 0;
    cudaEvent_t free_ev = nullptr;     // orders workspace reuse across streams (like Plan::ws_free)
    cudaStream_t last_stream = nullptr;
    bool used = false;
    bool scribble_on = false;          // PHASTFT_SCRIBBLE=1, read when the plan is built: also covers the owner's host staging
    int32_t init(size_t e) {
        scribble_on = scribble_env();
        CUDA_TRY(cudaMalloc(&ws, e * sizeof(cx<T>)));
        elems = e;
        CUDA_TRY(scribble_new(scribble_on, ws, e * sizeof(cx<T>)));
        CUDA_TRY(cudaEventCreateWithFlags(&free_ev, cudaEventDisableTiming));
        return PHASTFT_OK;
    }
    void destroy() {
        if (free_ev) cudaEventDestroy(free_ev);
        if (ws) cudaFree(ws);
    }
    // Grows to `e` values (`members` batch members).  Caller holds mu.  The new array is allocated before the old one is
    // released, so a failed allocation leaves the plan as it was.
    int32_t grow(size_t e, size_t members) {
        if (elems >= e) return PHASTFT_OK;
        cx<T>* w = nullptr;
        if (cudaMalloc(&w, e * sizeof(cx<T>)) != cudaSuccess) {
            (void)cudaGetLastError();
            return fail(PHASTFT_ERR_CUDA, "cudaMalloc of the plan's workspace for " + std::to_string(members) + " members failed");
        }
        CUDA_TRY(cudaDeviceSynchronize());   // every earlier user of the old workspace, on any stream, is done
        cudaFree(ws);
        ws = w; elems = e;
        CUDA_TRY(scribble_new(scribble_on, ws, e * sizeof(cx<T>)));
        return PHASTFT_OK;
    }
    // Before a call's first launch (caller holds mu): room for `e` values, and the previous user on another stream is done.
    // `reserve_fn` names the call that grows the workspace ahead of a capture.
    int32_t acquire(size_t e, size_t members, cudaStream_t stream, const char* reserve_fn, bool& capturing) {
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        CUDA_TRY(cudaStreamIsCapturing(stream, &cap));
        capturing = cap != cudaStreamCaptureStatusNone;
        if (elems < e) {
            if (capturing)
                return fail(PHASTFT_ERR_INVALID_ARG, std::string("the plan's workspace is too small for this batch and the stream is being "
                                                                 "captured: call ") + reserve_fn + "(batch) before capturing");
            if (int32_t st = grow(e, members)) return st;
        }
        if (!capturing && used && last_stream != stream) CUDA_TRY(cudaStreamWaitEvent(stream, free_ev, 0));
        CUDA_TRY(scribble(scribble_on, ws, e * sizeof(cx<T>), stream));
        return PHASTFT_OK;
    }
    // After a call's last launch.
    int32_t release(cudaStream_t stream, bool capturing) {
        if (!capturing) {
            CUDA_TRY(cudaEventRecord(free_ev, stream));
            last_stream = stream;
            used = true;
        }
        return PHASTFT_OK;
    }
};

// The Bluestein state of one length L: the chirp w[j] = exp(-pi i (j^2 mod 2L) / L), the transform of the convolution kernel,
// the M-point plan of both convolution transforms and the workspace, M = 2^ceil(log2(2L - 1)) but at least 4 (Cx16<float>
// moves two complex values per thread: M = 1 would launch no thread and write past a one-value workspace).  The complex plan
// runs it on N, the real plan on N or N/2.
template <typename T>
struct Bluestein {
    size_t l = 0;
    int log2m = 0;                     // 0: not built
    int device = 0;
    Plan<T>* inner = nullptr;          // the M-point plan
    cx<T>* chirp = nullptr;            // w[0 .. L), zero-padded to a multiple of Cx16<T>::V
    cx<T>* bhat = nullptr;             // FFT_M(b) / M, computed in f64
    mutable AnyWorkspace<T> w;         // members x M interleaved complex
    ~Bluestein() {
        if (!inner) return;
        DeviceGuard g(device);
        w.destroy();
        for (void* p : {(void*)chirp, (void*)bhat})
            if (p) cudaFree(p);
        delete inner;
    }
};

// =================================================================================================
// any length, smooth N = 2^a 3^b 5^c 7^d: the mixed-radix path (SMOOTH-PRE and the ODD kernels, fft_kernels.cuh)
// =================================================================================================
// Lengths on the mixed path stay below 2^30 (a workspace of N values, the exponent of W_N formed in 64 bits).
constexpr size_t MIXED_MAX_N = (size_t(1) << 30) - 1;

// N = P * Q_a * Q_b: P the power-of-two part, the odd part in one pass (Q_b = 1) or two, each of at most ODD_MAX_ROWS rows.
struct MixedSplit {
    size_t p = 0;
    int qa = 0, qb = 1;
};

// The split of n, or why it has none (`why` names the offending factor, and the length as `name`).
bool mixed_split(size_t n, MixedSplit& out, std::string& why, const char* name = "n") {
    const std::string nm = std::string(name) + " = " + std::to_string(n);
    if (n < 3 || is_pow2(n)) { why = nm + " has no odd factor (powers of two take the c2c plan)"; return false; }
    if (n > MIXED_MAX_N) { why = nm + " is above 2^30 - 1"; return false; }
    size_t p = 1, q = n;
    while (q % 2 == 0) { q /= 2; p *= 2; }
    size_t rest = q;
    for (size_t f : {3, 5, 7})
        while (rest % f == 0) rest /= f;
    if (rest > 1) {
        size_t f = 11;
        while (f * f <= rest && rest % f) f += 2;
        if (rest % f) f = rest;
        why = nm + " has the prime factor " + std::to_string(f) + " (the mixed-radix path takes 2, 3, 5 and 7)";
        return false;
    }
    out.p = p;
    if (q <= (size_t)ODD_MAX_ROWS) { out.qa = (int)q; out.qb = 1; return true; }
    size_t best = 0;                                   // the largest divisor a <= sqrt(q): the most balanced split
    for (size_t a = 3; a * a <= q; a += 2)
        if (q % a == 0 && q / a <= (size_t)ODD_MAX_ROWS) best = a;
    if (!best) {
        why = nm + ": its odd part " + std::to_string(q) + " is not a product of two factors of at most " +
              std::to_string(ODD_MAX_ROWS);
        return false;
    }
    out.qa = (int)best; out.qb = (int)(q / best);
    return true;
}

// "mixed 2^a x Q_a[ x Q_b]"
std::string mixed_description(const MixedSplit& s) {
    return "mixed 2^" + std::to_string(ilog2(s.p)) + " x " + std::to_string(s.qa) + (s.qb > 1 ? " x " + std::to_string(s.qb) : "");
}

// One ODD pass of R rows: the register kernel for one or two radices up to 35 rows (49 rows of f64 would spill), else the
// shared-memory tile.
template <typename T>
struct OddPass {
    int r = 0, nstages = 0, rad[ODD_MAX_STAGES] = {};
    int cw = 0;                        // tile kernel: columns per CTA; 0: the register kernel
    const cx<T>* wr = nullptr;         // W_R^j (in the plan's table blob)
    const unsigned short* perm = nullptr;
};

template <typename T>
struct Mixed {
    size_t n = 0;
    MixedSplit split;
    int device = 0;
    Plan<T>* inner = nullptr;          // the P-point plan (it also owns the host calls' stream); nullptr: not built
    char* tables = nullptr;            // W_N two-level, then per pass W_R and the digit reversal
    const cx<T>* wn_hi = nullptr;
    const cx<T>* wn_lo = nullptr;
    int lo_bits = 0;
    int npasses = 0;
    OddPass<T> pass[2];
    mutable AnyWorkspace<T> w;         // batch x N interleaved complex
    ~Mixed() {
        if (!inner) return;
        DeviceGuard g(device);
        w.destroy();
        if (tables) cudaFree(tables);
        delete inner;
    }
};

// radices of an R-row pass, largest first
inline int odd_stages(int r, int* rad) {
    int s = 0;
    for (int f : {7, 5, 3})
        while (r % f == 0) { r /= f; rad[s++] = f; }
    return s;
}

template <typename T>
int32_t build_mixed(Mixed<T>& mx, size_t n, const MixedSplit& split, int device) {
    mx.n = n; mx.split = split; mx.device = device;
    if (int32_t st = build_plan<T>(split.p, device, &mx.inner)) return st;
    DeviceGuard g(device);
    int ln = 0;
    while ((size_t(1) << ln) < n) ++ln;
    mx.lo_bits = (ln + 1) / 2;
    const size_t n_lo = size_t(1) << mx.lo_bits, n_hi = ((n - 1) >> mx.lo_bits) + 1;
    mx.npasses = split.qb > 1 ? 2 : 1;
    // one blob: every table starts on a 16-byte boundary
    auto pad = [](size_t b) { return (b + 15) / 16 * 16; };
    std::vector<char> host;
    auto append = [&](const void* src, size_t bytes) {
        const size_t off = host.size();
        host.resize(off + pad(bytes));
        memcpy(host.data() + off, src, bytes);
        return off;
    };
    auto roots = [&](size_t count, size_t mul, size_t of) {
        std::vector<cx<T>> v(count);
        for (size_t j = 0; j < count; ++j) {
            double re, im;
            root_of_unity_any(j * mul, of, re, im);
            v[j].x = (T)re; v[j].y = (T)im;
        }
        return append(v.data(), count * sizeof(cx<T>));
    };
    const size_t off_lo = roots(n_lo, 1, n), off_hi = roots(n_hi, n_lo, n);
    size_t off_wr[2] = {0, 0}, off_perm[2] = {0, 0};
    for (int i = 0; i < mx.npasses; ++i) {
        OddPass<T>& ps = mx.pass[i];
        ps.r = i == 0 ? split.qa : split.qb;
        ps.nstages = odd_stages(ps.r, ps.rad);
        off_wr[i] = roots((size_t)ps.r, 1, (size_t)ps.r);
        if (ps.nstages > 2 || ps.r == 49) {
            // as many columns as keep the tile under 48 KiB, at least a 128-byte row run
            const int cmin = 128 / (int)sizeof(cx<T>);
            ps.cw = ODD_NT;
            while (ps.cw > cmin && (size_t)ps.r * ps.cw * sizeof(cx<T>) > (size_t(48) << 10)) ps.cw /= 2;
            // stage 1's butterfly of rows b + q R / rad[0] goes to rows perm[b] rad[0] + q: b's digits, last radix first, reversed
            std::vector<unsigned short> perm(ps.r / ps.rad[0]);
            for (size_t b = 0; b < perm.size(); ++b) {
                size_t m = b, pos = 0, weight = perm.size();
                for (int s = ps.nstages - 1; s >= 1; --s) {
                    weight /= ps.rad[s];
                    pos += m % ps.rad[s] * weight;
                    m /= ps.rad[s];
                }
                perm[b] = (unsigned short)pos;
            }
            off_perm[i] = append(perm.data(), perm.size() * sizeof(unsigned short));
        }
    }
    CUDA_TRY(cudaMalloc(&mx.tables, host.size()));
    CUDA_TRY(cudaMemcpy(mx.tables, host.data(), host.size(), cudaMemcpyHostToDevice));
    mx.wn_lo = reinterpret_cast<const cx<T>*>(mx.tables + off_lo);
    mx.wn_hi = reinterpret_cast<const cx<T>*>(mx.tables + off_hi);
    for (int i = 0; i < mx.npasses; ++i) {
        mx.pass[i].wr = reinterpret_cast<const cx<T>*>(mx.tables + off_wr[i]);
        if (mx.pass[i].cw) mx.pass[i].perm = reinterpret_cast<const unsigned short*>(mx.tables + off_perm[i]);
    }
    CUDA_TRY(cudaFuncSetAttribute(odd_tile_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  ODD_MAX_ROWS * 128));
    CUDA_TRY(mixed_real_init<T>());
    CUDA_TRY(any_il_init<T>());
    CUDA_TRY(real_il_init<T>());
    return mx.w.init(n);                               // room for one member; batched calls grow it
}

// One ODD pass over `batch` members, MODE the last pass's store (C2C for pass A).  Launch record: R = rows, C = the columns a
// CTA covers; the kind carries -C2R / -R2C for the real stores, -IL for the interleaved ones (ODD-R2C-IL: the direct r2c's
// interleaved bins).
template <int MODE, typename T>
int32_t launch_odd(const Mixed<T>& mx, int i, OddParams<T> q, size_t batch, cudaStream_t stream) {
    const OddPass<T>& ps = mx.pass[i];
    const size_t P = mx.split.p;
    const bool last = i == mx.npasses - 1;
    q.role = mx.npasses == 1 ? ODD_SINGLE : i == 0 ? ODD_A : ODD_B;
    q.r = ps.r; q.qb = mx.split.qb; q.wr = ps.wr; q.perm = ps.perm; q.cw = ps.cw;
    q.nstages = ps.nstages;
    for (int s = 0; s < ps.nstages; ++s) q.rad[s] = ps.rad[s];
    q.cols = (long long)(mx.n / ps.r);
    q.total = (long long)batch * q.cols;
    q.in_rs = (long long)(q.role == ODD_A ? mx.split.qb * P : P);
    q.out_rs = (long long)(q.role == ODD_A ? mx.split.qb * P : q.role == ODD_B ? mx.split.qa * P : P);
    if (!last) q.scale = T(1);
    const int cover = ps.cw ? ps.cw : ODD_NT;
    const size_t blocks = ((size_t)q.total + cover - 1) / cover;
    if (blocks > 0x7fffffffu) return fail(PHASTFT_ERR_INVALID_ARG, "batch * N is too large for one launch of the odd pass");
    const size_t smem = ps.cw ? (size_t)ps.r * ps.cw * sizeof(cx<T>) : 0;
    const bool ok = MODE == CHIRP_C2C ? launch_odd_kernel<T, CHIRP_C2C>(q, ps.r, smem, (unsigned)blocks, stream)
                    : chirp_il<MODE>() ? launch_odd_il<T>(MODE, q, ps.r, smem, (unsigned)blocks, stream)
                    : MODE == CHIRP_R2C_DIRECT_IL ? launch_odd_r2c_il<T>(q, ps.r, smem, (unsigned)blocks, stream)
                                       : launch_odd_real<T>(MODE, q, ps.r, smem, (unsigned)blocks, stream);
    if (!ok) return fail(PHASTFT_ERR_INVALID_ARG, "no register kernel of " + std::to_string(ps.r) + " rows");
    CUDA_TRY(cudaGetLastError());
    const char* name = MODE == CHIRP_C2R_HALVED || MODE == CHIRP_C2R_DIRECT ? "ODD-C2R" : MODE == CHIRP_R2C_DIRECT ? "ODD-R2C"
                       : MODE == CHIRP_R2C_DIRECT_IL                        ? "ODD-R2C-IL"
                       : chirp_il<MODE>()                                   ? "ODD-IL"
                                                                            : "ODD";
    note_launch({name, ps.r, 0, cover, ODD_NT, 0, ps.cw ? "tile" : "reg", false});
    return PHASTFT_OK;
}

// W_N^e for e < count from two tables of about sqrt(count) roots each: W_N^e = hi[e >> lo_bits] lo[e & (2^lo_bits - 1)]
// (the real mixed plans' W_N, N = 2L, for the c2r pre-processing and the untangle)
template <typename T>
struct TwoLevelRoots {
    cx<T>* blob = nullptr;             // lo, then hi
    const cx<T>* hi = nullptr;
    const cx<T>* lo = nullptr;
    int lo_bits = 0;
};

template <typename T>
int32_t build_two_level(TwoLevelRoots<T>& t, size_t n, size_t count) {
    int lc = 0;
    while ((size_t(1) << lc) < count) ++lc;
    t.lo_bits = (lc + 1) / 2;
    const size_t n_lo = size_t(1) << t.lo_bits, n_hi = ((count - 1) >> t.lo_bits) + 1;
    std::vector<cx<T>> v(n_lo + n_hi);
    for (size_t j = 0; j < n_lo + n_hi; ++j) {
        double re, im;
        root_of_unity_any(j < n_lo ? j : (j - n_lo) << t.lo_bits, n, re, im);
        v[j].x = (T)re; v[j].y = (T)im;
    }
    CUDA_TRY(cudaMalloc(&t.blob, v.size() * sizeof(cx<T>)));
    CUDA_TRY(cudaMemcpy(t.blob, v.data(), v.size() * sizeof(cx<T>), cudaMemcpyHostToDevice));
    t.lo = t.blob; t.hi = t.blob + n_lo;
    return PHASTFT_OK;
}

// One mixed-radix call of `batch` members: SMOOTH-PRE, the P-point plan on Q * batch workspace members, the ODD pass(es), with
// the ends in MODE (CHIRP_C2C for the complex plan, C2C_IL / C2C_IL_SWAP for its interleaved calls; the real modes as in
// CHIRP-PRE / CHIRP-POST, fft_kernels.cuh).  in / out are the caller's arrays, swapped for the reverse direction (the
// interleaved modes: in_re and out_re, swapped by the mode); in_bstride counts T, out_bstride what the last pass stores (T, or
// complex values for C2R_HALVED and the interleaved modes); scale is 1, 1/N or 1/L.  `wn` is the real plan's W_(2L) for the
// halved modes.  The halved r2c ends with SMOOTH-POST-R2C on the bins.  The workspace follows AnyWorkspace's protocol (`reserve_fn` names the call that grows it).
// The real modes with an interleaved spectrum (CHIRP_*_IL, spectrum strides in complex values) run their mode at the spectrum's
// end only: r2c loads with the planar SMOOTH-PRE-R2C and stores ODD-IL + SMOOTH-POST-R2C-IL (halved) or ODD-R2C-IL (direct);
// c2r loads with SMOOTH-PRE-C2R-IL and stores with the planar ODD-C2R.
template <int MODE, typename T>
int32_t mixed_run(const Mixed<T>& mx, const T* in_re, const T* in_im, size_t in_bstride, T* out_re, T* out_im, size_t out_bstride,
                  T scale, size_t batch, cudaStream_t stream, const char* reserve_fn, const TwoLevelRoots<T>* wn = nullptr) {
    constexpr int PM = chirp_planar<MODE>();
    constexpr bool sil = chirp_spec_il<MODE>();
    constexpr bool r2c = PM == CHIRP_R2C_HALVED || PM == CHIRP_R2C_DIRECT, c2r = PM == CHIRP_C2R_HALVED || PM == CHIRP_C2R_DIRECT;
    constexpr bool il = chirp_il<MODE>();
    constexpr int PRE = r2c ? PM : MODE;                                // SMOOTH-PRE's mode
    // the halved r2c stores Z, then untangles it in place
    constexpr int LAST = MODE == CHIRP_R2C_HALVED ? CHIRP_C2C : MODE == CHIRP_R2C_HALVED_IL ? CHIRP_C2C_IL : c2r ? PM : MODE;
    DeviceGuard g(mx.device);
    const size_t P = mx.split.p, Q = (size_t)mx.split.qa * mx.split.qb;
    std::lock_guard<std::mutex> lock(mx.w.mu);
    bool capturing = false;
    if (int32_t st = mx.w.acquire(batch * mx.n, batch, stream, reserve_fn, capturing)) return st;
    SmoothParams<T> sp;
    memset(&sp, 0, sizeof(sp));
    sp.in_re = in_re; sp.in_im = in_im; sp.ws = mx.w.ws;
    sp.n = (long long)mx.n; sp.p = (long long)P; sp.q = (long long)Q; sp.bstride = (long long)in_bstride;
    if (wn) { sp.wn_hi = wn->hi; sp.wn_lo = wn->lo; sp.lo_bits = wn->lo_bits; }
    // runs as long as Q and P allow within SMOOTH_TILE values: up to 32 values of n_o, then n_2, then the rest of n_o when P is short
    size_t tq = std::min<size_t>(Q, 32), tq2 = 1;
    while (tq2 < tq) tq2 *= 2;
    const size_t tp = std::min<size_t>(P, SMOOTH_TILE / tq2);
    if (tp < 32) tq = std::min<size_t>(Q, SMOOTH_TILE / tp);
    sp.tq = (int)tq; sp.tp = (int)tp;
    sp.tiles_q = (unsigned)((Q + tq - 1) / tq);
    sp.tiles_per_member = sp.tiles_q * (unsigned)(P / tp);
    const size_t max_members = std::max<size_t>(1, grid_blocks_max() / sp.tiles_per_member);
    for (size_t done = 0; done < batch; done += max_members) {
        const size_t nb = std::min(batch - done, max_members);
        SmoothParams<T> s2 = sp;
        s2.in_re += done * in_bstride; s2.ws += done * mx.n;
        if (s2.in_im) s2.in_im += done * in_bstride;
        if constexpr (MODE == CHIRP_C2C) smooth_pre_kernel<T><<<(unsigned)(nb * sp.tiles_per_member), 256, 0, stream>>>(s2);
        else if constexpr (il) launch_smooth_pre_il<T>(MODE, s2, (unsigned)(nb * sp.tiles_per_member), stream);
        else if constexpr (chirp_spec_il<PRE>()) launch_smooth_pre_real_il<T>(PRE, s2, (unsigned)(nb * sp.tiles_per_member), stream);
        else launch_smooth_pre_real<T>(PRE, s2, (unsigned)(nb * sp.tiles_per_member), stream);
        CUDA_TRY(cudaGetLastError());
        note_launch({r2c ? "SMOOTH-PRE-R2C" : c2r ? (sil ? "SMOOTH-PRE-C2R-IL" : "SMOOTH-PRE-C2R") : il ? "SMOOTH-PRE-IL" : "SMOOTH-PRE",
                     (int)P, 0, (int)(nb * Q), 256, 0, "plain", false});
    }
    if (P > 1) {
        Io<T> io;
        io.in_re = reinterpret_cast<const T*>(mx.w.ws); io.in_im = nullptr;
        io.out_re = reinterpret_cast<T*>(mx.w.ws); io.out_im = nullptr;
        io.in_bstride = io.out_bstride = (long long)P;
        io.in_il = io.out_il = 1;
        if (int32_t st = run_c2c(*mx.inner, io, Q * batch, T(1), stream)) return st;
    }
    OddParams<T> q;
    memset(&q, 0, sizeof(q));
    q.ws = mx.w.ws; q.ws_out = mx.w.ws; q.out_re = out_re; q.out_im = out_im;
    q.wn_hi = mx.wn_hi; q.wn_lo = mx.wn_lo; q.lo_bits = mx.lo_bits;
    q.n = (long long)mx.n; q.p = (long long)P; q.bstride = (long long)out_bstride; q.scale = scale;
    for (int i = 0; i < mx.npasses; ++i)
        if (int32_t st = i + 1 < mx.npasses ? launch_odd<CHIRP_C2C>(mx, i, q, batch, stream) : launch_odd<LAST>(mx, i, q, batch, stream))
            return st;
    if constexpr (PM == CHIRP_R2C_HALVED) {
        // Launch record: R = L, C = the members of that launch
        SmoothPostParams<T> pp;
        pp.re = out_re; pp.im = out_im; pp.wn_hi = wn->hi; pp.wn_lo = wn->lo; pp.lo_bits = wn->lo_bits;
        pp.l = (long long)mx.n; pp.bstride = (long long)out_bstride;
        const size_t bpm = (mx.n / 2 + 1 + 255) / 256;
        pp.blocks_per_member = (unsigned)bpm;
        const size_t max_members = std::max<size_t>(1, grid_blocks_max() / bpm);
        for (size_t done = 0; done < batch; done += max_members) {
            const size_t nb = std::min(batch - done, max_members);
            SmoothPostParams<T> p2 = pp;
            p2.re += (sil ? 2 : 1) * done * out_bstride;
            if (p2.im) p2.im += done * out_bstride;
            if constexpr (sil) launch_smooth_post_r2c_il<T>(p2, (unsigned)(nb * bpm), stream);
            else launch_smooth_post_r2c<T>(p2, (unsigned)(nb * bpm), stream);
            CUDA_TRY(cudaGetLastError());
            note_launch({sil ? "SMOOTH-POST-R2C-IL" : "SMOOTH-POST-R2C", (int)mx.n, 0, (int)nb, 256, 0, "plain", false});
        }
    }
    return mx.w.release(stream, capturing);
}

// Every allocation a call of `batch` would make: the inner plan's workspace for Q * batch members and batch * N values here.
template <typename T>
int32_t mixed_reserve(const Mixed<T>& mx, size_t batch) {
    if (mx.split.p > 1)
        if (int32_t st = plan_reserve(mx.inner, (size_t)mx.split.qa * mx.split.qb * batch)) return st;
    DeviceGuard g(mx.device);
    std::lock_guard<std::mutex> lock(mx.w.mu);
    return mx.w.grow(batch * mx.n, batch);
}

template <typename T>
struct PlanAny {
    size_t n = 0;
    int device = 0;
    Plan<T>* pow2 = nullptr;           // N a power of two: the N-point plan, run as it is
    Bluestein<T> bs;                   // otherwise: Bluestein of L = N ...
    Mixed<T> mx;                       // ... or the mixed-radix path (mx.inner set)
    AnyWorkspace<T>& workspace() const { return mx.inner ? mx.w : bs.w; }
    cudaStream_t host_stream() const { return (mx.inner ? mx.inner : bs.inner)->stream; }
    mutable std::mutex host_mu;        // held for a whole *_host call (lock order: host_mu, then the workspace's mu)
    mutable T* stage_re = nullptr;     // host-API staging: N each
    mutable T* stage_im = nullptr;
    mutable T* stage_il = nullptr;     // the interleaved host calls' staging: N complex, allocated by the first such call
    std::string description;
    ~PlanAny() {
        DeviceGuard g(device);
        for (void* p : {(void*)stage_re, (void*)stage_im, (void*)stage_il})
            if (p) cudaFree(p);
        delete pow2;
    }
};

// f(i) for i in [0, count), spread over the host's cores for large counts (long-double tables of 2^29 entries take minutes
// on one)
template <typename F>
void host_parallel(size_t count, F f) {
    auto work = [&](size_t t, size_t step) {
        for (size_t i = t; i < count; i += step) f(i);
    };
    const size_t nt = std::min<size_t>(std::max(1u, std::thread::hardware_concurrency()), 64);
    if (count < 8192 || nt == 1) { work(0, 1); return; }
    std::vector<std::thread> th;
    for (size_t t = 0; t < nt; ++t) th.emplace_back(work, t, nt);
    for (std::thread& x : th) x.join();
}

// w[j] = exp(-pi i (j^2 mod 2N) / N) for j in [s, s + count): the phase is reduced exactly in integers (j^2 < 2^58 for
// j < 2^29) and evaluated in long double with octant symmetry.
void chirp_table(size_t n, size_t s, size_t count, double2* w) {
    host_parallel(count, [=](size_t i) {
        const uint64_t j = s + i;
        root_of_unity_any(j * j % (2 * n), 2 * n, w[i].x, w[i].y);
    });
}

template <typename T>
int32_t build_bluestein(Bluestein<T>& bs, size_t l, int device) {
    int lm = 2;
    while ((size_t(1) << lm) < 2 * l - 1) ++lm;
    const size_t M = size_t(1) << lm;
    bs.l = l; bs.device = device;
    if (int32_t st = build_plan<T>(M, device, &bs.inner)) return st;
    bs.log2m = lm;
    DeviceGuard g(device);
    // w in T for the kernels, and b[m] = conj(w[|m|]) on the circle of M points in f64 (0 where |m| >= L), built chunk by chunk
    constexpr size_t V = Cx16<T>::V;
    const size_t nc = (l + V - 1) / V * V;
    CUDA_TRY(cudaMalloc(&bs.chirp, nc * sizeof(cx<T>)));
    CUDA_TRY(cudaMemset(bs.chirp, 0, nc * sizeof(cx<T>)));
    double2* b = nullptr;
    CUDA_TRY(cudaMalloc(&b, M * sizeof(double2)));
    std::unique_ptr<double2, void (*)(double2*)> b_owner(b, [](double2* p) { cudaFree(p); });
    CUDA_TRY(cudaMemset(b, 0, M * sizeof(double2)));
    const size_t CH = size_t(1) << 20;
    std::vector<double2> w(std::min(CH, l)), rev(std::min(CH, l));
    std::vector<cx<T>> wt(std::min(CH, l));
    for (size_t s = 0; s < l; s += CH) {
        const size_t cnt = std::min(CH, l - s);
        chirp_table(l, s, cnt, w.data());
        for (size_t i = 0; i < cnt; ++i) {
            wt[i].x = (T)w[i].x; wt[i].y = (T)w[i].y;
            w[i].y = -w[i].y;                                         // b[m] = conj(w[m])
        }
        CUDA_TRY(cudaMemcpy(bs.chirp + s, wt.data(), cnt * sizeof(cx<T>), cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy(b + s, w.data(), cnt * sizeof(double2), cudaMemcpyHostToDevice));
        // b[M - m] = b[m] for 0 < m < L: m = s + cnt - 1 - i lands at M - m, ascending in i
        const size_t lo = std::max<size_t>(s, 1), k = s + cnt - lo;
        for (size_t i = 0; i < k; ++i) rev[i] = w[cnt - 1 - i];
        if (k) CUDA_TRY(cudaMemcpy(b + (M - (s + cnt - 1)), rev.data(), k * sizeof(double2), cudaMemcpyHostToDevice));
    }
    CUDA_TRY(cudaDeviceSynchronize());
    // Bh = FFT_M(b) / M in f64, in place (the scale is a power of two: exact): with the inner plan for f64, a temporary f64 plan
    // for f32.  Plan-time launches stay out of the caller's launch record.
    const std::vector<LaunchRec> saved = g_launch_log;
    {
        Plan<double>* p64 = nullptr;
        std::unique_ptr<Plan<double>> tmp;
        if constexpr (std::is_same<T, double>::value) {
            p64 = bs.inner;
        } else {
            if (int32_t st = build_plan<double>(M, device, &p64)) { g_launch_log = saved; return st; }
            tmp.reset(p64);
        }
        Io<double> io;
        io.in_re = reinterpret_cast<const double*>(b); io.in_im = nullptr; io.out_re = reinterpret_cast<double*>(b); io.out_im = nullptr;
        io.in_bstride = io.out_bstride = (long long)M;
        io.in_il = io.out_il = 1;
        int32_t st = run_c2c(*p64, io, 1, 1.0 / (double)M, p64->stream);
        g_launch_log = saved;
        if (st) return st;
        CUDA_TRY(cudaStreamSynchronize(p64->stream));
    }
    if constexpr (std::is_same<T, double>::value) {
        bs.bhat = b_owner.release();
    } else {
        CUDA_TRY(cudaMalloc(&bs.bhat, M * sizeof(cx<T>)));
        chirp_narrow_kernel<T><<<(unsigned)std::min<size_t>((M + 255) / 256, 65536), 256>>>(b, bs.bhat, (long long)M);
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaDeviceSynchronize());
    }
    return bs.w.init(M);                                             // room for one member; batched calls grow it
}

template <typename T>
int32_t build_plan_any(size_t n, int device, int algo, PlanAny<T>** out) {
    if (!out) return fail(PHASTFT_ERR_INVALID_ARG, "out == NULL");
    *out = nullptr;
    if (n == 0) return fail(PHASTFT_ERR_INVALID_ARG, "n must be >= 1");
    if (algo != PHASTFT_ANY_BLUESTEIN && algo != PHASTFT_ANY_MIXED && algo != PHASTFT_ANY_AUTO)
        return fail(PHASTFT_ERR_INVALID_ARG, "algo must be PHASTFT_ANY_BLUESTEIN, PHASTFT_ANY_MIXED or PHASTFT_ANY_AUTO");
    const bool pow2 = is_pow2(n);
    MixedSplit split;
    std::string why;
    const bool mixed = !pow2 && algo != PHASTFT_ANY_BLUESTEIN && mixed_split(n, split, why);
    if (!pow2 && algo == PHASTFT_ANY_MIXED && !mixed) return fail(PHASTFT_ERR_INVALID_ARG, "no mixed-radix plan: " + why);
    if (!pow2 && !mixed && n > ANY_MAX_N)
        return fail(PHASTFT_ERR_INVALID_ARG, "n = " + std::to_string(n) + " is not a power of two and above 2^29 - 1 (its convolution "
                                             "length 2^ceil(log2(2N - 1)) would exceed 2^30)");
    std::unique_ptr<PlanAny<T>> pl(new PlanAny<T>());
    pl->n = n; pl->device = device;
    const char* prec = sizeof(T) == 8 ? " f64" : " f32";
    if (pow2) {
        if (int32_t st = build_plan<T>(n, device, &pl->pow2)) return st;
        pl->description = "n=2^" + std::to_string(ilog2(n)) + prec + " any: power of two | inner: " + pl->pow2->description;
        *out = pl.release();
        return PHASTFT_OK;
    }
    if (mixed) {
        if (int32_t st = build_mixed(pl->mx, n, split, device)) return st;
        pl->description = "n=" + std::to_string(n) + prec + " any: " + mixed_description(split) + " | inner: " + pl->mx.inner->description;
        *out = pl.release();
        return PHASTFT_OK;
    }
    if (int32_t st = build_bluestein(pl->bs, n, device)) return st;
    pl->description = "n=" + std::to_string(n) + prec + " any: Bluestein M=2^" + std::to_string(pl->bs.log2m) + " | inner: " +
                      pl->bs.inner->description;
    *out = pl.release();
    return PHASTFT_OK;
}

enum ChirpKind { CHIRP_PRE, CHIRP_MUL, CHIRP_POST };

// One CHIRP-* kernel over `members` batch members, `per` threads each: a member-major grid of 256-thread blocks (as launch_real),
// several launches when it would exceed 2^31 - 1 blocks.  Launch record: R = M, C = the members of that launch; the kind carries
// -R2C / -C2R for the real modes' CHIRP-PRE and CHIRP-POST, -IL for the interleaved ones.  The real modes with an interleaved
// spectrum run it at the spectrum's end only (CHIRP-POST-R2C-IL, CHIRP-PRE-C2R-IL) and the planar mode's kernel at the other.
template <int MODE, typename T>
int32_t launch_chirp(ChirpKind kind, const ChirpParams<T>& cp, size_t per, size_t members, cudaStream_t stream) {
    const size_t bpm = (per + 255) / 256;
    const size_t max_members = std::max<size_t>(1, grid_blocks_max() / bpm);
    constexpr int PM = chirp_planar<MODE>();
    constexpr bool r2c = PM == CHIRP_R2C_HALVED || PM == CHIRP_R2C_DIRECT, c2r = PM == CHIRP_C2R_HALVED || PM == CHIRP_C2R_DIRECT;
    constexpr bool il = chirp_il<MODE>();
    constexpr int PRE = r2c ? PM : MODE, POST = c2r ? PM : MODE;
    const bool sil = kind == CHIRP_PRE ? chirp_spec_il<PRE>() : chirp_spec_il<POST>();
    for (size_t done = 0; done < members; done += max_members) {
        const size_t nb = std::min(members - done, max_members);
        ChirpParams<T> q = cp;
        const long long off = (long long)done * cp.bstride, ooff = (long long)done * cp.out_bstride;
        if constexpr (MODE == CHIRP_C2C) {
            q.in_re += off; q.in_im += off; q.out_re += off; q.out_im += off;
        } else {
            q.in_re += off;
            if (q.in_im) q.in_im += off;
            q.out_re += ooff;
            if (q.out_im) q.out_im += ooff;
        }
        q.ws += done << cp.log2m;
        q.blocks_per_member = (unsigned)bpm;
        const dim3 grid((unsigned)(nb * bpm));
        if (kind == CHIRP_MUL) chirp_mul_kernel<T><<<grid, 256, 0, stream>>>(q);
        else if constexpr (il) launch_chirp_il<T>(MODE, kind == CHIRP_POST, q, grid.x, stream);
        else if (kind == CHIRP_PRE) {
            if constexpr (chirp_spec_il<PRE>()) launch_chirp_real_il<T>(PRE, q, grid.x, stream);
            else chirp_pre_kernel<T, PRE><<<grid, 256, 0, stream>>>(q);
        } else {
            if constexpr (chirp_spec_il<POST>()) launch_chirp_real_il<T>(POST, q, grid.x, stream);
            else chirp_post_kernel<T, POST><<<grid, 256, 0, stream>>>(q);
        }
        CUDA_TRY(cudaGetLastError());
        const char* name = kind == CHIRP_MUL ? "CHIRP-MUL"
                           : kind == CHIRP_PRE ? (r2c ? "CHIRP-PRE-R2C" : c2r ? (sil ? "CHIRP-PRE-C2R-IL" : "CHIRP-PRE-C2R") : il ? "CHIRP-PRE-IL" : "CHIRP-PRE")
                                               : (r2c ? (sil ? "CHIRP-POST-R2C-IL" : "CHIRP-POST-R2C") : c2r ? "CHIRP-POST-C2R" : il ? "CHIRP-POST-IL" : "CHIRP-POST");
        note_launch({name, 1 << cp.log2m, 0, (int)nb, 256, 0, "plain", false});
    }
    return PHASTFT_OK;
}

// One Bluestein call of `batch` members: CHIRP-PRE, the M-point transform, CHIRP-MUL, the M-point transform, CHIRP-POST, with
// the kernels' MODE at both ends.  `cp` carries the caller's arrays, strides, scale and W_N table; this fills in the rest.  The
// workspace follows AnyWorkspace's protocol (`reserve_fn` names the call that grows it ahead of a capture).
template <int MODE, typename T>
int32_t bluestein_run(const Bluestein<T>& bs, ChirpParams<T> cp, size_t batch, cudaStream_t stream, const char* reserve_fn) {
    DeviceGuard g(bs.device);
    const size_t M = size_t(1) << bs.log2m;
    std::lock_guard<std::mutex> lock(bs.w.mu);
    bool capturing = false;
    if (int32_t st = bs.w.acquire(batch << bs.log2m, batch, stream, reserve_fn, capturing)) return st;
    cp.ws = bs.w.ws; cp.chirp = bs.chirp; cp.bhat = bs.bhat;
    cp.n = (long long)bs.l; cp.log2m = bs.log2m;
    constexpr size_t V = Cx16<T>::V;
    Io<T> io;
    io.in_re = reinterpret_cast<const T*>(bs.w.ws); io.in_im = nullptr;
    io.out_re = reinterpret_cast<T*>(bs.w.ws); io.out_im = nullptr;
    io.in_bstride = io.out_bstride = (long long)M;
    io.in_il = io.out_il = 1;
    const size_t post = (size_t)chirp_post_count<MODE>((long long)bs.l);
    if (int32_t st = launch_chirp<MODE>(CHIRP_PRE, cp, M / V, batch, stream)) return st;
    if (int32_t st = run_c2c(*bs.inner, io, batch, T(1), stream)) return st;
    if (int32_t st = launch_chirp<MODE>(CHIRP_MUL, cp, M / V, batch, stream)) return st;
    if (int32_t st = run_c2c(*bs.inner, io, batch, T(1), stream)) return st;
    if (int32_t st = launch_chirp<MODE>(CHIRP_POST, cp, (post + V - 1) / V, batch, stream)) return st;
    return bs.w.release(stream, capturing);
}

// Every allocation a call of `batch` would make: the inner plan's workspace and the Bluestein one.
template <typename T>
int32_t bluestein_reserve(const Bluestein<T>& bs, size_t batch) {
    if (int32_t st = plan_reserve(bs.inner, batch)) return st;
    DeviceGuard g(bs.device);
    std::lock_guard<std::mutex> lock(bs.w.mu);
    return bs.w.grow(batch << bs.log2m, batch);
}

// planar, in place, device pointers: the semantics of fft_dev for any N
template <typename T>
int32_t any_dev(const PlanAny<T>* pl, T* d_re, T* d_im, int direction, size_t batch, size_t bstride, cudaStream_t stream) {
    if (!pl || !d_re || !d_im) return fail(PHASTFT_ERR_INVALID_ARG, "NULL argument");
    if (direction != PHASTFT_FORWARD && direction != PHASTFT_REVERSE) return fail(PHASTFT_ERR_INVALID_ARG, "direction must be 1 or -1");
    if (batch > 1 && bstride < pl->n) return fail(PHASTFT_ERR_INVALID_ARG, "batch_stride < N");
    if (pl->pow2) return fft_dev(pl->pow2, d_re, d_im, direction, batch, bstride, stream);
    if (batch == 0) return PHASTFT_OK;
    // the reverse direction by the swap trick (fft_dev): re and im exchanged on the way in and out, 1/N folded into CHIRP-POST
    const bool fwd = direction == PHASTFT_FORWARD;
    if (pl->mx.inner)
        return mixed_run<CHIRP_C2C>(pl->mx, fwd ? d_re : d_im, fwd ? d_im : d_re, bstride, fwd ? d_re : d_im, fwd ? d_im : d_re, bstride,
                                    fwd ? T(1) : T(1) / (T)pl->n, batch, stream, "phastft_plan_any_*_reserve");
    ChirpParams<T> cp;
    memset(&cp, 0, sizeof(cp));
    cp.in_re = cp.out_re = fwd ? d_re : d_im;
    cp.in_im = cp.out_im = fwd ? d_im : d_re;
    cp.bstride = cp.out_bstride = (long long)bstride;
    cp.scale = fwd ? T(1) : T(1) / (T)pl->n;
    return bluestein_run<CHIRP_C2C>(pl->bs, cp, batch, stream, "phastft_plan_any_*_reserve");
}

// interleaved, in place, device pointers: the semantics of any_dev on Complex<T> members b * bstride complex values apart.  The
// Bluestein and mixed paths run any_dev's kernels with the interleaved modes at the ends (bit-identical results); powers of
// two run fft_interleaved_dev.
template <typename T>
int32_t any_interleaved_dev(const PlanAny<T>* pl, T* d_sig, int direction, size_t batch, size_t bstride, cudaStream_t stream) {
    if (!pl || !d_sig) return fail(PHASTFT_ERR_INVALID_ARG, "NULL argument");
    if (direction != PHASTFT_FORWARD && direction != PHASTFT_REVERSE) return fail(PHASTFT_ERR_INVALID_ARG, "direction must be 1 or -1");
    if (batch > 1 && bstride < pl->n) return fail(PHASTFT_ERR_INVALID_ARG, "batch_stride < N");
    if (int32_t st = check_pair_alignment(d_sig, "d_signal")) return st;
    if (pl->pow2) return fft_interleaved_dev(pl->pow2, d_sig, direction, batch, bstride, stream);
    if (batch == 0) return PHASTFT_OK;
    const bool fwd = direction == PHASTFT_FORWARD;
    const T scale = fwd ? T(1) : T(1) / (T)pl->n;
    const char* res = "phastft_plan_any_*_reserve";
    if (pl->mx.inner)
        return fwd ? mixed_run<CHIRP_C2C_IL, T>(pl->mx, d_sig, nullptr, 2 * bstride, d_sig, nullptr, bstride, scale, batch, stream, res)
                   : mixed_run<CHIRP_C2C_IL_SWAP, T>(pl->mx, d_sig, nullptr, 2 * bstride, d_sig, nullptr, bstride, scale, batch, stream, res);
    ChirpParams<T> cp;
    memset(&cp, 0, sizeof(cp));
    cp.in_re = cp.out_re = d_sig;
    cp.bstride = cp.out_bstride = 2 * (long long)bstride;
    cp.scale = scale;
    return fwd ? bluestein_run<CHIRP_C2C_IL>(pl->bs, cp, batch, stream, res) : bluestein_run<CHIRP_C2C_IL_SWAP>(pl->bs, cp, batch, stream, res);
}

template <typename T>
int32_t any_reserve(const PlanAny<T>* pl, size_t batch) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (pl->pow2) return plan_reserve(pl->pow2, batch);
    if (pl->mx.inner) return mixed_reserve(pl->mx, batch);
    return bluestein_reserve(pl->bs, batch);
}

// host slices: H2D, run, D2H, synchronous (fft_host for any N)
template <typename T>
int32_t any_host(const PlanAny<T>* pl, T* re, size_t len_re, T* im, size_t len_im, int direction) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (len_re != len_im) return fail(PHASTFT_ERR_LEN_MISMATCH);
    if (len_re != pl->n) return fail(PHASTFT_ERR_PLAN_MISMATCH, "slice length " + std::to_string(len_re) + ", plan n = " + std::to_string(pl->n));
    if (direction != PHASTFT_FORWARD && direction != PHASTFT_REVERSE) return fail(PHASTFT_ERR_INVALID_ARG, "direction must be 1 or -1");
    if (!re || !im) return fail(PHASTFT_ERR_INVALID_ARG, "NULL slice");
    if (pl->pow2) return fft_host(pl->pow2, re, len_re, im, len_im, direction);
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> host_lock(pl->host_mu);
    {
        std::lock_guard<std::mutex> lock(pl->workspace().mu);   // released before any_dev, which takes it
        if (!pl->stage_re) CUDA_TRY(cudaMalloc(&pl->stage_re, pl->n * sizeof(T)));
        if (!pl->stage_im) CUDA_TRY(cudaMalloc(&pl->stage_im, pl->n * sizeof(T)));
    }
    cudaStream_t s = pl->host_stream();
    const size_t bytes = pl->n * sizeof(T);
    CUDA_TRY(scribble(pl->workspace().scribble_on, pl->stage_re, bytes, s));
    CUDA_TRY(scribble(pl->workspace().scribble_on, pl->stage_im, bytes, s));
    CUDA_TRY(cudaMemcpyAsync(pl->stage_re, re, bytes, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(pl->stage_im, im, bytes, cudaMemcpyHostToDevice, s));
    if (int32_t st = any_dev(pl, pl->stage_re, pl->stage_im, direction, 1, pl->n, s)) return st;
    CUDA_TRY(cudaMemcpyAsync(re, pl->stage_re, bytes, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(im, pl->stage_im, bytes, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return PHASTFT_OK;
}

// an interleaved host slice of N complex values: H2D, run, D2H, synchronous
template <typename T>
int32_t any_interleaved_host(const PlanAny<T>* pl, T* sig, size_t len_complex, int direction) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (len_complex != pl->n)
        return fail(PHASTFT_ERR_PLAN_MISMATCH, "slice length " + std::to_string(len_complex) + ", plan n = " + std::to_string(pl->n));
    if (direction != PHASTFT_FORWARD && direction != PHASTFT_REVERSE) return fail(PHASTFT_ERR_INVALID_ARG, "direction must be 1 or -1");
    if (!sig) return fail(PHASTFT_ERR_INVALID_ARG, "NULL slice");
    if (pl->pow2) return fft_interleaved_host(pl->pow2, sig, len_complex, direction);
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> host_lock(pl->host_mu);
    {
        std::lock_guard<std::mutex> lock(pl->workspace().mu);   // released before any_interleaved_dev, which takes it
        if (!pl->stage_il) CUDA_TRY(cudaMalloc(&pl->stage_il, 2 * pl->n * sizeof(T)));
    }
    cudaStream_t s = pl->host_stream();
    const size_t bytes = 2 * pl->n * sizeof(T);
    CUDA_TRY(scribble(pl->workspace().scribble_on, pl->stage_il, bytes, s));
    CUDA_TRY(cudaMemcpyAsync(pl->stage_il, sig, bytes, cudaMemcpyHostToDevice, s));
    if (int32_t st = any_interleaved_dev(pl, pl->stage_il, direction, 1, pl->n, s)) return st;
    CUDA_TRY(cudaMemcpyAsync(sig, pl->stage_il, bytes, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return PHASTFT_OK;
}

// =================================================================================================
// real input of any length: r2c / c2r over Bluestein (the CHIRP-*-R2C / -C2R kernel modes) or the mixed-radix path (the same
// modes of SMOOTH-PRE and the last ODD pass, and SMOOTH-POST-R2C)
// =================================================================================================
// Even N up to 2^30 - 2 take the halved path (Bluestein of L = N/2, M <= 2^30); odd N the direct one (L = N, up to 2^29 - 1);
// powers of two from 4 the r2c plan.  On the mixed path even N go up to 2^31 - 2 (L = N/2 <= 2^30 - 1).
constexpr size_t R2C_ANY_MAX_EVEN = (size_t(1) << 30) - 2;

template <typename T>
struct PlanR2cAny {
    size_t n = 0;
    int device = 0;
    bool halved = false;               // even N: the L-point transform of z[m] = x[2m] + i x[2m+1], L = N/2; odd N: L = N
    PlanR2c<T>* pow2 = nullptr;        // N a power of two >= 4: the r2c plan, run as it is
    Bluestein<T> bs;                   // otherwise: Bluestein of L ...
    Mixed<T> mx;                       // ... or the mixed-radix path of L (mx.inner set)
    cx<T>* wn = nullptr;               // halved Bluestein: W_N^k for k = 0 .. floor(L/2), rounded to T
    TwoLevelRoots<T> wn2;              // halved mixed: W_N^e for e < L, two-level
    AnyWorkspace<T>& workspace() const { return mx.inner ? mx.w : bs.w; }
    cudaStream_t host_stream() const { return (mx.inner ? mx.inner : bs.inner)->stream; }
    mutable std::mutex host_mu;        // held for a whole *_host call (lock order: host_mu, then the workspace's mu)
    mutable T* stage_real = nullptr;   // host-API staging: N reals, floor(N/2) + 1 bins
    mutable T* stage_re = nullptr;
    mutable T* stage_im = nullptr;
    mutable T* stage_il_real = nullptr;   // the interleaved host calls' staging (N reals, floor(N/2) + 1 complex bins), allocated
    mutable T* stage_il_spec = nullptr;   // by the first such call
    std::string description;
    ~PlanR2cAny() {
        DeviceGuard g(device);
        for (void* p : {(void*)wn, (void*)wn2.blob, (void*)stage_real, (void*)stage_re, (void*)stage_im, (void*)stage_il_real,
                        (void*)stage_il_spec})
            if (p) cudaFree(p);
        delete pow2;
    }
};

template <typename T>
int32_t build_plan_r2c_any(size_t n, int device, int algo, PlanR2cAny<T>** out) {
    if (!out) return fail(PHASTFT_ERR_INVALID_ARG, "out == NULL");
    *out = nullptr;
    if (n == 0) return fail(PHASTFT_ERR_INVALID_ARG, "n must be >= 1");
    if (algo != PHASTFT_ANY_BLUESTEIN && algo != PHASTFT_ANY_MIXED && algo != PHASTFT_ANY_AUTO)
        return fail(PHASTFT_ERR_INVALID_ARG, "algo must be PHASTFT_ANY_BLUESTEIN, PHASTFT_ANY_MIXED or PHASTFT_ANY_AUTO");
    const bool pow2 = n >= 4 && is_pow2(n);
    if (pow2 && n > (size_t(1) << 31)) return fail(PHASTFT_ERR_INVALID_ARG, "n = " + std::to_string(n) + " is a power of two above 2^31");
    // the mixed path runs on L = N/2 (halved) or N (direct) when that length is eligible
    const size_t l = n % 2 == 0 ? n / 2 : n;
    MixedSplit split;
    std::string why;
    const bool mixed = !pow2 && algo != PHASTFT_ANY_BLUESTEIN && mixed_split(l, split, why, n % 2 == 0 ? "L = n/2" : "n");
    if (!pow2 && algo == PHASTFT_ANY_MIXED && !mixed) return fail(PHASTFT_ERR_INVALID_ARG, "no mixed-radix plan: " + why);
    if (!pow2 && !mixed && n % 2 == 0 && n > R2C_ANY_MAX_EVEN)
        return fail(PHASTFT_ERR_INVALID_ARG, "even n = " + std::to_string(n) + " above 2^30 - 2 (its half-length convolution would "
                                             "exceed 2^30 points)");
    if (!mixed && n % 2 && n > ANY_MAX_N)
        return fail(PHASTFT_ERR_INVALID_ARG, "odd n = " + std::to_string(n) + " above 2^29 - 1 (its convolution would exceed 2^30 points)");
    std::unique_ptr<PlanR2cAny<T>> pl(new PlanR2cAny<T>());
    pl->n = n; pl->device = device;
    const std::string head = (pow2 ? "n=2^" + std::to_string(ilog2(n)) : "n=" + std::to_string(n)) + (sizeof(T) == 8 ? " f64" : " f32") +
                             " r2c any: ";
    if (pow2) {
        if (int32_t st = build_plan_r2c<T>(n, device, &pl->pow2)) return st;
        pl->description = head + "power of two | ";       // + the r2c plan's describe(), built per call (it reads the environment)
        *out = pl.release();
        return PHASTFT_OK;
    }
    pl->halved = n % 2 == 0;
    if (mixed) {
        if (int32_t st = build_mixed(pl->mx, l, split, device)) return st;
        if (pl->halved) {
            DeviceGuard g(device);
            if (int32_t st = build_two_level(pl->wn2, n, l)) return st;
        }
        pl->description = head + (pl->halved ? "halved, " : "direct, ") + mixed_description(split) + " | inner: " +
                          pl->mx.inner->description;
        *out = pl.release();
        return PHASTFT_OK;
    }
    if (int32_t st = build_bluestein(pl->bs, l, device)) return st;
    if (pl->halved) {
        // W_N^k = exp(-2 pi i k / N) by exact integer reduction in long double, rounded to T, for the k <= L/2 the kernels read
        DeviceGuard g(device);
        const size_t cnt = l / 2 + 1;
        std::vector<double2> w(cnt);
        host_parallel(cnt, [&](size_t k) { root_of_unity_any(k, n, w[k].x, w[k].y); });
        std::vector<cx<T>> wt(cnt);
        for (size_t k = 0; k < cnt; ++k) { wt[k].x = (T)w[k].x; wt[k].y = (T)w[k].y; }
        CUDA_TRY(cudaMalloc(&pl->wn, cnt * sizeof(cx<T>)));
        CUDA_TRY(cudaMemcpy(pl->wn, wt.data(), cnt * sizeof(cx<T>), cudaMemcpyHostToDevice));
    }
    pl->description = head + (pl->halved ? "halved" : "direct") + ", Bluestein L=" + std::to_string(l) + " M=2^" +
                      std::to_string(pl->bs.log2m) + " | inner: " + pl->bs.inner->description;
    *out = pl.release();
    return PHASTFT_OK;
}

template <typename T>
std::string r2c_any_description(const PlanR2cAny<T>* pl) {
    return pl->pow2 ? pl->description + r2c_description(pl->pow2, 1) : pl->description;
}

// Member b reads N reals at d_in + b * in_stride and writes floor(N/2) + 1 bins at out_stride * b.  Powers of two run
// r2c_batch_dev with its rules; otherwise in_stride >= N, out_stride >= floor(N/2) + 1, and for even N (read as pairs) an even
// in_stride and a base aligned to 2 * sizeof(T).
template <typename T>
int32_t r2c_any_dev(const PlanR2cAny<T>* pl, const T* d_in, size_t in_stride, T* d_ore, T* d_oim, size_t out_stride, size_t batch,
                    cudaStream_t stream) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (pl->pow2) return r2c_batch_dev(pl->pow2, d_in, in_stride, d_ore, d_oim, out_stride, batch, stream);
    if (!d_in) return fail(PHASTFT_ERR_INVALID_ARG, "d_input == NULL");
    if (!d_ore) return fail(PHASTFT_ERR_INVALID_ARG, "d_out_re == NULL");
    if (!d_oim) return fail(PHASTFT_ERR_INVALID_ARG, "d_out_im == NULL");
    const size_t n = pl->n, bins = n / 2 + 1;
    if (in_stride < n) return fail(PHASTFT_ERR_INVALID_ARG, "in_stride must be >= N = " + std::to_string(n) + " (got " + std::to_string(in_stride) + ")");
    if (out_stride < bins)
        return fail(PHASTFT_ERR_INVALID_ARG, "out_stride must be >= N/2 + 1 = " + std::to_string(bins) + " (got " + std::to_string(out_stride) + ")");
    if (pl->halved) {
        if (in_stride % 2) return fail(PHASTFT_ERR_INVALID_ARG, "in_stride must be even for even N (the input is read as pairs)");
        if (int32_t st = check_pair_alignment(d_in, "d_input")) return st;
    }
    if (batch == 0) return PHASTFT_OK;
    const char* res = "phastft_plan_r2c_any_*_reserve";
    if (pl->mx.inner)
        return pl->halved ? mixed_run<CHIRP_R2C_HALVED, T>(pl->mx, d_in, nullptr, in_stride, d_ore, d_oim, out_stride, T(1), batch, stream,
                                                        res, &pl->wn2)
                          : mixed_run<CHIRP_R2C_DIRECT, T>(pl->mx, d_in, nullptr, in_stride, d_ore, d_oim, out_stride, T(1), batch, stream,
                                                        res);
    ChirpParams<T> cp;
    memset(&cp, 0, sizeof(cp));
    cp.in_re = d_in; cp.out_re = d_ore; cp.out_im = d_oim;
    cp.bstride = (long long)in_stride; cp.out_bstride = (long long)out_stride;
    cp.scale = T(1);
    cp.wn = pl->wn;
    return pl->halved ? bluestein_run<CHIRP_R2C_HALVED>(pl->bs, cp, batch, stream, res)
                      : bluestein_run<CHIRP_R2C_DIRECT>(pl->bs, cp, batch, stream, res);
}

// Member b reads floor(N/2) + 1 bins at in_stride * b and writes N reals at d_out + b * out_stride, scaled so that
// c2r(r2c(x)) == x.  The mirror of r2c_any_dev's rules.
template <typename T>
int32_t c2r_any_dev(const PlanR2cAny<T>* pl, const T* d_ire, const T* d_iim, size_t in_stride, T* d_out, size_t out_stride, size_t batch,
                    cudaStream_t stream) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (pl->pow2) return c2r_batch_dev(pl->pow2, d_ire, d_iim, in_stride, d_out, out_stride, (T*)nullptr, (T*)nullptr, batch, stream);
    if (!d_ire) return fail(PHASTFT_ERR_INVALID_ARG, "d_in_re == NULL");
    if (!d_iim) return fail(PHASTFT_ERR_INVALID_ARG, "d_in_im == NULL");
    if (!d_out) return fail(PHASTFT_ERR_INVALID_ARG, "d_output == NULL");
    const size_t n = pl->n, bins = n / 2 + 1;
    if (in_stride < bins)
        return fail(PHASTFT_ERR_INVALID_ARG, "in_stride must be >= N/2 + 1 = " + std::to_string(bins) + " (got " + std::to_string(in_stride) + ")");
    if (out_stride < n) return fail(PHASTFT_ERR_INVALID_ARG, "out_stride must be >= N = " + std::to_string(n) + " (got " + std::to_string(out_stride) + ")");
    if (pl->halved) {
        if (out_stride % 2) return fail(PHASTFT_ERR_INVALID_ARG, "out_stride must be even for even N (the output is written as pairs)");
        if (int32_t st = check_pair_alignment(d_out, "d_output")) return st;
    }
    if (batch == 0) return PHASTFT_OK;
    const char* res = "phastft_plan_r2c_any_*_reserve";
    if (pl->mx.inner) {
        const T scale = T(1) / (T)pl->mx.n;
        // the halved c2r stores the pairs (y[2k], y[2k+1]): its member stride counts pairs
        return pl->halved ? mixed_run<CHIRP_C2R_HALVED, T>(pl->mx, d_ire, d_iim, in_stride, d_out, nullptr, out_stride / 2, scale, batch,
                                                        stream, res, &pl->wn2)
                          : mixed_run<CHIRP_C2R_DIRECT, T>(pl->mx, d_ire, d_iim, in_stride, d_out, nullptr, out_stride, scale, batch,
                                                        stream, res);
    }
    ChirpParams<T> cp;
    memset(&cp, 0, sizeof(cp));
    cp.in_re = d_ire; cp.in_im = d_iim; cp.out_re = d_out;
    cp.bstride = (long long)in_stride; cp.out_bstride = (long long)out_stride;
    cp.scale = T(1) / (T)pl->bs.l;
    cp.wn = pl->wn;
    return pl->halved ? bluestein_run<CHIRP_C2R_HALVED>(pl->bs, cp, batch, stream, res)
                      : bluestein_run<CHIRP_C2R_DIRECT>(pl->bs, cp, batch, stream, res);
}

// The same transforms with the spectrum as interleaved Complex<T> bins: member b's floor(N/2) + 1 bins start at complex element
// b * spec_stride of d_spec (>= floor(N/2) + 1), aligned to 2 * sizeof(T).  The real side keeps the planar call's rules.  Every
// path runs the planar call's launches with the spectrum's end kernels in their interleaved modes, so the results are the
// planar call's bit for bit.
template <typename T>
int32_t check_spec_il(const PlanR2cAny<T>* pl, const T* d_real, const T* d_spec, size_t real_stride, size_t spec_stride, bool r2c) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (!d_real) return fail(PHASTFT_ERR_INVALID_ARG, r2c ? "d_input == NULL" : "d_output == NULL");
    if (!d_spec) return fail(PHASTFT_ERR_INVALID_ARG, r2c ? "d_out == NULL" : "d_in == NULL");
    const size_t n = pl->n, bins = n / 2 + 1;
    const char* rs = r2c ? "in_stride" : "out_stride";
    const char* ss = r2c ? "out_stride_complex" : "in_stride_complex";
    if (real_stride < n) return fail(PHASTFT_ERR_INVALID_ARG, std::string(rs) + " must be >= N = " + std::to_string(n) + " (got " + std::to_string(real_stride) + ")");
    if (spec_stride < bins)
        return fail(PHASTFT_ERR_INVALID_ARG, std::string(ss) + " must be >= N/2 + 1 = " + std::to_string(bins) + " (got " + std::to_string(spec_stride) + ")");
    if (n % 2 == 0) {   // the real side is read or written as pairs
        if (real_stride % 2) return fail(PHASTFT_ERR_INVALID_ARG, std::string(rs) + " must be even for even N (the reals are accessed as pairs)");
        if (int32_t st = check_pair_alignment(d_real, r2c ? "d_input" : "d_output")) return st;
    }
    return check_pair_alignment(d_spec, r2c ? "d_out" : "d_in");
}

template <typename T>
int32_t r2c_il_any_dev(const PlanR2cAny<T>* pl, const T* d_in, size_t in_stride, T* d_out, size_t out_stride, size_t batch,
                       cudaStream_t stream) {
    if (int32_t st = check_spec_il(pl, d_in, d_out, in_stride, out_stride, true)) return st;
    if (batch == 0) return PHASTFT_OK;
    if (pl->pow2) return r2c_il_dev(pl->pow2, d_in, in_stride, d_out, out_stride, batch, stream);
    const char* res = "phastft_plan_r2c_any_*_reserve";
    if (pl->mx.inner)
        return pl->halved ? mixed_run<CHIRP_R2C_HALVED_IL, T>(pl->mx, d_in, nullptr, in_stride, d_out, nullptr, out_stride, T(1), batch,
                                                           stream, res, &pl->wn2)
                          : mixed_run<CHIRP_R2C_DIRECT_IL, T>(pl->mx, d_in, nullptr, in_stride, d_out, nullptr, out_stride, T(1), batch,
                                                           stream, res);
    ChirpParams<T> cp;
    memset(&cp, 0, sizeof(cp));
    cp.in_re = d_in; cp.out_re = d_out;
    cp.bstride = (long long)in_stride; cp.out_bstride = 2 * (long long)out_stride;
    cp.scale = T(1);
    cp.wn = pl->wn;
    return pl->halved ? bluestein_run<CHIRP_R2C_HALVED_IL>(pl->bs, cp, batch, stream, res)
                      : bluestein_run<CHIRP_R2C_DIRECT_IL>(pl->bs, cp, batch, stream, res);
}

template <typename T>
int32_t c2r_il_any_dev(const PlanR2cAny<T>* pl, const T* d_in, size_t in_stride, T* d_out, size_t out_stride, size_t batch,
                       cudaStream_t stream) {
    if (int32_t st = check_spec_il(pl, d_out, d_in, out_stride, in_stride, false)) return st;
    if (batch == 0) return PHASTFT_OK;
    if (pl->pow2) return c2r_il_dev(pl->pow2, d_in, in_stride, d_out, out_stride, batch, stream);
    const char* res = "phastft_plan_r2c_any_*_reserve";
    if (pl->mx.inner) {
        const T scale = T(1) / (T)pl->mx.n;
        return pl->halved ? mixed_run<CHIRP_C2R_HALVED_IL, T>(pl->mx, d_in, nullptr, 2 * in_stride, d_out, nullptr, out_stride / 2, scale,
                                                           batch, stream, res, &pl->wn2)
                          : mixed_run<CHIRP_C2R_DIRECT_IL, T>(pl->mx, d_in, nullptr, 2 * in_stride, d_out, nullptr, out_stride, scale,
                                                           batch, stream, res);
    }
    ChirpParams<T> cp;
    memset(&cp, 0, sizeof(cp));
    cp.in_re = d_in; cp.out_re = d_out;
    cp.bstride = 2 * (long long)in_stride; cp.out_bstride = (long long)out_stride;
    cp.scale = T(1) / (T)pl->bs.l;
    cp.wn = pl->wn;
    return pl->halved ? bluestein_run<CHIRP_C2R_HALVED_IL>(pl->bs, cp, batch, stream, res)
                      : bluestein_run<CHIRP_C2R_DIRECT_IL>(pl->bs, cp, batch, stream, res);
}

template <typename T>
int32_t r2c_any_reserve(const PlanR2cAny<T>* pl, size_t batch) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (pl->pow2) return r2c_reserve(pl->pow2, batch);
    if (pl->mx.inner) return mixed_reserve(pl->mx, batch);
    return bluestein_reserve(pl->bs, batch);
}

// Caller holds host_mu.  Under PHASTFT_SCRIBBLE=1 the staging is poisoned on `s` before the call's copies.
template <typename T>
int32_t ensure_r2c_any_staging(const PlanR2cAny<T>* pl, cudaStream_t s) {
    std::lock_guard<std::mutex> lock(pl->workspace().mu);   // released before the device call, which takes it
    if (!pl->stage_real) CUDA_TRY(cudaMalloc(&pl->stage_real, pl->n * sizeof(T)));
    if (!pl->stage_re) CUDA_TRY(cudaMalloc(&pl->stage_re, (pl->n / 2 + 1) * sizeof(T)));
    if (!pl->stage_im) CUDA_TRY(cudaMalloc(&pl->stage_im, (pl->n / 2 + 1) * sizeof(T)));
    const bool on = pl->workspace().scribble_on;
    CUDA_TRY(scribble(on, pl->stage_real, pl->n * sizeof(T), s));
    CUDA_TRY(scribble(on, pl->stage_re, (pl->n / 2 + 1) * sizeof(T), s));
    CUDA_TRY(scribble(on, pl->stage_im, (pl->n / 2 + 1) * sizeof(T), s));
    return PHASTFT_OK;
}

// host slices, synchronous: the length codes of r2c_host / c2r_host with N/2 + 1 = floor(N/2) + 1
template <typename T>
int32_t r2c_any_host(const PlanR2cAny<T>* pl, const T* in, size_t len_in, T* ore, size_t len_ore, T* oim, size_t len_oim) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (pl->pow2) return r2c_host(pl->pow2, in, len_in, ore, len_ore, oim, len_oim);
    const size_t n = pl->n, bins = n / 2 + 1;
    if (len_in != n) return fail(PHASTFT_ERR_INPUT_LEN);
    if (len_ore != bins) return fail(PHASTFT_ERR_OUTPUT_RE_LEN);
    if (len_oim != bins) return fail(PHASTFT_ERR_OUTPUT_IM_LEN);
    if (!in || !ore || !oim) return fail(PHASTFT_ERR_INVALID_ARG, "NULL slice");
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> host_lock(pl->host_mu);
    cudaStream_t s = pl->host_stream();
    if (int32_t st = ensure_r2c_any_staging(pl, s)) return st;
    CUDA_TRY(cudaMemcpyAsync(pl->stage_real, in, n * sizeof(T), cudaMemcpyHostToDevice, s));
    if (int32_t st = r2c_any_dev(pl, pl->stage_real, n, pl->stage_re, pl->stage_im, bins, 1, s)) return st;
    CUDA_TRY(cudaMemcpyAsync(ore, pl->stage_re, bins * sizeof(T), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(oim, pl->stage_im, bins * sizeof(T), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return PHASTFT_OK;
}

// Caller holds host_mu: the interleaved host calls' staging, poisoned under PHASTFT_SCRIBBLE=1 like the planar one.  Allocated
// under the lock the device call takes (the r2c plan's for a power of two, else the workspace's), released before that call.
template <typename T>
int32_t ensure_r2c_any_il_staging(const PlanR2cAny<T>* pl, cudaStream_t s) {
    const size_t n = pl->n, bins = n / 2 + 1;
    {
        std::lock_guard<std::mutex> lock(pl->pow2 ? pl->pow2->mu : pl->workspace().mu);
        if (!pl->stage_il_real) CUDA_TRY(cudaMalloc(&pl->stage_il_real, n * sizeof(T)));
        if (!pl->stage_il_spec) CUDA_TRY(cudaMalloc(&pl->stage_il_spec, 2 * bins * sizeof(T)));
    }
    const bool on = pl->pow2 ? pl->pow2->inner->scribble_on : pl->workspace().scribble_on;
    CUDA_TRY(scribble(on, pl->stage_il_real, n * sizeof(T), s));
    CUDA_TRY(scribble(on, pl->stage_il_spec, 2 * bins * sizeof(T), s));
    return PHASTFT_OK;
}

// interleaved host slices, synchronous: the planar host calls' length codes (spectrum lengths in complex values)
template <typename T>
int32_t r2c_il_any_host(const PlanR2cAny<T>* pl, const T* in, size_t len_in, T* out, size_t len_out) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    const size_t n = pl->n, bins = n / 2 + 1;
    if (len_in != n) return fail(PHASTFT_ERR_INPUT_LEN);
    if (len_out != bins) return fail(PHASTFT_ERR_OUTPUT_RE_LEN);
    if (!in || !out) return fail(PHASTFT_ERR_INVALID_ARG, "NULL slice");
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> host_lock(pl->host_mu);
    cudaStream_t s = pl->pow2 ? pl->pow2->inner->stream : pl->host_stream();
    if (int32_t st = ensure_r2c_any_il_staging(pl, s)) return st;
    CUDA_TRY(cudaMemcpyAsync(pl->stage_il_real, in, n * sizeof(T), cudaMemcpyHostToDevice, s));
    if (int32_t st = r2c_il_any_dev(pl, pl->stage_il_real, n, pl->stage_il_spec, bins, 1, s)) return st;
    CUDA_TRY(cudaMemcpyAsync(out, pl->stage_il_spec, 2 * bins * sizeof(T), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return PHASTFT_OK;
}

template <typename T>
int32_t c2r_il_any_host(const PlanR2cAny<T>* pl, const T* in, size_t len_in, T* out, size_t len_out) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    const size_t n = pl->n, bins = n / 2 + 1;
    if (len_out != n) return fail(PHASTFT_ERR_OUTPUT_LEN);
    if (len_in != bins) return fail(PHASTFT_ERR_INPUT_RE_LEN);
    if (!in || !out) return fail(PHASTFT_ERR_INVALID_ARG, "NULL slice");
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> host_lock(pl->host_mu);
    cudaStream_t s = pl->pow2 ? pl->pow2->inner->stream : pl->host_stream();
    if (int32_t st = ensure_r2c_any_il_staging(pl, s)) return st;
    CUDA_TRY(cudaMemcpyAsync(pl->stage_il_spec, in, 2 * bins * sizeof(T), cudaMemcpyHostToDevice, s));
    if (int32_t st = c2r_il_any_dev(pl, pl->stage_il_spec, bins, pl->stage_il_real, n, 1, s)) return st;
    CUDA_TRY(cudaMemcpyAsync(out, pl->stage_il_real, n * sizeof(T), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return PHASTFT_OK;
}

template <typename T>
int32_t c2r_any_host(const PlanR2cAny<T>* pl, const T* ire, size_t len_ire, const T* iim, size_t len_iim, T* out, size_t len_out) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (pl->pow2) return c2r_host(pl->pow2, ire, len_ire, iim, len_iim, out, len_out, (T*)nullptr, 0, (T*)nullptr, 0);
    const size_t n = pl->n, bins = n / 2 + 1;
    if (len_out != n) return fail(PHASTFT_ERR_OUTPUT_LEN);
    if (len_ire != bins) return fail(PHASTFT_ERR_INPUT_RE_LEN);
    if (len_iim != bins) return fail(PHASTFT_ERR_INPUT_IM_LEN);
    if (!ire || !iim || !out) return fail(PHASTFT_ERR_INVALID_ARG, "NULL slice");
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> host_lock(pl->host_mu);
    cudaStream_t s = pl->host_stream();
    if (int32_t st = ensure_r2c_any_staging(pl, s)) return st;
    CUDA_TRY(cudaMemcpyAsync(pl->stage_re, ire, bins * sizeof(T), cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(pl->stage_im, iim, bins * sizeof(T), cudaMemcpyHostToDevice, s));
    if (int32_t st = c2r_any_dev(pl, pl->stage_re, pl->stage_im, bins, pl->stage_real, n, 1, s)) return st;
    CUDA_TRY(cudaMemcpyAsync(out, pl->stage_real, n * sizeof(T), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return PHASTFT_OK;
}

// =================================================================================================
// DCT / DST types 2 and 3 of any length: DCT-PRE, the real any-length plan's interleaved r2c (type 2) or c2r (type 3) on the
// plan's workspace, DCT-POST (fft_kernels.cuh, Makhoul 1980)
// =================================================================================================
template <typename T>
struct PlanDct {
    size_t n = 0;
    int device = 0;
    PlanR2cAny<T>* inner = nullptr;    // the N-point real plan
    TwoLevelRoots<T> w4n;              // W_(4N)^k for k <= N/2
    // per call of `batch` members: batch x vstride() reals v, then batch x (N/2 + 1) bins; the AnyWorkspace protocol
    mutable AnyWorkspace<T> w;
    mutable std::mutex host_mu;        // held for a whole *_host call (lock order: host_mu, then w.mu, then the inner plan's)
    mutable T* stage = nullptr;        // host-API staging: N reals, transformed in place; allocated by the first host call
    std::string description;
    size_t vstride() const { return n + (n & 1); }                 // even, so the inner r2c may read v as pairs
    size_t member_elems() const { return vstride() / 2 + n / 2 + 1; }   // complex values
    cudaStream_t host_stream() const { return inner->pow2 ? inner->pow2->inner->stream : inner->host_stream(); }
    ~PlanDct() {
        DeviceGuard g(device);
        w.destroy();
        if (w4n.blob) cudaFree(w4n.blob);
        if (stage) cudaFree(stage);
        delete inner;
    }
};

template <typename T>
int32_t build_plan_dct(size_t n, int device, int algo, PlanDct<T>** out) {
    if (!out) return fail(PHASTFT_ERR_INVALID_ARG, "out == NULL");
    *out = nullptr;
    if (n == 0) return fail(PHASTFT_ERR_INVALID_ARG, "n must be >= 1");
    std::unique_ptr<PlanDct<T>> pl(new PlanDct<T>());
    pl->n = n; pl->device = device;
    if (int32_t st = build_plan_r2c_any<T>(n, device, algo, &pl->inner)) return st;
    DeviceGuard g(device);
    if (int32_t st = build_two_level(pl->w4n, 4 * n, n / 2 + 1)) return st;
    if (int32_t st = pl->w.init(pl->member_elems())) return st;   // room for one member; batched calls grow it
    pl->description = "n=" + std::to_string(n) + (sizeof(T) == 8 ? " f64" : " f32") + " dct | ";
    *out = pl.release();
    return PHASTFT_OK;
}

template <typename T>
std::string dct_description(const PlanDct<T>* pl) { return pl->description + r2c_any_description(pl->inner); }

template <typename T>
int32_t dct_reserve(const PlanDct<T>* pl, size_t batch) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (int32_t st = r2c_any_reserve(pl->inner, batch)) return st;
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> lock(pl->w.mu);
    return pl->w.grow(batch * pl->member_elems(), batch);
}

// One DCT-PRE or DCT-POST over `batch` members, in launches of at most 2^31 - 1 blocks.  Launch record: R = N, C = the members
// of that launch.
template <typename T>
int32_t launch_dct_end(bool post, int kind, DctParams<T> p, size_t threads, size_t batch, cudaStream_t stream) {
    static const char* const names[2][4] = {{"DCT-PRE-DCT2", "DCT-PRE-DCT3", "DCT-PRE-DST2", "DCT-PRE-DST3"},
                                             {"DCT-POST-DCT2", "DCT-POST-DCT3", "DCT-POST-DST2", "DCT-POST-DST3"}};
    const size_t bpm = (threads + 255) / 256;
    p.blocks_per_member = (unsigned)bpm;
    const size_t max_members = std::max<size_t>(1, grid_blocks_max() / bpm);
    for (size_t done = 0; done < batch; done += max_members) {
        const size_t nb = std::min(batch - done, max_members);
        DctParams<T> q = p;
        q.in += done * p.in_stride;
        q.out += done * p.out_stride;
        q.bins += done * p.bin_stride;
        launch_dct<T>(post, kind, q, (unsigned)(nb * bpm), stream);
        CUDA_TRY(cudaGetLastError());
        note_launch({names[post][kind], (int)std::min<size_t>(p.n, INT32_MAX), 0, (int)nb, 256, 0, "plain", false});
    }
    return PHASTFT_OK;
}

// Member b reads N reals at d_in + b * in_stride and writes N reals at d_out + b * out_stride (any strides >= N, any element
// offsets, d_out == d_in with equal strides in place).  kind PHASTFT_R2R_*, norm PHASTFT_NORM_* with scipy.fft's meanings.
template <typename T>
int32_t dct_dev(const PlanDct<T>* pl, int kind, int norm, const T* d_in, size_t in_stride, T* d_out, size_t out_stride, size_t batch,
                cudaStream_t stream) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (kind < PHASTFT_R2R_DCT2 || kind > PHASTFT_R2R_DST3)
        return fail(PHASTFT_ERR_INVALID_ARG, "kind must be PHASTFT_R2R_DCT2, _DCT3, _DST2 or _DST3");
    if (norm < PHASTFT_NORM_BACKWARD || norm > PHASTFT_NORM_FORWARD)
        return fail(PHASTFT_ERR_INVALID_ARG, "norm must be PHASTFT_NORM_BACKWARD, _ORTHO or _FORWARD");
    if (!d_in) return fail(PHASTFT_ERR_INVALID_ARG, "d_in == NULL");
    if (!d_out) return fail(PHASTFT_ERR_INVALID_ARG, "d_out == NULL");
    const size_t n = pl->n, bins = n / 2 + 1, vs = pl->vstride();
    if (in_stride < n) return fail(PHASTFT_ERR_INVALID_ARG, "in_stride must be >= N = " + std::to_string(n) + " (got " + std::to_string(in_stride) + ")");
    if (out_stride < n) return fail(PHASTFT_ERR_INVALID_ARG, "out_stride must be >= N = " + std::to_string(n) + " (got " + std::to_string(out_stride) + ")");
    if (batch == 0) return PHASTFT_OK;
    const bool type2 = kind == PHASTFT_R2R_DCT2 || kind == PHASTFT_R2R_DST2;
    // scipy's norms: type 2 y = 2 c sum(...), type 3 y = c (x[0] + 2 sum(...)), c = 1, 1/sqrt(2N) or 1/(2N); ortho also scales
    // output 0 of type 2 by 1/sqrt(2) and input 0 of type 3 by sqrt(2) (element N-1 for DST).  Type 3 also undoes the c2r's 1/N.
    const long double c = norm == PHASTFT_NORM_BACKWARD ? 1.0L : norm == PHASTFT_NORM_ORTHO ? 1.0L / sqrtl(2.0L * n) : 1.0L / (2.0L * n);
    const long double s = type2 ? 2.0L * c : (long double)n * c;
    const long double s0 = norm != PHASTFT_NORM_ORTHO ? s : type2 ? s / sqrtl(2.0L) : s * sqrtl(2.0L);
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> lock(pl->w.mu);
    bool capturing = false;
    if (int32_t st = pl->w.acquire(batch * pl->member_elems(), batch, stream, "phastft_plan_dct_*_reserve", capturing)) return st;
    T* v = reinterpret_cast<T*>(pl->w.ws);
    cx<T>* spec = pl->w.ws + batch * vs / 2;
    DctParams<T> p;
    memset(&p, 0, sizeof(p));
    p.bins = spec; p.bin_stride = (long long)bins;
    p.w_hi = pl->w4n.hi; p.w_lo = pl->w4n.lo; p.lo_bits = pl->w4n.lo_bits;
    p.n = (long long)n; p.scale = (T)s; p.scale0 = (T)s0;
    // type 2: x -> v (pairs), r2c, bins -> y (bins); type 3: x -> bins (bins), c2r, v -> y (pairs)
    DctParams<T> pre = p, post = p;
    pre.in = d_in; pre.in_stride = (long long)in_stride;
    post.out = d_out; post.out_stride = (long long)out_stride;
    if (type2) { pre.out = v; pre.out_stride = (long long)vs; }
    else { post.in = v; post.in_stride = (long long)vs; }
    const size_t pairs = (n + 1) / 2;
    int32_t st = launch_dct_end<T>(false, kind, pre, type2 ? pairs : bins, batch, stream);
    if (!st) st = type2 ? r2c_il_any_dev(pl->inner, v, vs, reinterpret_cast<T*>(spec), bins, batch, stream)
                        : c2r_il_any_dev(pl->inner, reinterpret_cast<const T*>(spec), bins, v, vs, batch, stream);
    if (!st) st = launch_dct_end<T>(true, kind, post, type2 ? bins : pairs, batch, stream);
    const int32_t rel = pl->w.release(stream, capturing);   // also after a failed launch: the kernels queued so far used it
    return st ? st : rel;
}

// host slices, synchronous: the N reals are staged through one plan-owned buffer and transformed in place there
template <typename T>
int32_t dct_host(const PlanDct<T>* pl, int kind, int norm, const T* in, size_t len_in, T* out, size_t len_out) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (kind < PHASTFT_R2R_DCT2 || kind > PHASTFT_R2R_DST3)
        return fail(PHASTFT_ERR_INVALID_ARG, "kind must be PHASTFT_R2R_DCT2, _DCT3, _DST2 or _DST3");
    if (norm < PHASTFT_NORM_BACKWARD || norm > PHASTFT_NORM_FORWARD)
        return fail(PHASTFT_ERR_INVALID_ARG, "norm must be PHASTFT_NORM_BACKWARD, _ORTHO or _FORWARD");
    const size_t n = pl->n;
    if (len_in != n) return fail(PHASTFT_ERR_INPUT_LEN);
    if (len_out != n) return fail(PHASTFT_ERR_OUTPUT_LEN);
    if (!in || !out) return fail(PHASTFT_ERR_INVALID_ARG, "NULL slice");
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> host_lock(pl->host_mu);
    cudaStream_t s = pl->host_stream();
    {
        std::lock_guard<std::mutex> lock(pl->w.mu);   // released before the device call, which takes it
        if (!pl->stage) CUDA_TRY(cudaMalloc(&pl->stage, n * sizeof(T)));
    }
    CUDA_TRY(scribble(pl->w.scribble_on, pl->stage, n * sizeof(T), s));
    CUDA_TRY(cudaMemcpyAsync(pl->stage, in, n * sizeof(T), cudaMemcpyHostToDevice, s));
    if (int32_t st = dct_dev(pl, kind, norm, pl->stage, n, pl->stage, n, 1, s)) return st;
    CUDA_TRY(cudaMemcpyAsync(out, pl->stage, n * sizeof(T), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return PHASTFT_OK;
}

// =================================================================================================
// linear convolution and correlation of real or complex signals of any lengths: CONV-PRE, the L-point real plan's interleaved
// r2c (or the complex plan's forward transform) on x and h together, CONV-MUL, the c2r (or reverse transform) on x, CONV-POST
// (fft_kernels.cuh).  L = 2^ceil(log2(n_x + n_h - 1)), at least 4, so the circular convolution at L is the linear one.
// =================================================================================================
// The window of the full convolution (n_x + n_h - 1 values) that each PHASTFT_CONV_* mode returns, scipy.signal's; length 0
// for a bad mode or an empty operand.
size_t conv_out_len(size_t n_x, size_t n_h, int mode) {
    if (n_x == 0 || n_h == 0) return 0;
    switch (mode) {
        case PHASTFT_CONV_FULL: return n_x + n_h - 1;
        case PHASTFT_CONV_SAME: return n_x;
        case PHASTFT_CONV_VALID: return std::max(n_x, n_h) - std::min(n_x, n_h) + 1;
        default: return 0;
    }
}
size_t conv_start(size_t n_x, size_t n_h, int mode) {
    return mode == PHASTFT_CONV_SAME ? (n_h - 1) / 2 : mode == PHASTFT_CONV_VALID ? std::min(n_x, n_h) - 1 : 0;
}

template <typename T>
struct PlanConv {
    size_t n_x = 0, n_h = 0, L = 0;
    int device = 0;
    bool cplx = false;
    PlanR2cAny<T>* real = nullptr;     // real signals: the L-point real plan (its power-of-two r2c plan)
    PlanAny<T>* cinner = nullptr;      // complex signals: the L-point complex plan
    // per call of C = B + H members (B signals, H = B filters or one broadcast): real, C x L reals then C x (L/2 + 1) bins;
    // complex, C x L values transformed in place.  The AnyWorkspace protocol.
    mutable AnyWorkspace<T> w;
    mutable std::mutex host_mu;        // held for a whole *_host call (lock order: host_mu, then w.mu, then the inner plan's)
    mutable T* stage = nullptr;        // host-API staging: x, h and y back to back; allocated by the first host call
    std::string description;
    size_t member_elems() const { return cplx ? L : L + 1; }        // complex values
    size_t stage_elems() const { return n_x + n_h + conv_out_len(n_x, n_h, PHASTFT_CONV_FULL); }   // values (T or complex)
    cudaStream_t host_stream() const { return cplx ? cinner->pow2->stream : real->pow2->inner->stream; }
    ~PlanConv() {
        DeviceGuard g(device);
        w.destroy();
        if (stage) cudaFree(stage);
        delete real;
        delete cinner;
    }
};

template <typename T>
int32_t build_plan_conv(size_t n_x, size_t n_h, int domain, int device, PlanConv<T>** out) {
    if (!out) return fail(PHASTFT_ERR_INVALID_ARG, "out == NULL");
    *out = nullptr;
    if (n_x == 0 || n_h == 0) return fail(PHASTFT_ERR_INVALID_ARG, "n_x and n_h must be >= 1");
    if (domain != PHASTFT_CONV_REAL && domain != PHASTFT_CONV_COMPLEX)
        return fail(PHASTFT_ERR_INVALID_ARG, "domain must be PHASTFT_CONV_REAL or PHASTFT_CONV_COMPLEX");
    const bool cplx = domain == PHASTFT_CONV_COMPLEX;
    const int lmax = cplx ? 30 : 31;       // the largest complex plan, the largest real one
    const size_t top = size_t(1) << lmax;
    if (n_x > top || n_h > top || n_x + n_h - 1 > top)
        return fail(PHASTFT_ERR_INVALID_ARG, "n_x + n_h - 1 = " + std::to_string(n_x + n_h - 1) + " is above 2^" + std::to_string(lmax) +
                                             " (the largest " + (cplx ? "complex" : "real") + " transform length L)");
    int ll = 2;
    while ((size_t(1) << ll) < n_x + n_h - 1) ++ll;
    std::unique_ptr<PlanConv<T>> pl(new PlanConv<T>());
    pl->n_x = n_x; pl->n_h = n_h; pl->L = size_t(1) << ll; pl->device = device; pl->cplx = cplx;
    if (int32_t st = cplx ? build_plan_any<T>(pl->L, device, PHASTFT_ANY_AUTO, &pl->cinner)
                          : build_plan_r2c_any<T>(pl->L, device, PHASTFT_ANY_AUTO, &pl->real))
        return st;
    DeviceGuard g(device);
    if (int32_t st = pl->w.init(2 * pl->member_elems())) return st;   // room for one lone call; batched calls grow it
    pl->description = "n_x=" + std::to_string(n_x) + " n_h=" + std::to_string(n_h) + (sizeof(T) == 8 ? " f64" : " f32") + " conv " +
                      (cplx ? "complex" : "real") + " L=2^" + std::to_string(ll) + " | ";
    *out = pl.release();
    return PHASTFT_OK;
}

template <typename T>
std::string conv_description(const PlanConv<T>* pl) {
    return pl->description + (pl->cplx ? pl->cinner->description : r2c_any_description(pl->real));
}

// Every allocation a call of `batch` pairwise members would make: the inner plan's for the forward call of 2 x batch members
// and the inverse of batch, and the workspace.
template <typename T>
int32_t conv_reserve(const PlanConv<T>* pl, size_t batch) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    for (size_t b : {2 * batch, batch})
        if (int32_t st = pl->cplx ? any_reserve(pl->cinner, b) : r2c_any_reserve(pl->real, b)) return st;
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> lock(pl->w.mu);
    return pl->w.grow(2 * batch * pl->member_elems(), 2 * batch);
}

// One CONV-PRE, CONV-MUL or CONV-POST over `members` members from member 0, `threads` threads each, in launches of at most
// 2^31 - 1 blocks.  Launch record: R = L, C = the members of that launch.
template <typename T>
int32_t launch_conv_stage(int stage, bool cplx, bool corr, ConvParams<T> p, size_t threads, size_t members, cudaStream_t stream) {
    static const char* const names[3] = {"CONV-PRE", "CONV-MUL", "CONV-POST"};
    const size_t bpm = (threads + 255) / 256;
    p.blocks_per_member = (unsigned)bpm;
    const size_t max_members = std::max<size_t>(1, grid_blocks_max() / bpm);
    for (size_t done = 0; done < members; done += max_members) {
        const size_t nb = std::min(members - done, max_members);
        p.m0 = (long long)done;
        launch_conv<T>(stage, cplx, corr, p, (unsigned)(nb * bpm), stream);
        CUDA_TRY(cudaGetLastError());
        note_launch({names[stage], (int)std::min<long long>(p.L, INT32_MAX), 0, (int)nb, 256, 0, "plain", false});
    }
    return PHASTFT_OK;
}

// Member b convolves (op PHASTFT_CONV_CONVOLVE) or correlates the n_x values at d_x + b * x_stride with the n_h values at
// d_h + b * h_stride (h_stride 0: one filter for every member) and writes the mode's window at d_y + b * y_stride.  Values are
// reals, or complex (re, im) pairs with strides in complex values and pointers aligned to 2 * sizeof(T).  Any element offsets;
// d_y may be d_x or d_h (CONV-PRE reads every input before CONV-POST writes).
template <typename T>
int32_t conv_dev(const PlanConv<T>* pl, int op, int mode, const T* d_x, size_t x_stride, const T* d_h, size_t h_stride, T* d_y,
                 size_t y_stride, size_t batch, cudaStream_t stream) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (op != PHASTFT_CONV_CONVOLVE && op != PHASTFT_CONV_CORRELATE)
        return fail(PHASTFT_ERR_INVALID_ARG, "op must be PHASTFT_CONV_CONVOLVE or PHASTFT_CONV_CORRELATE");
    if (mode != PHASTFT_CONV_FULL && mode != PHASTFT_CONV_SAME && mode != PHASTFT_CONV_VALID)
        return fail(PHASTFT_ERR_INVALID_ARG, "mode must be PHASTFT_CONV_FULL, _SAME or _VALID");
    if (!d_x) return fail(PHASTFT_ERR_INVALID_ARG, "d_x == NULL");
    if (!d_h) return fail(PHASTFT_ERR_INVALID_ARG, "d_h == NULL");
    if (!d_y) return fail(PHASTFT_ERR_INVALID_ARG, "d_y == NULL");
    const size_t n_x = pl->n_x, n_h = pl->n_h, L = pl->L, out_len = conv_out_len(n_x, n_h, mode);
    if (batch > 1) {
        if (x_stride < n_x) return fail(PHASTFT_ERR_INVALID_ARG, "x_stride must be >= n_x = " + std::to_string(n_x) + " (got " + std::to_string(x_stride) + ")");
        if (h_stride != 0 && h_stride < n_h)
            return fail(PHASTFT_ERR_INVALID_ARG, "h_stride must be 0 (one filter) or >= n_h = " + std::to_string(n_h) + " (got " + std::to_string(h_stride) + ")");
        if (y_stride < out_len)
            return fail(PHASTFT_ERR_INVALID_ARG, "y_stride must be >= the output length " + std::to_string(out_len) + " (got " + std::to_string(y_stride) + ")");
    }
    if (pl->cplx) {
        if (int32_t st = check_pair_alignment(d_x, "d_x")) return st;
        if (int32_t st = check_pair_alignment(d_h, "d_h")) return st;
        if (int32_t st = check_pair_alignment(d_y, "d_y")) return st;
    }
    if (batch == 0) return PHASTFT_OK;
    const size_t nh_members = batch == 1 || h_stride == 0 ? 1 : batch, members = batch + nh_members;
    const size_t bins = pl->cplx ? L : L / 2 + 1;
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> lock(pl->w.mu);
    bool capturing = false;
    if (int32_t st = pl->w.acquire(members * pl->member_elems(), members, stream, "phastft_plan_conv_*_reserve", capturing)) return st;
    T* sig = reinterpret_cast<T*>(pl->w.ws);
    cx<T>* spec = pl->cplx ? pl->w.ws : pl->w.ws + members * L / 2;
    ConvParams<T> p;
    memset(&p, 0, sizeof(p));
    p.x = d_x; p.h = d_h; p.y = d_y; p.sig = sig; p.spec = spec;
    p.n_x = (long long)n_x; p.n_h = (long long)n_h; p.L = (long long)L;
    p.x_stride = (long long)x_stride; p.h_stride = (long long)h_stride; p.y_stride = (long long)y_stride;
    p.n_xm = (long long)batch;
    p.start = (long long)conv_start(n_x, n_h, mode); p.out_len = (long long)out_len;
    p.spec_stride = (long long)bins; p.bins = (long long)bins;
    p.h_bcast = nh_members == 1;
    const bool cplx = pl->cplx, corr = op == PHASTFT_CONV_CORRELATE;
    int32_t st = launch_conv_stage<T>(CONV_STAGE_PRE, cplx, corr, p, L, members, stream);
    if (!st) st = cplx ? any_interleaved_dev(pl->cinner, sig, PHASTFT_FORWARD, members, L, stream)
                       : r2c_il_any_dev(pl->real, sig, L, reinterpret_cast<T*>(spec), bins, members, stream);
    if (!st) st = launch_conv_stage<T>(CONV_STAGE_MUL, cplx, corr, p, bins, batch, stream);
    if (!st) st = cplx ? any_interleaved_dev(pl->cinner, sig, PHASTFT_REVERSE, batch, L, stream)
                       : c2r_il_any_dev(pl->real, reinterpret_cast<const T*>(spec), bins, sig, L, batch, stream);
    if (!st) st = launch_conv_stage<T>(CONV_STAGE_POST, cplx, corr, p, out_len, batch, stream);
    const int32_t rel = pl->w.release(stream, capturing);   // also after a failed launch: the kernels queued so far used it
    return st ? st : rel;
}

// host slices, synchronous: x, h and y staged through one plan-owned buffer.  Lengths in values (complex ones for complex
// signals): len_x != n_x or len_h != n_h is PHASTFT_ERR_INPUT_LEN, len_y != the mode's output length PHASTFT_ERR_OUTPUT_LEN.
template <typename T>
int32_t conv_host(const PlanConv<T>* pl, int op, int mode, const T* x, size_t len_x, const T* h, size_t len_h, T* y, size_t len_y) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    if (op != PHASTFT_CONV_CONVOLVE && op != PHASTFT_CONV_CORRELATE)
        return fail(PHASTFT_ERR_INVALID_ARG, "op must be PHASTFT_CONV_CONVOLVE or PHASTFT_CONV_CORRELATE");
    if (mode != PHASTFT_CONV_FULL && mode != PHASTFT_CONV_SAME && mode != PHASTFT_CONV_VALID)
        return fail(PHASTFT_ERR_INVALID_ARG, "mode must be PHASTFT_CONV_FULL, _SAME or _VALID");
    const size_t n_x = pl->n_x, n_h = pl->n_h, out_len = conv_out_len(n_x, n_h, mode);
    if (len_x != n_x) return fail(PHASTFT_ERR_INPUT_LEN, "len_x " + std::to_string(len_x) + ", plan n_x = " + std::to_string(n_x));
    if (len_h != n_h) return fail(PHASTFT_ERR_INPUT_LEN, "len_h " + std::to_string(len_h) + ", plan n_h = " + std::to_string(n_h));
    if (len_y != out_len) return fail(PHASTFT_ERR_OUTPUT_LEN, "len_y " + std::to_string(len_y) + ", output length " + std::to_string(out_len));
    if (!x || !h || !y) return fail(PHASTFT_ERR_INVALID_ARG, "NULL slice");
    const size_t v = pl->cplx ? 2 : 1;        // T per value
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> host_lock(pl->host_mu);
    cudaStream_t s = pl->host_stream();
    {
        std::lock_guard<std::mutex> lock(pl->w.mu);   // released before the device call, which takes it
        if (!pl->stage) CUDA_TRY(cudaMalloc(&pl->stage, pl->stage_elems() * v * sizeof(T)));
    }
    T* sx = pl->stage;
    T* sh = sx + n_x * v;
    T* sy = sh + n_h * v;
    CUDA_TRY(scribble(pl->w.scribble_on, pl->stage, pl->stage_elems() * v * sizeof(T), s));
    CUDA_TRY(cudaMemcpyAsync(sx, x, n_x * v * sizeof(T), cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(sh, h, n_h * v * sizeof(T), cudaMemcpyHostToDevice, s));
    if (int32_t st = conv_dev(pl, op, mode, sx, n_x, sh, n_h, sy, out_len, 1, s)) return st;
    CUDA_TRY(cudaMemcpyAsync(y, sy, out_len * v * sizeof(T), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return PHASTFT_OK;
}

// =================================================================================================
// short-time Fourier transform and its inverse of real or complex signals (torch.stft(..., return_complex=True) /
// torch.istft(..., length=n)): STFT-FRAME and the n_fft-point real plan's interleaved r2c (or the complex plan's forward
// transform) over every frame of the batch; the c2r (or reverse transform) into workspace frames and ISTFT-OLA
// (fft_kernels.cuh).  Frame f of member b is global frame b * F + f, frame_stride complex values apart in the caller's spectrum.
// =================================================================================================
template <typename T>
struct PlanStft {
    size_t n = 0, n_fft = 0, hop = 0, pad = 0, frames = 0, bins = 0;   // frames: F per member
    int device = 0;
    bool cplx = false, reflect = true;
    PlanR2cAny<T>* real = nullptr;     // real signals: the n_fft-point real plan
    PlanAny<T>* cinner = nullptr;      // complex signals: the n_fft-point complex plan
    T* win = nullptr;                  // 2 x n_fft: the window zero-padded to n_fft, then the same times n_fft^(-1/2)
    long long nola_fail = -1;          // the first retained sample whose overlap-add envelope is below 1e-11, or -1
    long double nola_env = 0;          // its envelope
    // per call of B members: B x F frames of fstride() reals (real) or n_fft complex values (complex; istft only).  The
    // AnyWorkspace protocol.
    mutable AnyWorkspace<T> w;
    mutable std::mutex host_mu;        // held for a whole *_host call (lock order: host_mu, then w.mu, then the inner plan's)
    mutable T* stage = nullptr;        // host-API staging: F x bins complex values, then n signal values; allocated by the first host call
    std::string description;
    size_t fstride() const { return cplx ? n_fft : n_fft + (n_fft & 1); }   // workspace frame stride in values: even for reals,
    size_t member_elems() const { return cplx ? n_fft : fstride() / 2; }     // so the inner r2c / c2r may access them as pairs
    size_t vals() const { return cplx ? 2 : 1; }                             // T per signal value
    size_t stage_elems() const { return 2 * frames * bins + vals() * n; }    // T
    cudaStream_t host_stream() const {
        if (cplx) return cinner->pow2 ? cinner->pow2->stream : cinner->host_stream();
        return real->pow2 ? real->pow2->inner->stream : real->host_stream();
    }
    ~PlanStft() {
        DeviceGuard g(device);
        w.destroy();
        for (void* p : {(void*)win, (void*)stage})
            if (p) cudaFree(p);
        delete real;
        delete cinner;
    }
};

// torch.istft's NOLA check in long double: the envelope env(u) = sum_f wl[u - f * hop]^2 over the frames 0 <= f < F covering
// the padded sample u must reach 1e-11 wherever a retained sample (u in [pad, pad + n)) is covered (u < n_fft + hop (F - 1)).
// Between the head (u < n_fft - 1, where frame 0 clips the sum) and the tail (u >= F hop, where frame F - 1 does), env is
// periodic in hop, so the first n_fft + hop and the last n_fft + hop retained samples hold every value it takes; scanned in
// ascending u, the first failure found is the first there is.  Sets nola_fail to that sample (t = u - pad) or -1.
template <typename T>
void stft_nola(PlanStft<T>* pl, const std::vector<long double>& wl) {
    const size_t n_fft = pl->n_fft, hop = pl->hop, F = pl->frames;
    auto env = [&](size_t u) {
        const size_t f_hi = std::min(u / hop, F - 1), f_lo = u >= n_fft ? (u - n_fft) / hop + 1 : 0;
        long double s = 0;
        for (size_t f = f_lo; f <= f_hi; ++f) s += wl[u - f * hop] * wl[u - f * hop];
        return s;
    };
    const size_t lo = pl->pad, hi = std::min(pl->pad + pl->n, n_fft + hop * (F - 1)), span = n_fft + hop;
    const size_t head_end = std::min(hi, lo + span), tail_lo = std::max(head_end, hi > span ? hi - span : 0);
    for (size_t r = 0; r < 2; ++r)
        for (size_t u = r ? tail_lo : lo; u < (r ? hi : head_end); ++u) {
            const long double e = env(u);
            if (e < 1e-11L) { pl->nola_fail = (long long)(u - lo); pl->nola_env = e; return; }
        }
    pl->nola_fail = -1;
}

template <typename T>
int32_t build_plan_stft(size_t n, size_t n_fft, size_t hop, const T* window, size_t win_length, int center, int pad_mode, int domain,
                        int device, PlanStft<T>** out) {
    if (!out) return fail(PHASTFT_ERR_INVALID_ARG, "out == NULL");
    *out = nullptr;
    if (n == 0) return fail(PHASTFT_ERR_INVALID_ARG, "n must be >= 1");
    if (n_fft == 0) return fail(PHASTFT_ERR_INVALID_ARG, "n_fft must be >= 1");
    if (hop == 0) return fail(PHASTFT_ERR_INVALID_ARG, "hop must be >= 1");
    if (win_length == 0 || win_length > n_fft)
        return fail(PHASTFT_ERR_INVALID_ARG, "win_length must be in [1, n_fft = " + std::to_string(n_fft) + "] (got " + std::to_string(win_length) + ")");
    if (pad_mode != PHASTFT_STFT_PAD_REFLECT && pad_mode != PHASTFT_STFT_PAD_CONSTANT)
        return fail(PHASTFT_ERR_INVALID_ARG, "pad_mode must be PHASTFT_STFT_PAD_REFLECT or PHASTFT_STFT_PAD_CONSTANT");
    if (domain != PHASTFT_STFT_REAL && domain != PHASTFT_STFT_COMPLEX)
        return fail(PHASTFT_ERR_INVALID_ARG, "domain must be PHASTFT_STFT_REAL or PHASTFT_STFT_COMPLEX");
    const size_t pad = center ? n_fft / 2 : 0;
    if (center && pad_mode == PHASTFT_STFT_PAD_REFLECT && pad >= n)
        return fail(PHASTFT_ERR_INVALID_ARG, "reflect padding of n_fft / 2 = " + std::to_string(pad) + " needs n > " + std::to_string(pad) +
                                             " (got n = " + std::to_string(n) + ")");
    if (!center && n < n_fft)
        return fail(PHASTFT_ERR_INVALID_ARG, "without centering n must be >= n_fft = " + std::to_string(n_fft) + " (got n = " + std::to_string(n) + ")");
    const bool cplx = domain == PHASTFT_STFT_COMPLEX;
    std::unique_ptr<PlanStft<T>> pl(new PlanStft<T>());
    pl->n = n; pl->n_fft = n_fft; pl->hop = hop; pl->pad = pad; pl->device = device; pl->cplx = cplx;
    pl->reflect = center && pad_mode == PHASTFT_STFT_PAD_REFLECT;
    pl->frames = 1 + (n + 2 * pad - n_fft) / hop;
    pl->bins = cplx ? n_fft : n_fft / 2 + 1;
    if (int32_t st = cplx ? build_plan_any<T>(n_fft, device, PHASTFT_ANY_AUTO, &pl->cinner)
                          : build_plan_r2c_any<T>(n_fft, device, PHASTFT_ANY_AUTO, &pl->real))
        return st;
    // torch's window: win_length values (ones when NULL) centred in n_fft, left offset (n_fft - win_length) / 2
    std::vector<long double> wl(n_fft, 0.0L);
    const size_t left = (n_fft - win_length) / 2;
    for (size_t i = 0; i < win_length; ++i) wl[left + i] = window ? (long double)window[i] : 1.0L;
    std::vector<T> wt(2 * n_fft);
    const long double norm = 1.0L / sqrtl((long double)n_fft);
    for (size_t i = 0; i < n_fft; ++i) { wt[i] = (T)wl[i]; wt[n_fft + i] = (T)(wl[i] * norm); }
    stft_nola(pl.get(), wl);
    DeviceGuard g(device);
    CUDA_TRY(cudaMalloc(&pl->win, 2 * n_fft * sizeof(T)));
    CUDA_TRY(cudaMemcpy(pl->win, wt.data(), 2 * n_fft * sizeof(T), cudaMemcpyHostToDevice));
    if (int32_t st = pl->w.init(pl->frames * pl->member_elems())) return st;   // room for one member; batched calls grow it
    pl->description = "n=" + std::to_string(n) + " n_fft=" + std::to_string(n_fft) + " hop=" + std::to_string(hop) +
                      (sizeof(T) == 8 ? " f64" : " f32") + " stft " + (cplx ? "complex" : "real") + " F=" + std::to_string(pl->frames) + " | ";
    *out = pl.release();
    return PHASTFT_OK;
}

template <typename T>
std::string stft_description(const PlanStft<T>* pl) {
    return pl->description + (pl->cplx ? pl->cinner->description : r2c_any_description(pl->real));
}

// Every allocation a call of `batch` members would make: the inner plan's for batch x F frames, and the workspace.
template <typename T>
int32_t stft_reserve(const PlanStft<T>* pl, size_t batch) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    const size_t frames = batch * pl->frames;
    if (int32_t st = pl->cplx ? any_reserve(pl->cinner, frames) : r2c_any_reserve(pl->real, frames)) return st;
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> lock(pl->w.mu);
    return pl->w.grow(frames * pl->member_elems(), batch);
}

// One STFT-FRAME (over frames) or ISTFT-OLA (over members), `threads` threads per member, from member 0, in launches of at most
// 2^31 - 1 blocks.  Launch record: R = n_fft, C = the members of that launch.
template <typename T>
int32_t launch_stft_stage(bool ola, bool cplx, bool even_fix, StftParams<T> p, size_t threads, size_t members, cudaStream_t stream) {
    const size_t bpm = (threads + 255) / 256;
    p.blocks_per_member = (unsigned)bpm;
    const size_t max_members = std::max<size_t>(1, grid_blocks_max() / bpm);
    for (size_t done = 0; done < members; done += max_members) {
        const size_t nb = std::min(members - done, max_members);
        p.m0 = (long long)done;
        launch_stft<T>(ola, cplx, even_fix, p, (unsigned)(nb * bpm), stream);
        CUDA_TRY(cudaGetLastError());
        note_launch({ola ? "ISTFT-OLA" : "STFT-FRAME", (int)std::min<long long>(p.n_fft, INT32_MAX), 0, (int)nb, 256, 0, "plain", false});
    }
    return PHASTFT_OK;
}

// The arguments both directions share: `sig` the caller's signals (member b at sig + b * sig_stride values, n of them), `spec`
// the caller's spectra (frame b * F + f at spec + (b * F + f) * frame_stride complex values, bins of them).
template <typename T>
int32_t stft_check(const PlanStft<T>* pl, int normalized, const T* sig, size_t sig_stride, const T* spec, size_t frame_stride,
                   size_t batch, bool inverse) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    const char* sname = inverse ? "d_y" : "d_x";
    if (normalized != 0 && normalized != 1) return fail(PHASTFT_ERR_INVALID_ARG, "normalized must be 0 or 1");
    if (!sig) return fail(PHASTFT_ERR_INVALID_ARG, std::string(sname) + " == NULL");
    if (!spec) return fail(PHASTFT_ERR_INVALID_ARG, "d_spec == NULL");
    const size_t n = pl->n, bins = pl->bins, F = pl->frames, v = pl->vals();
    if (frame_stride < bins)
        return fail(PHASTFT_ERR_INVALID_ARG, "frame_stride must be >= the bin count " + std::to_string(bins) + " (got " + std::to_string(frame_stride) + ")");
    if (batch > 1 && sig_stride < n)
        return fail(PHASTFT_ERR_INVALID_ARG, std::string(inverse ? "y_stride" : "x_stride") + " must be >= n = " + std::to_string(n) +
                                             " (got " + std::to_string(sig_stride) + ")");
    if (int32_t st = check_pair_alignment(spec, "d_spec")) return st;
    if (pl->cplx)
        if (int32_t st = check_pair_alignment(sig, sname)) return st;
    if (batch == 0) return PHASTFT_OK;
    const uintptr_t s0 = reinterpret_cast<uintptr_t>(sig), s1 = s0 + ((batch - 1) * sig_stride + n) * v * sizeof(T);
    const uintptr_t p0 = reinterpret_cast<uintptr_t>(spec), p1 = p0 + ((batch * F - 1) * frame_stride + bins) * 2 * sizeof(T);
    if (s0 < p1 && p0 < s1) return fail(PHASTFT_ERR_INVALID_ARG, std::string("d_spec's frames overlap ") + sname + "'s members");
    return PHASTFT_OK;
}

// Member b's n values at d_x + b * x_stride (reals, or complex pairs aligned to 2 * sizeof(T)) give F frames of bins bins at
// d_spec + (b * F + f) * frame_stride complex values; the values between frames are never written.
template <typename T>
int32_t stft_dev(const PlanStft<T>* pl, int normalized, const T* d_x, size_t x_stride, T* d_spec, size_t frame_stride, size_t batch,
                 cudaStream_t stream) {
    if (int32_t st = stft_check(pl, normalized, d_x, x_stride, d_spec, frame_stride, batch, false)) return st;
    if (batch == 0) return PHASTFT_OK;
    const size_t n_fft = pl->n_fft, frames = batch * pl->frames;
    DeviceGuard g(pl->device);
    StftParams<T> p;
    memset(&p, 0, sizeof(p));
    p.x = d_x; p.win = pl->win + (normalized ? n_fft : 0);
    p.n = (long long)pl->n; p.n_fft = (long long)n_fft; p.hop = (long long)pl->hop; p.pad = (long long)pl->pad;
    p.n_frames = (long long)pl->frames; p.x_stride = (long long)x_stride; p.reflect = pl->reflect;
    if (pl->cplx) {   // framed straight into the caller's slots and transformed in place there
        p.frames = d_spec; p.fstride = (long long)frame_stride;
        int32_t st = launch_stft_stage<T>(false, true, false, p, n_fft, frames, stream);
        if (!st) st = any_interleaved_dev(pl->cinner, d_spec, PHASTFT_FORWARD, frames, frame_stride, stream);
        return st;
    }
    std::lock_guard<std::mutex> lock(pl->w.mu);
    bool capturing = false;
    if (int32_t st = pl->w.acquire(frames * pl->member_elems(), batch, stream, "phastft_plan_stft_*_reserve", capturing)) return st;
    T* ws = reinterpret_cast<T*>(pl->w.ws);
    p.frames = ws; p.fstride = (long long)pl->fstride();
    int32_t st = launch_stft_stage<T>(false, false, false, p, n_fft, frames, stream);
    if (!st) st = r2c_il_any_dev(pl->real, ws, pl->fstride(), d_spec, frame_stride, frames, stream);
    const int32_t rel = pl->w.release(stream, capturing);   // also after a failed launch: the kernels queued so far used it
    return st ? st : rel;
}

// The inverse: member b's F frames at d_spec + (b * F + f) * frame_stride (never written) give n values at d_y + b * y_stride.
template <typename T>
int32_t istft_dev(const PlanStft<T>* pl, int normalized, const T* d_spec, size_t frame_stride, T* d_y, size_t y_stride, size_t batch,
                  cudaStream_t stream) {
    if (int32_t st = stft_check(pl, normalized, d_y, y_stride, d_spec, frame_stride, batch, true)) return st;
    if (pl->nola_fail >= 0) {
        char env[32];
        snprintf(env, sizeof(env), "%.3Lg", pl->nola_env);
        return fail(PHASTFT_ERR_INVALID_ARG, "the window's overlap-add envelope is " + std::string(env) + " < 1e-11 at sample " +
                                             std::to_string(pl->nola_fail) + " (the NOLA condition fails): the istft is not defined there");
    }
    if (batch == 0) return PHASTFT_OK;
    const size_t n_fft = pl->n_fft, frames = batch * pl->frames;
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> lock(pl->w.mu);
    bool capturing = false;
    if (int32_t st = pl->w.acquire(frames * pl->member_elems(), batch, stream, "phastft_plan_stft_*_reserve", capturing)) return st;
    T* ws = reinterpret_cast<T*>(pl->w.ws);
    int32_t st = PHASTFT_OK;
    if (pl->cplx) {
        const size_t row = n_fft * sizeof(cx<T>);
        if (cudaMemcpy2DAsync(ws, row, d_spec, frame_stride * sizeof(cx<T>), row, frames, cudaMemcpyDeviceToDevice, stream) != cudaSuccess) {
            (void)cudaGetLastError();
            st = fail(PHASTFT_ERR_CUDA, "cudaMemcpy2DAsync of the frames into the workspace failed");
        }
        if (!st) st = any_interleaved_dev(pl->cinner, ws, PHASTFT_REVERSE, frames, n_fft, stream);
    } else {
        st = c2r_il_any_dev(pl->real, d_spec, frame_stride, ws, pl->fstride(), frames, stream);
    }
    StftParams<T> p;
    memset(&p, 0, sizeof(p));
    p.frames = ws; p.fstride = (long long)pl->fstride();
    p.spec = reinterpret_cast<const cx<T>*>(d_spec); p.spec_stride = (long long)frame_stride;
    p.y = d_y; p.y_stride = (long long)y_stride; p.win = pl->win;
    p.n = (long long)pl->n; p.n_fft = (long long)n_fft; p.hop = (long long)pl->hop; p.pad = (long long)pl->pad;
    p.n_frames = (long long)pl->frames;
    p.scale = normalized ? (T)sqrtl((long double)n_fft) : T(1);
    p.inv_n = (T)(1.0L / (long double)n_fft);
    const bool even_fix = !pl->cplx && n_fft % 2 == 0;
    if (!st) st = launch_stft_stage<T>(true, pl->cplx, even_fix, p, pl->n, batch, stream);
    const int32_t rel = pl->w.release(stream, capturing);
    return st ? st : rel;
}

// host slices, synchronous, through one plan-owned buffer: the F x bins dense frames, then the n signal values.  Lengths in
// values (complex ones for complex signals and for the spectrum).
template <typename T>
int32_t stft_stage(const PlanStft<T>* pl, cudaStream_t s) {
    {
        std::lock_guard<std::mutex> lock(pl->w.mu);   // released before the device call, which takes it
        if (!pl->stage) CUDA_TRY(cudaMalloc(&pl->stage, pl->stage_elems() * sizeof(T)));
    }
    CUDA_TRY(scribble(pl->w.scribble_on, pl->stage, pl->stage_elems() * sizeof(T), s));
    return PHASTFT_OK;
}

template <typename T>
int32_t stft_host(const PlanStft<T>* pl, int normalized, const T* x, size_t len_x, T* spec, size_t len_spec) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    const size_t n = pl->n, cnt = pl->frames * pl->bins, v = pl->vals();
    if (len_x != n) return fail(PHASTFT_ERR_INPUT_LEN, "len_x " + std::to_string(len_x) + ", plan n = " + std::to_string(n));
    if (len_spec != cnt) return fail(PHASTFT_ERR_OUTPUT_LEN, "len_spec " + std::to_string(len_spec) + ", F x bins = " + std::to_string(cnt));
    if (!x || !spec) return fail(PHASTFT_ERR_INVALID_ARG, "NULL slice");
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> host_lock(pl->host_mu);
    cudaStream_t s = pl->host_stream();
    if (int32_t st = stft_stage(pl, s)) return st;
    T* sspec = pl->stage;
    T* sx = sspec + 2 * cnt;
    CUDA_TRY(cudaMemcpyAsync(sx, x, n * v * sizeof(T), cudaMemcpyHostToDevice, s));
    if (int32_t st = stft_dev(pl, normalized, sx, n, sspec, pl->bins, 1, s)) return st;
    CUDA_TRY(cudaMemcpyAsync(spec, sspec, 2 * cnt * sizeof(T), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return PHASTFT_OK;
}

template <typename T>
int32_t istft_host(const PlanStft<T>* pl, int normalized, const T* spec, size_t len_spec, T* y, size_t len_y) {
    if (!pl) return fail(PHASTFT_ERR_INVALID_ARG, "plan == NULL");
    const size_t n = pl->n, cnt = pl->frames * pl->bins, v = pl->vals();
    if (len_spec != cnt) return fail(PHASTFT_ERR_INPUT_LEN, "len_spec " + std::to_string(len_spec) + ", F x bins = " + std::to_string(cnt));
    if (len_y != n) return fail(PHASTFT_ERR_OUTPUT_LEN, "len_y " + std::to_string(len_y) + ", plan n = " + std::to_string(n));
    if (!spec || !y) return fail(PHASTFT_ERR_INVALID_ARG, "NULL slice");
    DeviceGuard g(pl->device);
    std::lock_guard<std::mutex> host_lock(pl->host_mu);
    cudaStream_t s = pl->host_stream();
    if (int32_t st = stft_stage(pl, s)) return st;
    T* sspec = pl->stage;
    T* sy = sspec + 2 * cnt;
    CUDA_TRY(cudaMemcpyAsync(sspec, spec, 2 * cnt * sizeof(T), cudaMemcpyHostToDevice, s));
    if (int32_t st = istft_dev(pl, normalized, sspec, pl->bins, sy, n, 1, s)) return st;
    CUDA_TRY(cudaMemcpyAsync(y, sy, n * v * sizeof(T), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return PHASTFT_OK;
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
#define AS_PLAN(T, p) reinterpret_cast<Plan<T>*>(p)
#define AS_CPLAN(T, p) reinterpret_cast<const Plan<T>*>(p)
#define AS_R2C(T, p) reinterpret_cast<PlanR2c<T>*>(p)
#define AS_CR2C(T, p) reinterpret_cast<const PlanR2c<T>*>(p)
#define AS_ANY(T, p) reinterpret_cast<PlanAny<T>*>(p)
#define AS_CANY(T, p) reinterpret_cast<const PlanAny<T>*>(p)
#define AS_R2CANY(T, p) reinterpret_cast<PlanR2cAny<T>*>(p)
#define AS_CR2CANY(T, p) reinterpret_cast<const PlanR2cAny<T>*>(p)
#define AS_DCT(T, p) reinterpret_cast<PlanDct<T>*>(p)
#define AS_CDCT(T, p) reinterpret_cast<const PlanDct<T>*>(p)
#define AS_CONV(T, p) reinterpret_cast<PlanConv<T>*>(p)
#define AS_CCONV(T, p) reinterpret_cast<const PlanConv<T>*>(p)
#define AS_STFT(T, p) reinterpret_cast<PlanStft<T>*>(p)
#define AS_CSTFT(T, p) reinterpret_cast<const PlanStft<T>*>(p)

extern "C" {

const char* phastft_last_error(void) { return g_last_error.c_str(); }
const char* phastft_version(void) { return "phastft_cuda 0.2.0 (sm_90a)"; }
int32_t phastft_host_register(void* host_ptr, size_t bytes) {
    if (!host_ptr || !bytes) return fail(PHASTFT_ERR_INVALID_ARG, "NULL or empty range");
    CUDA_TRY(cudaHostRegister(host_ptr, bytes, cudaHostRegisterPortable));
    return PHASTFT_OK;
}
int32_t phastft_host_unregister(void* host_ptr) {
    if (!host_ptr) return fail(PHASTFT_ERR_INVALID_ARG, "NULL pointer");
    CUDA_TRY(cudaHostUnregister(host_ptr));
    return PHASTFT_OK;
}
void phastft_oneshot_cache_clear(void) {
    oneshot_c2c_cache<double>().clear();
    oneshot_c2c_cache<float>().clear();
    oneshot_r2c_cache<double>().clear();
    oneshot_r2c_cache<float>().clear();
}

uint64_t phastft_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
uint64_t phastft_last_scribble_bytes(void) { return g_scribble_bytes; }
const char* phastft_last_launches(void) {
    std::string& s = g_launch_text;
    s.clear();
    for (const LaunchRec& r : g_launch_log) {
        if (!s.empty()) s += "; ";
        s += std::string(r.kind) + " R=" + std::to_string(r.R);
        if (r.R2) s += "x" + std::to_string(r.R2);
        s += (strcmp(r.kind, "CLUSTER") == 0 ? " K=" : " C=") + std::to_string(r.C) + " NT=" + std::to_string(r.NT) + " v" +
             std::to_string(r.variant) + " " + r.mode + (r.pdl ? " pdl" : "");
    }
    return s.c_str();
}
int32_t phastft_device_count(int* count) {
    if (!count) return fail(PHASTFT_ERR_INVALID_ARG, "count == NULL");
    *count = 0;
    cudaError_t e = cudaGetDeviceCount(count);
    if (e != cudaSuccess || *count == 0) { *count = 0; return fail(PHASTFT_ERR_NO_DEVICE, e != cudaSuccess ? cudaGetErrorString(e) : ""); }
    return PHASTFT_OK;
}

int32_t phastft_plan_factorization(size_t n, int precision_bits, int* log2_factors, int* num_passes) {
    if (!log2_factors || !num_passes) return fail(PHASTFT_ERR_INVALID_ARG, "NULL argument");
    if (!is_pow2(n)) return fail(PHASTFT_ERR_NOT_POW2);
    if (precision_bits != 32 && precision_bits != 64) return fail(PHASTFT_ERR_INVALID_ARG, "precision_bits must be 32 or 64");
    const int ln = ilog2(n);
    std::vector<int> f = ln == 0 ? std::vector<int>{} : (precision_bits == 64 ? choose_factors<double>(ln) : choose_factors<float>(ln));
    *num_passes = (int)f.size();
    for (size_t i = 0; i < f.size(); ++i) log2_factors[i] = f[i];
    return PHASTFT_OK;
}

int32_t phastft_any_mixed_factorization(size_t n, size_t* p, int* q_a, int* q_b) {
    if (!p || !q_a || !q_b) return fail(PHASTFT_ERR_INVALID_ARG, "NULL argument");
    MixedSplit s;
    std::string why;
    if (!mixed_split(n, s, why)) return fail(PHASTFT_ERR_INVALID_ARG, "no mixed-radix plan: " + why);
    *p = s.p; *q_a = s.qa; *q_b = s.qb;
    return PHASTFT_OK;
}

int32_t phastft_plan_tune_candidates(size_t n, int precision_bits, int* log2_factors, int* pass_c, int max, int* count) {
    if (!count || (max > 0 && (!log2_factors || !pass_c))) return fail(PHASTFT_ERR_INVALID_ARG, "NULL argument");
    if (!is_pow2(n)) return fail(PHASTFT_ERR_NOT_POW2);
    if (precision_bits != 32 && precision_bits != 64) return fail(PHASTFT_ERR_INVALID_ARG, "precision_bits must be 32 or 64");
    const int ln = ilog2(n);
    const std::vector<PlanChoice> c = precision_bits == 64 ? tune_candidates<double>(ln) : tune_candidates<float>(ln);
    *count = (int)c.size();
    for (int i = 0; i < std::min(max, (int)c.size()); ++i)
        for (int p = 0; p < MAX_PASSES; ++p) {
            const bool used = p < (int)c[i].factors.size();
            log2_factors[MAX_PASSES * i + p] = used ? c[i].factors[p] : 0;
            pass_c[MAX_PASSES * i + p] = used ? c[i].pass_c[p] : 0;
        }
    return PHASTFT_OK;
}

void phastft_options_default(phastft_options* out) {
    if (!out) return;
    out->multithreaded_bit_reversal = 0;
    out->smallest_parallel_chunk_size = 16384;
}
void phastft_options_guess(size_t input_size, phastft_options* out) {
    if (!out) return;
    phastft_options_default(out);
    out->multithreaded_bit_reversal = input_size ? (ilog2(input_size) >= 16) : 0;
}

#define DEFINE_DIT_API(T, SFX)                                                                                          \
    int32_t phastft_plan_dit_##SFX##_create(size_t n, int device, int mode, phastft_plan_dit_##SFX** out) {             \
        Plan<T>* pl = nullptr;                                                                                          \
        int32_t st = (mode == PHASTFT_MODE_TUNE) ? build_plan_tuned<T>(n, device, &pl) : build_plan<T>(n, device, &pl); \
        if (out) *out = reinterpret_cast<phastft_plan_dit_##SFX*>(pl);                                                  \
        else if (pl) delete pl;                                                                                         \
        return st;                                                                                                      \
    }                                                                                                                   \
    void phastft_plan_dit_##SFX##_destroy(phastft_plan_dit_##SFX* p) { delete AS_PLAN(T, p); }                          \
    size_t phastft_plan_dit_##SFX##_size(const phastft_plan_dit_##SFX* p) { return p ? AS_CPLAN(T, p)->n : 0; }         \
    const char* phastft_plan_dit_##SFX##_describe(const phastft_plan_dit_##SFX* p) {                                    \
        return p ? AS_CPLAN(T, p)->description.c_str() : "";                                                            \
    }                                                                                                                   \
    int32_t phastft_plan_dit_##SFX##_reserve(const phastft_plan_dit_##SFX* p, size_t batch) {                           \
        return plan_reserve<T>(AS_CPLAN(T, p), batch);                                                                  \
    }                                                                                                                   \
    size_t phastft_plan_dit_##SFX##_tables_bytes(const phastft_plan_dit_##SFX* p) {                                     \
        return p ? AS_CPLAN(T, p)->blob_host.size() : 0;                                                                \
    }                                                                                                                   \
    int32_t phastft_plan_dit_##SFX##_tables_export(const phastft_plan_dit_##SFX* p, void* dst, void* s) {               \
        return tables_export<T>(AS_CPLAN(T, p), dst, (cudaStream_t)s);                                                  \
    }                                                                                                                   \
    int32_t phastft_plan_dit_##SFX##_tables_import(phastft_plan_dit_##SFX* p, const void* src, void* s) {               \
        return tables_import<T>(AS_PLAN(T, p), src, (cudaStream_t)s);                                                   \
    }                                                                                                                   \
    int32_t phastft_plan_dit_##SFX##_tables_broadcast(phastft_plan_dit_##SFX* p, void* comm, int root, void* s) {       \
        return tables_broadcast<T>(AS_PLAN(T, p), comm, root, (cudaStream_t)s);                                         \
    }                                                                                                                   \
    int32_t phastft_fft_dit_##SFX##_host(const phastft_plan_dit_##SFX* p, T* re, size_t lre, T* im, size_t lim,        \
                                         int dir, const phastft_options* opts) {                                        \
        (void)opts;                                                                                                     \
        launches_reset();                                                                                               \
        return fft_host<T>(AS_CPLAN(T, p), re, lre, im, lim, dir);                                                      \
    }                                                                                                                   \
    int32_t phastft_fft_dit_##SFX##_oneshot(T* re, size_t lre, T* im, size_t lim, int dir, int device) {                \
        launches_reset();                                                                                               \
        return fft_oneshot<T>(re, lre, im, lim, dir, device);                                                           \
    }                                                                                                                   \
    int32_t phastft_fft_dit_##SFX##_dev(const phastft_plan_dit_##SFX* p, T* re, T* im, int dir, size_t batch,          \
                                        size_t bstride, void* s) {                                                      \
        launches_reset();                                                                                               \
        return fft_dev<T>(AS_CPLAN(T, p), re, im, dir, batch, bstride, (cudaStream_t)s);                                \
    }                                                                                                                   \
    int32_t phastft_fft_dit_##SFX##_dev_profile(const phastft_plan_dit_##SFX* p, T* re, T* im, int dir, size_t batch,  \
                                                size_t bstride, void* s, float* pass_ms, int* num_passes) {             \
        launches_reset();                                                                                               \
        return fft_dev_profile<T>(AS_CPLAN(T, p), re, im, dir, batch, bstride, (cudaStream_t)s, pass_ms, num_passes);   \
    }                                                                                                                   \
    int32_t phastft_fft_dit_##SFX##_batch_sharded_host(phastft_plan_dit_##SFX* const* plans, int np, T* re, T* im,     \
                                                       size_t batch, size_t bstride, int dir) {                         \
        launches_reset();                                                                                               \
        return batch_sharded_host<T>(reinterpret_cast<Plan<T>* const*>(plans), np, re, im, batch, bstride, dir);        \
    }                                                                                                                   \
    int32_t phastft_fft_interleaved_##SFX##_host(const phastft_plan_dit_##SFX* p, T* sig, size_t len, int dir) {        \
        launches_reset();                                                                                               \
        return fft_interleaved_host<T>(AS_CPLAN(T, p), sig, len, dir);                                                  \
    }                                                                                                                   \
    int32_t phastft_fft_interleaved_##SFX##_dev(const phastft_plan_dit_##SFX* p, T* sig, int dir, size_t batch,        \
                                                size_t bstride, void* s) {                                              \
        launches_reset();                                                                                               \
        return fft_interleaved_dev<T>(AS_CPLAN(T, p), sig, dir, batch, bstride, (cudaStream_t)s);                       \
    }                                                                                                                   \
    int32_t phastft_plan_r2c_##SFX##_create(size_t n, int device, phastft_plan_r2c_##SFX** out) {                       \
        PlanR2c<T>* pl = nullptr;                                                                                       \
        int32_t st = build_plan_r2c<T>(n, device, &pl);                                                                 \
        if (out) *out = reinterpret_cast<phastft_plan_r2c_##SFX*>(pl);                                                  \
        else if (pl) delete pl;                                                                                         \
        return st;                                                                                                      \
    }                                                                                                                   \
    void phastft_plan_r2c_##SFX##_destroy(phastft_plan_r2c_##SFX* p) { delete AS_R2C(T, p); }                           \
    size_t phastft_plan_r2c_##SFX##_size(const phastft_plan_r2c_##SFX* p) { return p ? AS_CR2C(T, p)->n : 0; }          \
    const char* phastft_plan_r2c_##SFX##_describe(const phastft_plan_r2c_##SFX* p) {                                    \
        if (!p) return "";                                                                                              \
        g_r2c_desc_text = r2c_description<T>(AS_CR2C(T, p), 1);                                                         \
        return g_r2c_desc_text.c_str();                                                                                 \
    }                                                                                                                   \
    const char* phastft_plan_r2c_##SFX##_describe_batch(const phastft_plan_r2c_##SFX* p, size_t batch) {                \
        if (!p) return "";                                                                                              \
        g_r2c_desc_text = r2c_description<T>(AS_CR2C(T, p), batch);                                                     \
        return g_r2c_desc_text.c_str();                                                                                 \
    }                                                                                                                   \
    int32_t phastft_plan_r2c_##SFX##_reserve(const phastft_plan_r2c_##SFX* p, size_t batch) {                           \
        return r2c_reserve<T>(AS_CR2C(T, p), batch);                                                                    \
    }                                                                                                                   \
    int32_t phastft_r2c_##SFX##_batch_dev(const phastft_plan_r2c_##SFX* p, const T* in, size_t in_stride, T* ore,      \
                                          T* oim, size_t out_stride, size_t batch, void* s) {                           \
        launches_reset();                                                                                               \
        return r2c_batch_dev<T>(AS_CR2C(T, p), in, in_stride, ore, oim, out_stride, batch, (cudaStream_t)s);            \
    }                                                                                                                   \
    int32_t phastft_c2r_##SFX##_batch_dev(const phastft_plan_r2c_##SFX* p, const T* ire, const T* iim,                 \
                                          size_t in_stride, T* out, size_t out_stride, T* sre, T* sim, size_t batch,    \
                                          void* s) {                                                                    \
        launches_reset();                                                                                               \
        return c2r_batch_dev<T>(AS_CR2C(T, p), ire, iim, in_stride, out, out_stride, sre, sim, batch, (cudaStream_t)s); \
    }                                                                                                                   \
    int32_t phastft_r2c_##SFX##_host(const phastft_plan_r2c_##SFX* p, const T* in, size_t lin, T* ore, size_t lore,    \
                                     T* oim, size_t loim) {                                                             \
        launches_reset();                                                                                               \
        return r2c_host<T>(AS_CR2C(T, p), in, lin, ore, lore, oim, loim);                                               \
    }                                                                                                                   \
    int32_t phastft_r2c_##SFX##_oneshot(const T* in, size_t lin, T* ore, size_t lore, T* oim, size_t loim, int dev) {   \
        launches_reset();                                                                                               \
        PlanR2c<T>* pl = nullptr; /* r2c.rs:522: PlannerR2c::new(input_re.len()), kept for the next same-size call */  \
        auto& c = oneshot_r2c_cache<T>();                                                                               \
        std::lock_guard<std::mutex> lock(c.mu);                                                                         \
        int32_t st = oneshot_r2c_plan<T>(c, lin, dev, &pl);                                                             \
        if (st) return st;                                                                                              \
        return r2c_host<T>(pl, in, lin, ore, lore, oim, loim);                                                          \
    }                                                                                                                   \
    int32_t phastft_r2c_##SFX##_dev(const phastft_plan_r2c_##SFX* p, const T* in, T* ore, T* oim, void* s) {            \
        launches_reset();                                                                                               \
        return r2c_dev<T>(AS_CR2C(T, p), in, ore, oim, (cudaStream_t)s);                                                \
    }                                                                                                                   \
    int32_t phastft_c2r_##SFX##_host(const phastft_plan_r2c_##SFX* p, const T* ire, size_t lire, const T* iim,          \
                                     size_t liim, T* out, size_t lout, T* sre, size_t lsre, T* sim, size_t lsim) {      \
        launches_reset();                                                                                               \
        return c2r_host<T>(AS_CR2C(T, p), ire, lire, iim, liim, out, lout, sre, lsre, sim, lsim);                       \
    }                                                                                                                   \
    int32_t phastft_c2r_##SFX##_oneshot(const T* ire, size_t lire, const T* iim, size_t liim, T* out, size_t lout,     \
                                        int dev) {                                                                      \
        launches_reset();                                                                                               \
        PlanR2c<T>* pl = nullptr; /* r2c.rs:696: PlannerR2c::new(output.len()), kept for the next same-size call */    \
        auto& c = oneshot_r2c_cache<T>();                                                                               \
        std::lock_guard<std::mutex> lock(c.mu);                                                                         \
        int32_t st = oneshot_r2c_plan<T>(c, lout, dev, &pl);                                                            \
        if (st) return st;                                                                                              \
        return c2r_host<T>(pl, ire, lire, iim, liim, out, lout, nullptr, 0, nullptr, 0);                                \
    }                                                                                                                   \
    int32_t phastft_c2r_##SFX##_dev(const phastft_plan_r2c_##SFX* p, const T* ire, const T* iim, T* out, T* sre,        \
                                    T* sim, void* s) {                                                                  \
        launches_reset();                                                                                               \
        return c2r_dev<T>(AS_CR2C(T, p), ire, iim, out, sre, sim, (cudaStream_t)s);                                     \
    }                                                                                                                   \
    int32_t phastft_plan_any_##SFX##_create(size_t n, int device, phastft_plan_any_##SFX** out) {                       \
        PlanAny<T>* pl = nullptr;                                                                                       \
        int32_t st = build_plan_any<T>(n, device, PHASTFT_ANY_BLUESTEIN, &pl);                                          \
        if (out) *out = reinterpret_cast<phastft_plan_any_##SFX*>(pl);                                                  \
        else if (pl) delete pl;                                                                                         \
        return st;                                                                                                      \
    }                                                                                                                   \
    int32_t phastft_plan_any_##SFX##_create_with(size_t n, int device, int algo, phastft_plan_any_##SFX** out) {        \
        PlanAny<T>* pl = nullptr;                                                                                       \
        int32_t st = build_plan_any<T>(n, device, algo, &pl);                                                           \
        if (out) *out = reinterpret_cast<phastft_plan_any_##SFX*>(pl);                                                  \
        else if (pl) delete pl;                                                                                         \
        return st;                                                                                                      \
    }                                                                                                                   \
    void phastft_plan_any_##SFX##_destroy(phastft_plan_any_##SFX* p) { delete AS_ANY(T, p); }                           \
    size_t phastft_plan_any_##SFX##_size(const phastft_plan_any_##SFX* p) { return p ? AS_CANY(T, p)->n : 0; }          \
    const char* phastft_plan_any_##SFX##_describe(const phastft_plan_any_##SFX* p) {                                    \
        return p ? AS_CANY(T, p)->description.c_str() : "";                                                             \
    }                                                                                                                   \
    int32_t phastft_plan_any_##SFX##_reserve(const phastft_plan_any_##SFX* p, size_t batch) {                           \
        return any_reserve<T>(AS_CANY(T, p), batch);                                                                    \
    }                                                                                                                   \
    int32_t phastft_fft_any_##SFX##_dev(const phastft_plan_any_##SFX* p, T* re, T* im, int dir, size_t batch,          \
                                        size_t bstride, void* s) {                                                      \
        launches_reset();                                                                                               \
        return any_dev<T>(AS_CANY(T, p), re, im, dir, batch, bstride, (cudaStream_t)s);                                 \
    }                                                                                                                   \
    int32_t phastft_fft_any_##SFX##_host(const phastft_plan_any_##SFX* p, T* re, size_t lre, T* im, size_t lim,        \
                                         int dir) {                                                                     \
        launches_reset();                                                                                               \
        return any_host<T>(AS_CANY(T, p), re, lre, im, lim, dir);                                                       \
    }                                                                                                                   \
    int32_t phastft_fft_interleaved_any_##SFX##_dev(const phastft_plan_any_##SFX* p, T* sig, int dir, size_t batch,    \
                                                    size_t bstride, void* s) {                                          \
        launches_reset();                                                                                               \
        return any_interleaved_dev<T>(AS_CANY(T, p), sig, dir, batch, bstride, (cudaStream_t)s);                        \
    }                                                                                                                   \
    int32_t phastft_fft_interleaved_any_##SFX##_host(const phastft_plan_any_##SFX* p, T* sig, size_t len, int dir) {    \
        launches_reset();                                                                                               \
        return any_interleaved_host<T>(AS_CANY(T, p), sig, len, dir);                                                   \
    }                                                                                                                   \
    int32_t phastft_plan_r2c_any_##SFX##_create(size_t n, int device, phastft_plan_r2c_any_##SFX** out) {               \
        PlanR2cAny<T>* pl = nullptr;                                                                                    \
        int32_t st = build_plan_r2c_any<T>(n, device, PHASTFT_ANY_BLUESTEIN, &pl);                                      \
        if (out) *out = reinterpret_cast<phastft_plan_r2c_any_##SFX*>(pl);                                              \
        else if (pl) delete pl;                                                                                         \
        return st;                                                                                                      \
    }                                                                                                                   \
    int32_t phastft_plan_r2c_any_##SFX##_create_with(size_t n, int device, int algo, phastft_plan_r2c_any_##SFX** out) {\
        PlanR2cAny<T>* pl = nullptr;                                                                                    \
        int32_t st = build_plan_r2c_any<T>(n, device, algo, &pl);                                                       \
        if (out) *out = reinterpret_cast<phastft_plan_r2c_any_##SFX*>(pl);                                              \
        else if (pl) delete pl;                                                                                         \
        return st;                                                                                                      \
    }                                                                                                                   \
    void phastft_plan_r2c_any_##SFX##_destroy(phastft_plan_r2c_any_##SFX* p) { delete AS_R2CANY(T, p); }                \
    size_t phastft_plan_r2c_any_##SFX##_size(const phastft_plan_r2c_any_##SFX* p) { return p ? AS_CR2CANY(T, p)->n : 0; }\
    const char* phastft_plan_r2c_any_##SFX##_describe(const phastft_plan_r2c_any_##SFX* p) {                            \
        if (!p) return "";                                                                                              \
        g_r2c_desc_text = r2c_any_description<T>(AS_CR2CANY(T, p));                                                     \
        return g_r2c_desc_text.c_str();                                                                                 \
    }                                                                                                                   \
    int32_t phastft_plan_r2c_any_##SFX##_reserve(const phastft_plan_r2c_any_##SFX* p, size_t batch) {                   \
        return r2c_any_reserve<T>(AS_CR2CANY(T, p), batch);                                                             \
    }                                                                                                                   \
    int32_t phastft_r2c_any_##SFX##_dev(const phastft_plan_r2c_any_##SFX* p, const T* in, size_t in_stride, T* ore,     \
                                        T* oim, size_t out_stride, size_t batch, void* s) {                             \
        launches_reset();                                                                                               \
        return r2c_any_dev<T>(AS_CR2CANY(T, p), in, in_stride, ore, oim, out_stride, batch, (cudaStream_t)s);           \
    }                                                                                                                   \
    int32_t phastft_c2r_any_##SFX##_dev(const phastft_plan_r2c_any_##SFX* p, const T* ire, const T* iim,                \
                                        size_t in_stride, T* out, size_t out_stride, size_t batch, void* s) {           \
        launches_reset();                                                                                               \
        return c2r_any_dev<T>(AS_CR2CANY(T, p), ire, iim, in_stride, out, out_stride, batch, (cudaStream_t)s);          \
    }                                                                                                                   \
    int32_t phastft_r2c_any_##SFX##_host(const phastft_plan_r2c_any_##SFX* p, const T* in, size_t lin, T* ore,          \
                                         size_t lore, T* oim, size_t loim) {                                            \
        launches_reset();                                                                                               \
        return r2c_any_host<T>(AS_CR2CANY(T, p), in, lin, ore, lore, oim, loim);                                        \
    }                                                                                                                   \
    int32_t phastft_r2c_interleaved_any_##SFX##_dev(const phastft_plan_r2c_any_##SFX* p, const T* in, size_t in_stride,  \
                                                     T* out, size_t out_stride, size_t batch, void* s) {                \
        launches_reset();                                                                                               \
        return r2c_il_any_dev<T>(AS_CR2CANY(T, p), in, in_stride, out, out_stride, batch, (cudaStream_t)s);             \
    }                                                                                                                   \
    int32_t phastft_c2r_interleaved_any_##SFX##_dev(const phastft_plan_r2c_any_##SFX* p, const T* in, size_t in_stride,  \
                                                     T* out, size_t out_stride, size_t batch, void* s) {                \
        launches_reset();                                                                                               \
        return c2r_il_any_dev<T>(AS_CR2CANY(T, p), in, in_stride, out, out_stride, batch, (cudaStream_t)s);             \
    }                                                                                                                   \
    int32_t phastft_r2c_interleaved_any_##SFX##_host(const phastft_plan_r2c_any_##SFX* p, const T* in, size_t lin,     \
                                                      T* out, size_t lout) {                                            \
        launches_reset();                                                                                               \
        return r2c_il_any_host<T>(AS_CR2CANY(T, p), in, lin, out, lout);                                                \
    }                                                                                                                   \
    int32_t phastft_c2r_interleaved_any_##SFX##_host(const phastft_plan_r2c_any_##SFX* p, const T* in, size_t lin,     \
                                                      T* out, size_t lout) {                                            \
        launches_reset();                                                                                               \
        return c2r_il_any_host<T>(AS_CR2CANY(T, p), in, lin, out, lout);                                                \
    }                                                                                                                   \
    int32_t phastft_c2r_any_##SFX##_host(const phastft_plan_r2c_any_##SFX* p, const T* ire, size_t lire, const T* iim,  \
                                         size_t liim, T* out, size_t lout) {                                            \
        launches_reset();                                                                                               \
        return c2r_any_host<T>(AS_CR2CANY(T, p), ire, lire, iim, liim, out, lout);                                      \
    }                                                                                                                   \
    int32_t phastft_plan_dct_##SFX##_create_with(size_t n, int device, int algo, phastft_plan_dct_##SFX** out) {        \
        PlanDct<T>* pl = nullptr;                                                                                       \
        int32_t st = build_plan_dct<T>(n, device, algo, &pl);                                                           \
        if (out) *out = reinterpret_cast<phastft_plan_dct_##SFX*>(pl);                                                  \
        else if (pl) delete pl;                                                                                         \
        return st;                                                                                                      \
    }                                                                                                                   \
    void phastft_plan_dct_##SFX##_destroy(phastft_plan_dct_##SFX* p) { delete AS_DCT(T, p); }                           \
    size_t phastft_plan_dct_##SFX##_size(const phastft_plan_dct_##SFX* p) { return p ? AS_CDCT(T, p)->n : 0; }          \
    const char* phastft_plan_dct_##SFX##_describe(const phastft_plan_dct_##SFX* p) {                                    \
        if (!p) return "";                                                                                              \
        g_r2c_desc_text = dct_description<T>(AS_CDCT(T, p));                                                            \
        return g_r2c_desc_text.c_str();                                                                                 \
    }                                                                                                                   \
    int32_t phastft_plan_dct_##SFX##_reserve(const phastft_plan_dct_##SFX* p, size_t batch) {                           \
        return dct_reserve<T>(AS_CDCT(T, p), batch);                                                                    \
    }                                                                                                                   \
    int32_t phastft_dct_##SFX##_dev(const phastft_plan_dct_##SFX* p, int kind, int norm, const T* in, size_t in_stride,  \
                                    T* out, size_t out_stride, size_t batch, void* s) {                                 \
        launches_reset();                                                                                               \
        return dct_dev<T>(AS_CDCT(T, p), kind, norm, in, in_stride, out, out_stride, batch, (cudaStream_t)s);           \
    }                                                                                                                   \
    int32_t phastft_dct_##SFX##_host(const phastft_plan_dct_##SFX* p, int kind, int norm, const T* in, size_t lin,       \
                                     T* out, size_t lout) {                                                             \
        launches_reset();                                                                                               \
        return dct_host<T>(AS_CDCT(T, p), kind, norm, in, lin, out, lout);                                              \
    }                                                                                                                   \
    int32_t phastft_plan_conv_##SFX##_create(size_t n_x, size_t n_h, int domain, int device,                            \
                                             phastft_plan_conv_##SFX** out) {                                           \
        PlanConv<T>* pl = nullptr;                                                                                      \
        int32_t st = build_plan_conv<T>(n_x, n_h, domain, device, &pl);                                                 \
        if (out) *out = reinterpret_cast<phastft_plan_conv_##SFX*>(pl);                                                 \
        else if (pl) delete pl;                                                                                         \
        return st;                                                                                                      \
    }                                                                                                                   \
    void phastft_plan_conv_##SFX##_destroy(phastft_plan_conv_##SFX* p) { delete AS_CONV(T, p); }                        \
    size_t phastft_plan_conv_##SFX##_fft_len(const phastft_plan_conv_##SFX* p) { return p ? AS_CCONV(T, p)->L : 0; }    \
    const char* phastft_plan_conv_##SFX##_describe(const phastft_plan_conv_##SFX* p) {                                  \
        if (!p) return "";                                                                                              \
        g_r2c_desc_text = conv_description<T>(AS_CCONV(T, p));                                                          \
        return g_r2c_desc_text.c_str();                                                                                 \
    }                                                                                                                   \
    int32_t phastft_plan_conv_##SFX##_reserve(const phastft_plan_conv_##SFX* p, size_t batch) {                         \
        return conv_reserve<T>(AS_CCONV(T, p), batch);                                                                  \
    }                                                                                                                   \
    int32_t phastft_conv_##SFX##_dev(const phastft_plan_conv_##SFX* p, int op, int mode, const T* x, size_t x_stride,   \
                                     const T* h, size_t h_stride, T* y, size_t y_stride, size_t batch, void* s) {       \
        launches_reset();                                                                                               \
        return conv_dev<T>(AS_CCONV(T, p), op, mode, x, x_stride, h, h_stride, y, y_stride, batch, (cudaStream_t)s);    \
    }                                                                                                                   \
    int32_t phastft_conv_##SFX##_host(const phastft_plan_conv_##SFX* p, int op, int mode, const T* x, size_t len_x,     \
                                      const T* h, size_t len_h, T* y, size_t len_y) {                                   \
        launches_reset();                                                                                               \
        return conv_host<T>(AS_CCONV(T, p), op, mode, x, len_x, h, len_h, y, len_y);                                    \
    }                                                                                                                   \
    int32_t phastft_plan_stft_##SFX##_create(size_t n, size_t n_fft, size_t hop, const T* window, size_t win_length,    \
                                             int center, int pad_mode, int domain, int device,                          \
                                             phastft_plan_stft_##SFX** out) {                                           \
        PlanStft<T>* pl = nullptr;                                                                                      \
        int32_t st = build_plan_stft<T>(n, n_fft, hop, window, win_length, center, pad_mode, domain, device, &pl);     \
        if (out) *out = reinterpret_cast<phastft_plan_stft_##SFX*>(pl);                                                 \
        else if (pl) delete pl;                                                                                         \
        return st;                                                                                                      \
    }                                                                                                                   \
    void phastft_plan_stft_##SFX##_destroy(phastft_plan_stft_##SFX* p) { delete AS_STFT(T, p); }                        \
    size_t phastft_plan_stft_##SFX##_frames(const phastft_plan_stft_##SFX* p) { return p ? AS_CSTFT(T, p)->frames : 0; }\
    size_t phastft_plan_stft_##SFX##_bins(const phastft_plan_stft_##SFX* p) { return p ? AS_CSTFT(T, p)->bins : 0; }    \
    const char* phastft_plan_stft_##SFX##_describe(const phastft_plan_stft_##SFX* p) {                                  \
        if (!p) return "";                                                                                              \
        g_r2c_desc_text = stft_description<T>(AS_CSTFT(T, p));                                                          \
        return g_r2c_desc_text.c_str();                                                                                 \
    }                                                                                                                   \
    int32_t phastft_plan_stft_##SFX##_reserve(const phastft_plan_stft_##SFX* p, size_t batch) {                         \
        return stft_reserve<T>(AS_CSTFT(T, p), batch);                                                                  \
    }                                                                                                                   \
    int32_t phastft_stft_##SFX##_dev(const phastft_plan_stft_##SFX* p, int normalized, const T* x, size_t x_stride,     \
                                     T* spec, size_t frame_stride, size_t batch, void* s) {                             \
        launches_reset();                                                                                               \
        return stft_dev<T>(AS_CSTFT(T, p), normalized, x, x_stride, spec, frame_stride, batch, (cudaStream_t)s);        \
    }                                                                                                                   \
    int32_t phastft_istft_##SFX##_dev(const phastft_plan_stft_##SFX* p, int normalized, const T* spec,                  \
                                      size_t frame_stride, T* y, size_t y_stride, size_t batch, void* s) {              \
        launches_reset();                                                                                               \
        return istft_dev<T>(AS_CSTFT(T, p), normalized, spec, frame_stride, y, y_stride, batch, (cudaStream_t)s);       \
    }                                                                                                                   \
    int32_t phastft_stft_##SFX##_host(const phastft_plan_stft_##SFX* p, int normalized, const T* x, size_t len_x,       \
                                      T* spec, size_t len_spec) {                                                       \
        launches_reset();                                                                                               \
        return stft_host<T>(AS_CSTFT(T, p), normalized, x, len_x, spec, len_spec);                                      \
    }                                                                                                                   \
    int32_t phastft_istft_##SFX##_host(const phastft_plan_stft_##SFX* p, int normalized, const T* spec,                 \
                                       size_t len_spec, T* y, size_t len_y) {                                           \
        launches_reset();                                                                                               \
        return istft_host<T>(AS_CSTFT(T, p), normalized, spec, len_spec, y, len_y);                                     \
    }

DEFINE_DIT_API(double, f64)
DEFINE_DIT_API(float, f32)

size_t phastft_conv_out_len(size_t n_x, size_t n_h, int mode) { return conv_out_len(n_x, n_h, mode); }

}  // extern "C"
