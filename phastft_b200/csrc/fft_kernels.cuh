// fft_kernels.cuh -- the three sm_90a pass kernels of the H100 FFT.
//
// One launch = one "pass" over the whole signal: every CTA owns an R x C tile (R-point
// sub-transform x C adjacent columns/rows), runs all log2(R) butterfly stages on it with
// the tile held in shared memory between register-resident radix-4/8/16 stages, and
// touches HBM exactly once for the read and once for the write.  A transform of
// N = R_1 * R_2 [* R_3] points is 1, 2 or 3 such launches (DESIGN.md section 3).
//
// What this replaces in the reference (all CPU, one sweep over memory per radix-2 stage):
//   algorithms/dit.rs:33-164   recursive cache-blocked DIT driver      -> the pass decomposition
//   algorithms/bravo.rs:82-251 BRAVO / CO-BRAVO bit-reversal           -> folded into addressing:
//        digit-reversed placement into shared memory on load (stage 1) and the transposed
//        store of the last pass; no separate permutation pass exists on the GPU
//   kernels/dit.rs:971-1115    fft_dit_chunk_n (planner-twiddle stage) -> stage twiddles from the
//        per-pass W_R table, inter-pass twiddles from a two-level W_N table built by the planner
//   algorithms/dit.rs:325-331  inverse 1/N scaling loop                -> fused into the last store
//
// Kernel kinds
//   KIND_COL   first / middle pass: tile rows are strided (stride B), columns contiguous.
//              load [r][c] -> store [k][c], same addresses (layout preserving, in-place safe).
//   KIND_TRANS last pass of a multi-pass plan: tile rows are contiguous sub-sequences, the C rows
//              of a tile are C adjacent values of the slowest input digit; the store is the
//              digit-reversing transpose, written as C-element contiguous runs.
//   KIND_ROW   whole transform in one CTA (N <= 4096 f64 / 8192 f32): rows contiguous in and out.
#pragma once
#ifndef PHAST_EXP_STAGE_TW
#define PHAST_EXP_STAGE_TW 0
#endif
#include <cuda.h>
#include <type_traits>

#include "fft_device.cuh"

namespace phast {

enum { KIND_COL = 0, KIND_TRANS = 1, KIND_ROW = 2 };

template <typename T>
struct PassParams {
    const T* in_re;                // planar input (or interleaved (re,im) pairs if in_interleaved)
    const T* in_im;                // (no __restrict__: in-place passes alias in and out)
    T* out_re;                     // planar output (or interleaved if out_interleaved)
    T* out_im;
    long long in_bstride;          // elements between consecutive transforms of the batch
    long long out_bstride;
    int batch;                     // number of transforms (KIND_ROW: may not be a multiple of C)
    int in_interleaved;            // 1: in_re points at N (re,im) pairs (r2c first pass); 2: pairs, re/im swapped
    int out_interleaved;           // 1: out_re points at N pairs; 2: pairs with re/im swapped (c2r)
    // geometry
    int log2A;                     // A = number of sub-transform groups before this digit
    int log2B;                     // B = stride of this pass's digit = product of later pass sizes
    int log2R1;                    // KIND_TRANS: size of the first pass digit (tile columns run over it)
    int log2Rprev;                 // size of the previous pass digit (0 if no inter-pass twiddle)
    int blk_offset;                // KIND_COL: first linear tile index of this launch (L2-blocked sub-range of `a`)
    int kt_base;                   // KIND_TRANS: first k1 tile of this launch ...
    int log2_ktn;                  // ... and log2 of the number of k1 tiles it covers
    int pdl;                       // launched with programmatic stream serialization
    int has_tw;                    // apply inter-pass twiddle on load
    int tw_shift;                  // exponent scale: e_N = e_L << tw_shift   (N / L)
    Tw2 tw2;                       // two-level W_N table
    const cx<T>* __restrict__ tw_stage;  // W_R^e, e < R           (stage twiddles)
    const cx<T>* __restrict__ tw_stage_im;  // KIND_ROW: per stage s >= 1 the table [i][m] = W_L^(m*i), L = Ns(s)*rad(s), concatenated
                                         // (lanes run along m in a one-CTA kernel: consecutive lanes read consecutive entries);
                                         // KIND_COL / KIND_TRANS with a radix-32 last stage: its table [m][i] = W_R^(m*i), i < 32
                                         // (stage32_table_kernel); otherwise unused
    const cx<T>* __restrict__ tw_wc;     // KIND_TRANS, 2-pass plans: W_L^(c*m), [c][m] layout
    T scale;                       // multiplied into the stored result (1/N for the inverse)
    // cluster exchange (XCH = 1 producer only): the consuming pass's tile is [CB rows][P2 points]
    int xch_log2P2;                // log2 of the consumer's row length (= its R)
    int xch_log2CB;                // log2 of the consumer's rows per CTA (= its C)
    // ring of workspace slots (fft_pipe2_kernel): transform b's intermediate lives in slot b % ring (ring a power of two; 0 = none)
    int out_ring;                  // KIND_COL: applied to the batch index of the OUTPUT address
    int in_ring;                   // KIND_TRANS: applied to the batch index of the INPUT address
    // c2r pre-processing on load (MODE_C2R_IN only): in_re / in_im are the N/2 + 1 bins of the half-spectrum, the pass's
    // input element k is built from bins k and N/2 - k with the twiddle W_N^k out of this table
    Tw2 pre_tw2;
    int pre_log2half;              // log2(N/2); 0 = no pre-processing
    double2 pre_wc[32];            // W_(2 R1)^i, i < R1 = the kernel's first radix
    // TMA tile input (MODE_TMA_IN only): one tensor map per planar array, dims {B columns, R rows, batch}
    alignas(64) CUtensorMap tmap_re;
    alignas(64) CUtensorMap tmap_im;
};

// Shared-memory tile addressing (units: complex elements).
//   CFAST kernels (COL, TRANS): [pos][c'] with c' = c ^ swz(pos)  (swz == 0 for COL)
//   ROW kernel: [c][pos'] with pos' = pos ^ swz(pos)
// swz(pos) takes the bits of `pos` in which the low bits of the *memory-order* index of stage 1
// land after digit reversal, so that the stage-1 scatter of a coalesced global read is
// bank-conflict free; later stages address whole rows / aligned runs and are unaffected.
template <class RL, int C, int KIND, typename T>
struct TileAddr {
    static constexpr int R = RL::R();
    static constexpr int LOG2R = ilog2_c(R);
    static constexpr int RS_LAST = RL::rad(RL::S - 1);
    static constexpr int SWZ_SHIFT = LOG2R - ilog2_c(RS_LAST);
    // 16-byte (f64) / 8-byte (f32) complex elements: a 128-byte wavefront holds 8 / 16 of them
    static constexpr int LANES_PER_WF = 128 / (2 * (int)sizeof(T));
    static constexpr int SWZ_MASK_WANT = LANES_PER_WF - 1;
    static constexpr int SWZ_MASK_TRANS = (C - 1) < SWZ_MASK_WANT ? (C - 1) : SWZ_MASK_WANT;
    static constexpr int SWZ_MASK_ROW = (R >= 4 * LANES_PER_WF) ? SWZ_MASK_WANT : 0;
    static __device__ __forceinline__ int at(int pos, int c) {
        if constexpr (KIND == KIND_COL) {
            return pos * C + c;
        } else if constexpr (KIND == KIND_TRANS) {
            return pos * C + (c ^ ((pos >> SWZ_SHIFT) & SWZ_MASK_TRANS));
        } else {
            return c * R + (pos ^ ((pos >> SWZ_SHIFT) & SWZ_MASK_ROW));
        }
    }
};

// ---------------------------------------------------------------------------------------------
// The pass kernel.
// ---------------------------------------------------------------------------------------------
// Cluster exchange helpers (thread-block clusters + distributed shared memory, sm_90+):
//   cluster_sync()        barrier.cluster arrive(release) + wait(acquire) by every thread of every CTA of the cluster
//   st_cluster(addr, v)   store into the shared memory of CTA `rank` of the cluster (mapa + st.shared::cluster)
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ unsigned cluster_ctarank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ unsigned map_to_rank(unsigned smem_addr, unsigned rank) {
    unsigned r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void st_cluster(unsigned addr, const double2& v) {
    asm volatile("st.shared::cluster.v2.f64 [%0], {%1, %2};" ::"r"(addr), "d"(v.x), "d"(v.y) : "memory");
}
__device__ __forceinline__ void st_cluster(unsigned addr, const float2& v) {
    asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v.x), "f"(v.y) : "memory");
}

// TMA / mbarrier helpers (sm_90+; SASS: UTMALDG for the tensor copy, UBLKCP for the 1-D bulk copy, SYNCS for the mbarrier)
__device__ __forceinline__ void mbar_init(unsigned mbar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned mbar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned mbar, unsigned parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n"
        "DONE_%=:\n\t}" ::"r"(mbar), "r"(parity) : "memory");
}
// 3-D tensor tile (box fixed in the map) global -> shared, completion counted on `mbar`
__device__ __forceinline__ void tma_load_3d(unsigned smem_dst, const CUtensorMap* map, int x, int y, int z, unsigned mbar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(smem_dst), "l"(map), "r"(x), "r"(y), "r"(z), "r"(mbar) : "memory");
}
// contiguous bytes global -> shared (16-byte aligned, size a multiple of 16)
__device__ __forceinline__ void bulk_load_1d(unsigned smem_dst, const void* gsrc, unsigned bytes, unsigned mbar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_dst), "l"(gsrc), "r"(bytes), "r"(mbar) : "memory");
}

// XCH (how this pass gets its input tile / where its last stage puts its results):
//   0  plain pass: global memory in, global memory out
//   1  producer (KIND_COL): the LAST stage does not store to global memory; every thread keeps its results in
//      registers across a cluster barrier and then scatters them into the shared-memory tiles of the CTAs that own
//      the rows in the next pass, in the layout [row c'][t] that pass's global loads would have read
//   2  consumer (KIND_TRANS): stage 1 reads that tile instead of global memory (all threads first, then a
//      __syncthreads, then the tile is overwritten in the pass's own layout)
//   3  TMA tile input (KIND_COL, first pass, planar input): one thread issues cp.async.bulk.tensor copies of the tile's
//      R x C boxes of the re and im arrays straight into the tile's shared memory (no per-thread address generation, no
//      LSU sector waste on the 32-byte runs of a 4-column f64 tile -- which is what lets a 1024-row tile be 64 KB and three
//      CTAs share an SM); the threads wait on the mbarrier, read their stage-1 inputs out of the landing zone, and go on as usual
//   4  bulk tile input (KIND_TRANS, interleaved intermediates): the tile's C rows are contiguous in the workspace -- C
//      cp.async.bulk copies land them as [c][t], then as mode 2
//   5  c2r pre-processing on load (first pass of the half-length inverse transform inside c2r): the input element k is
//      computed from bins k and N/2 - k of the half-spectrum while it is being loaded (the reference's separate sweep
//      r2c.rs:764-780 and its scratch round trip disappear: one HBM pass less per c2r)
//   6  bulk tile input AND output (KIND_ROW, batches whose transforms lie back to back in planar arrays): the CTA's C transforms
//      are one contiguous run per plane -- two cp.async.bulk copies bring them in (landing zone = the tile, planar [c][r]), the
//      last stage writes its results into a second planar staging area and two cp.async.bulk copies take them out.  The
//      per-lane 4/8-byte accesses of the plain kernel (128 bytes per f32 warp instruction, the bound of the 16..128-point
//      batches) become two asynchronous copies per CTA.
//   7  as 5 with the half-spectrum's bins interleaved (phastft_c2r_interleaved_any_*): in_re holds N/2 + 1 Complex<T> values
//      per member and bins k and N/2 - k are one Complex<T> load each; the arithmetic is mode 5's
enum { MODE_PLAIN = 0, MODE_XCH_PRODUCE = 1, MODE_XCH_CONSUME = 2, MODE_TMA_IN = 3, MODE_BULK_IN = 4, MODE_C2R_IN = 5, MODE_ROW_BULK = 6,
       MODE_C2R_IN_IL = 7 };
template <typename T, class RL, int C, int NT, int KIND, int XCH = 0, int VARIANT = 0>
struct PassKernel {
    static constexpr int S = RL::S;
    static constexpr int R = RL::R();
    static constexpr int LOG2R = ilog2_c(R);
    static constexpr int TILE_C = C;               // tile width (columns for COL, rows for TRANS / ROW)
    static constexpr int R1 = RL::rad(0);          // first-stage radix
    static constexpr int M = R / R1;               // stage-1 tasks per column
    static constexpr int LOG2C = ilog2_c(C);
    using Addr = TileAddr<RL, C, KIND, T>;
    // shared memory: tile (only if S >= 2) + Um[M] + G[C][R1]
    static constexpr int TILE_ELEMS = (S >= 2) ? R * C : 0;
    static constexpr int G_ELEMS = (KIND == KIND_TRANS) ? C * R1 : R1;
    static constexpr bool ASYNC_IN = (XCH == MODE_TMA_IN || XCH == MODE_BULK_IN || XCH == MODE_ROW_BULK);
    static constexpr bool C2R_IN = (XCH == MODE_C2R_IN || XCH == MODE_C2R_IN_IL);   // c2r pre-processing on load
    // strided tiles whose last stage is radix 32 (1024 = 32 x 32, 512 = 16 x 32): that stage reads W_R^(m*i) from the plan's
    // [m][i] table (PassParams::tw_stage_im), and stage 1 is written as a single trip when it can be (see body())
    static constexpr bool STAGE32 = KIND != KIND_ROW && S >= 2 && RL::rad(S - 1) == 32;
    static constexpr size_t TABLE_END = sizeof(cx<T>) * (size_t)(TILE_ELEMS + M + G_ELEMS);
    static constexpr size_t MBAR_OFF = (TABLE_END + 15) & ~size_t(15);
    static constexpr size_t OUT_OFF = (MBAR_OFF + 16 + 127) & ~size_t(127);      // MODE_ROW_BULK: planar output staging [2][C][R]
    static constexpr size_t SMEM_BYTES = XCH == MODE_ROW_BULK ? OUT_OFF + sizeof(cx<T>) * (size_t)TILE_ELEMS : ASYNC_IN ? MBAR_OFF + 16 : TABLE_END;
    static_assert(XCH == 0 || S >= 2, "an exchanging pass needs a shared-memory tile");
    static_assert(XCH != 1 || KIND == KIND_COL, "the producer of a cluster exchange is a COL pass");
    static_assert(XCH != 2 || KIND == KIND_TRANS, "the consumer of a cluster exchange is a TRANS pass");
    static_assert(XCH != MODE_TMA_IN || (KIND == KIND_COL && C * sizeof(T) >= 16), "TMA tile input: COL pass, rows of >= 16 bytes");
    static_assert(XCH != MODE_BULK_IN || KIND == KIND_TRANS, "bulk tile input: TRANS pass");
    static_assert(XCH != MODE_ROW_BULK || KIND == KIND_ROW, "bulk tile input and output: one-CTA kernels");

    // ---- global element access -------------------------------------------------------------
    static __device__ __forceinline__ void gload(const PassParams<T>& p, long long idx, T& re, T& im) {
        if (p.in_interleaved) {
            cx<T> v = reinterpret_cast<const cx<T>*>(p.in_re)[idx];
            if (p.in_interleaved == 1) { re = v.x; im = v.y; } else { re = v.y; im = v.x; }
        } else {
            re = p.in_re[idx];
            im = p.in_im[idx];
        }
    }
    static __device__ __forceinline__ void gstore(const PassParams<T>& p, long long idx, T re, T im) {
        if (p.scale != T(1)) { re *= p.scale; im *= p.scale; }
        if (p.out_interleaved == 0) {
            p.out_re[idx] = re;
            p.out_im[idx] = im;
        } else if (p.out_interleaved == 1) {
            reinterpret_cast<cx<T>*>(p.out_re)[idx] = make_cx<T>(re, im);
        } else {
            reinterpret_cast<cx<T>*>(p.out_re)[idx] = make_cx<T>(im, re);
        }
    }

    // N strided elements at once.  The layout test is hoisted out of the unrolled loop so each layout gets
    // its own straight-line block behind a uniform branch: with the test inside the loop the compiler
    // predicates both layouts into one stream (every launch then issues the other layout's dead loads and
    // selects, and the selects of the interleaved path split its loads into two dependent batches).
    // Layout class: 0 planar, 1 interleaved (re, im), 2 interleaved swapped (im, re), -1 = test at run time.
    // MODE_C2R_IN: element k of the half-length inverse transform's input, built on the fly from the half-spectrum
    // (same arithmetic, in the same order, as c2r_preprocess_kernel below; r2c.rs:263-347).  The inverse runs as a forward
    // transform of the swapped parts (r2c.rs:782), so the kernel is handed (im, re).
    // `mbase`: where the batch member's spectrum starts (member * in_bstride); a0 - mbase is the bin index.
    // MODE_C2R_IN_IL: the same bins as one Complex<T> each (indices and strides count complex values).
    template <int N>
    static __device__ __forceinline__ void gload_c2r(const PassParams<T>& p, long long a0, long long step, cx<T> (&x)[N],
                                                     long long mbase) {
        // element i is bin k = k0 + i * step with step = (N/2) / R1 (first pass: R * B = N/2), so its twiddle
        // W_N^k = W_N^k0 * W_(2 R1)^i: one table lookup per task, the second factors are launch constants (pre_wc).
        // Its partner bin N/2 - k lies in the same member.
        // Loads in groups of 8 (f64): 4 scalars per element, all of a group in flight at once.
        const long long half = 1LL << p.pre_log2half;
        const long long k0 = a0 - mbase;
        const T* __restrict__ fr = p.in_re + a0;
        const T* __restrict__ fi = p.in_im + a0;
        const T* __restrict__ sr = p.in_re + (mbase + half - k0);
        const T* __restrict__ si = p.in_im + (mbase + half - k0);
        [[maybe_unused]] const cx<T>* __restrict__ fc = reinterpret_cast<const cx<T>*>(p.in_re) + a0;
        [[maybe_unused]] const cx<T>* __restrict__ sc = reinterpret_cast<const cx<T>*>(p.in_re) + (mbase + half - k0);
        const double2 wb = p.pre_tw2.get((uint32_t)k0);
        constexpr int G = (sizeof(T) == 8 && N > 8) ? 8 : N;
#pragma unroll
        for (int g0 = 0; g0 < N; g0 += G) {
            T re_f[G], im_f[G], re_s[G], im_s[G];
#pragma unroll
            for (int i = 0; i < G; ++i) {
                const long long off = (long long)(g0 + i) * step;
                if constexpr (XCH == MODE_C2R_IN_IL) {
                    const cx<T> f = fc[off], s = sc[-off];
                    re_f[i] = f.x; im_f[i] = f.y;
                    re_s[i] = s.x; im_s[i] = -s.y;
                } else {
                    re_f[i] = fr[off]; im_f[i] = fi[off];
                    re_s[i] = sr[-off]; im_s[i] = -si[-off];
                }
            }
#pragma unroll
            for (int i = 0; i < G; ++i) {
                const double2 wd = (g0 + i == 0) ? wb : cmul_d(wb, p.pre_wc[g0 + i]);
                const T c_h = T(0.5 * wd.x), s_h = T(0.5 * wd.y);
                const T zx_re = T(0.5) * (re_f[i] + re_s[i]), zx_im = T(0.5) * (im_f[i] + im_s[i]);
                const T dr = re_f[i] - re_s[i], di = im_f[i] - im_s[i];
                const T zy_re = c_h * dr + s_h * di;
                const T zy_im = c_h * di - s_h * dr;
                x[g0 + i] = make_cx<T>(zx_im + zy_re, zx_re - zy_im);
            }
        }
    }
    template <int N, int IL = -1>
    static __device__ __forceinline__ void gload_n(const PassParams<T>& p, long long a0, long long step, cx<T> (&x)[N],
                                                   [[maybe_unused]] long long mbase = 0) {
        if constexpr (C2R_IN) {
            gload_c2r<N>(p, a0, step, x, mbase);
        } else if constexpr (IL < 0) {
            if (p.in_interleaved == 0) gload_n<N, 0>(p, a0, step, x);
            else if (p.in_interleaved == 1) gload_n<N, 1>(p, a0, step, x);
            else gload_n<N, 2>(p, a0, step, x);
        } else if constexpr (IL == 0) {
            const T* pr = p.in_re + a0;
            const T* pi = p.in_im + a0;
#pragma unroll
            for (int i = 0; i < N; ++i) x[i] = make_cx<T>(pr[(long long)i * step], pi[(long long)i * step]);
        } else {
            const cx<T>* pc = reinterpret_cast<const cx<T>*>(p.in_re) + a0;
#pragma unroll
            for (int i = 0; i < N; ++i) {
                const cx<T> v = pc[(long long)i * step];
                x[i] = (IL == 1) ? v : make_cx<T>(v.y, v.x);
            }
        }
    }
    template <int N, int OL = -1>
    static __device__ __forceinline__ void gstore_n(const PassParams<T>& p, long long a0, long long step, cx<T> (&x)[N]) {
        if constexpr (OL < 0) {
            if (p.out_interleaved == 0) gstore_n<N, 0>(p, a0, step, x);
            else if (p.out_interleaved == 1) gstore_n<N, 1>(p, a0, step, x);
            else gstore_n<N, 2>(p, a0, step, x);
        } else {
            if (p.scale != T(1)) {
#pragma unroll
                for (int i = 0; i < N; ++i) x[i] = cscale<T>(x[i], p.scale);
            }
            if constexpr (OL == 0) {
                T* pr = p.out_re + a0;
                T* pi = p.out_im + a0;
#pragma unroll
                for (int i = 0; i < N; ++i) { pr[(long long)i * step] = x[i].x; pi[(long long)i * step] = x[i].y; }
            } else {
                cx<T>* pc = reinterpret_cast<cx<T>*>(p.out_re) + a0;
#pragma unroll
                for (int i = 0; i < N; ++i) pc[(long long)i * step] = (OL == 1) ? x[i] : make_cx<T>(x[i].y, x[i].x);
            }
        }
    }

    // OL: output layout class of the LAST stage's stores (see gload_n); the test is made once
    // per stage (run_stages), outside the task loop, so each layout is a straight-line loop.
    template <int s, int OL = -1>
    static __device__ __forceinline__ void stage_from_tile(const PassParams<T>& p, cx<T>* tile, long long out_base,
                                                           long long out_kstride, int tile_rows_valid, int tid) {
        constexpr int RAD = RL::rad(s);
        constexpr int NS = RL::Ns(s);
        constexpr int J = R / RAD;                      // tasks per column
        constexpr int TW_SHIFT = LOG2R - ilog2_c(NS * RAD);
        constexpr bool LAST = (s == S - 1);
        constexpr int NTASK = J * C;
        constexpr int TRIPS = (NTASK + NT - 1) / NT;
#pragma unroll((VARIANT & 1) ? TRIPS : 1)
        for (int t = tid; t < NTASK; t += NT) {
            int c, j;
            if constexpr (KIND == KIND_ROW) { j = t % J; c = t / J; } else { c = t % C; j = t / C; }
            const int m = j & (NS - 1);
            const int g = j / NS;
            const int base = g * NS * RAD + m;
            cx<T> x[RAD];
#pragma unroll
            for (int i = 0; i < RAD; ++i) x[i] = tile[Addr::at(base + i * NS, c)];
            if constexpr ((VARIANT & 2) && RAD == 8) {
                // 3 table loads (W^m, W^2m, W^4m), the other four twiddles by complex products
                cx<T> w1 = __ldg(p.tw_stage + ((m * 1) << TW_SHIFT));
                cx<T> w2 = __ldg(p.tw_stage + ((m * 2) << TW_SHIFT));
                cx<T> w4 = __ldg(p.tw_stage + ((m * 4) << TW_SHIFT));
                cx<T> w3 = ctwid<T>(w1, w2), w5 = ctwid<T>(w1, w4), w6 = ctwid<T>(w2, w4);
                cx<T> w7 = ctwid<T>(w3, w4);
                const cx<T> ws[8] = {w1, w1, w2, w3, w4, w5, w6, w7};
#pragma unroll
                for (int i = 1; i < RAD; ++i) x[i] = ctwid<T>(x[i], ws[i]);
            } else if constexpr (KIND == KIND_ROW) {
                // One-CTA kernels run their lanes along the row, so m differs from lane to lane: W_R^(m*i) out of the plain W_R table is
                // a 32-way gather (15 of them per radix-16 task: measured at 40-50 % of these kernels' time).
                // The per-stage table in [i][m] order makes every one of those loads a contiguous run.
                constexpr int TW_OFF = tw_im_offset<RL>(s);
                const cx<T>* tws = p.tw_stage_im + TW_OFF + m;
                // only the rows i = 1, 2, 4, 8, ... are loaded; W^(m*i) for the other i is the product of two earlier ones
                // (i = hi + lo, hi the top bit: at most popcount(i) - 1 <= 3 products deep for radix 16): 4 loads + 11 products
                // instead of 15 loads per radix-16 task
                cx<T> w[RAD];
#pragma unroll
                for (int i = 1; i < RAD; ++i) {
                    const int hi = 1 << (31 - __builtin_clz((unsigned)i));
                    if (i == hi) w[i] = __ldg(tws + i * NS);
                    else w[i] = ctwid<T>(w[hi], w[i - hi]);
                    x[i] = ctwid<T>(x[i], w[i]);
                }
            } else if constexpr (STAGE32 && LAST) {
                // The product chain below would keep up to 15 complex twiddles live beside the 32 values and spill the
                // 1024-row tiles on sm_90a.  Its results for every m come instead from the plan's [m][i] table, which
                // stage32_table_kernel fills with that same chain (bit-identical values): 31 loads (L1-resident), no products.
                static_assert(RAD == 32 && NS * RAD == R, "the radix-32 table holds the tile's last stage");
                const cx<T>* tws = p.tw_stage_im + m * RAD;
#pragma unroll
                for (int i = 1; i < RAD; ++i) x[i] = ctwid<T>(x[i], __ldg(tws + i));
            } else {
#if PHAST_EXP_STAGE_TW == 1      // experiment: no stage twiddles (wrong results; prices them)
#elif PHAST_EXP_STAGE_TW == 2    // experiment: the round-1 form, one table load per twiddle
#pragma unroll
                for (int i = 1; i < RAD; ++i) x[i] = ctwid<T>(x[i], __ldg(p.tw_stage + ((m * i) << TW_SHIFT)));
#else
                // Lanes run along c here, so a warp holds 32 / C distinct m: each W_R^(m*i) load is a 2...8-way gather with a
                // stride that grows with i.  Loads for i = 1, 2, 4, ... only, the others by products as above: a few per cent of
                // the whole transform.
                cx<T> w[RAD];
#pragma unroll
                for (int i = 1; i < RAD; ++i) {
                    const int hi = 1 << (31 - __builtin_clz((unsigned)i));
                    if (i == hi) w[i] = __ldg(p.tw_stage + ((m * i) << TW_SHIFT));
                    else w[i] = ctwid<T>(w[hi], w[i - hi]);
                    x[i] = ctwid<T>(x[i], w[i]);
                }
#endif
            }
            DftC<T, RAD>::run(x);
            if constexpr (!LAST) {
#pragma unroll
                for (int k = 0; k < RAD; ++k) tile[Addr::at(base + k * NS, c)] = x[k];
            } else if constexpr (XCH == 1) {
                // last stage of the producing pass of a cluster exchange.  Output row h = m + k*NS of this CTA's column
                // tcol belongs, in the next pass, to CTA h / CB of the cluster, which wants it at [h % CB][tcol] of its tile
                // (the layout its global loads would have read from the workspace).  All tiles of the cluster are still
                // being read by this very stage, so: results stay in registers, cluster barrier, then the scatter.
                // Lanes run along c, so one store instruction writes 32 consecutive elements of one destination row.
                static_assert(TRIPS == 1 && NTASK == NT, "the exchanging stage must be a single trip: one task per thread");
                cluster_sync();
                const unsigned tile_s = (unsigned)__cvta_generic_to_shared(tile);
                const unsigned tcol = (unsigned)out_base + (unsigned)c;     // body() passes the tile's first column in out_base
                const unsigned cb_mask = (1u << p.xch_log2CB) - 1u;
#pragma unroll
                for (int k = 0; k < RAD; ++k) {
                    const unsigned h = (unsigned)(m + k * NS);
                    const unsigned off = ((h & cb_mask) << p.xch_log2P2) + tcol;
                    st_cluster(map_to_rank(tile_s + off * (unsigned)sizeof(cx<T>), h >> p.xch_log2CB), x[k]);
                }
            } else {
                // last stage: g == 0, natural-order outputs kr = m + k*NS
                if (KIND == KIND_ROW && c >= tile_rows_valid) continue;
                if constexpr (XCH == MODE_ROW_BULK) {
                    // natural-order planar staging; the bulk copies at the end of body() take it out
                    T* ore = reinterpret_cast<T*>(reinterpret_cast<unsigned char*>(tile) + OUT_OFF) + c * R + m;
                    T* oim = ore + C * R;
                    const T sc = p.scale;
#pragma unroll
                    for (int k = 0; k < RAD; ++k) { ore[k * NS] = x[k].x * sc; oim[k * NS] = x[k].y * sc; }
                } else
                if constexpr (KIND == KIND_ROW) gstore_n<RAD, OL>(p, out_base + (long long)c * p.out_bstride + m, (long long)NS, x);
                else gstore_n<RAD, OL>(p, out_base + (long long)m * out_kstride + c, (long long)NS * out_kstride, x);
            }
        }
    }

    template <int s>
    static __device__ __forceinline__ void run_stages(const PassParams<T>& p, cx<T>* tile, long long out_base,
                                                      long long out_kstride, int rows_valid, int tid) {
        if constexpr (s < S) {
            __syncthreads();
            if constexpr (s == S - 1) {
                if (p.out_interleaved == 0) stage_from_tile<s, 0>(p, tile, out_base, out_kstride, rows_valid, tid);
                else if (p.out_interleaved == 1) stage_from_tile<s, 1>(p, tile, out_base, out_kstride, rows_valid, tid);
                else stage_from_tile<s, 2>(p, tile, out_base, out_kstride, rows_valid, tid);
            } else {
                stage_from_tile<s>(p, tile, out_base, out_kstride, rows_valid, tid);
            }
            run_stages<s + 1>(p, tile, out_base, out_kstride, rows_valid, tid);
        }
    }

    // ---- the kernel body ------------------------------------------------------------------------
    // `tile_index` is the linear tile id (blockIdx.x for a plain launch; a fused launch loops over tiles).
    // Threads with threadIdx.x >= NT (a fused launch whose other pass needs more threads) take part in
    // the barriers only: their task index starts beyond every task count.
    static __device__ __forceinline__ void body(const PassParams<T>& p, unsigned tile_index) {
        extern __shared__ __align__(128) unsigned char smem_raw[];
        cx<T>* tile = reinterpret_cast<cx<T>*>(smem_raw);
        cx<T>* s_um = tile + TILE_ELEMS;   // [M]       per-CTA  W_L^(kp*B*m')
        cx<T>* s_g = s_um + M;             // [C][R1] or [R1]     W_L^(kp(c)*M*B*i)

        const int tid = (threadIdx.x < NT) ? (int)threadIdx.x : (1 << 28);
        // Programmatic dependent launch (sm_90+): this grid may have been scheduled while the previous
        // pass is still draining; wait for its memory to be visible before touching global data, and
        // let the next pass's CTAs be scheduled as soon as every CTA of this grid is resident.
        // With an asynchronous tile input only the thread that issues the copies waits: the others build the
        // twiddle tables meanwhile and meet the data at the mbarrier (every later access depends on that data).
        if (p.pdl) {
            asm volatile("griddepcontrol.launch_dependents;");
            if constexpr (!ASYNC_IN) asm volatile("griddepcontrol.wait;" ::: "memory");
        }
        long long in_base, out_base, out_kstride;
        long long in_rstride;          // element stride of the tile row index r (COL) / 1 (ROW, TRANS)
        long long in_cstride;          // element stride between tile columns
        int rows_valid = C;
        uint32_t kp0 = 0;              // previous-pass output digit of column c = 0
        uint32_t kp_cstep = 0;         // ... and its increment per column
        uint32_t bcol0 = 0;            // flat index of the remaining digits for column 0 (COL only)
        [[maybe_unused]] long long mbase = 0;   // MODE_C2R_IN(_IL): first input element of this tile's batch member

        if constexpr (KIND == KIND_COL) {
            const int tilesB = 1 << (p.log2B - LOG2C);
            const unsigned blk = tile_index + (unsigned)p.blk_offset;
            const int bt = blk & (tilesB - 1);
            const int rest = blk >> (p.log2B - LOG2C);
            const int a = rest & ((1 << p.log2A) - 1);
            const int batch = rest >> p.log2A;
            const long long off = ((long long)a << (LOG2R + p.log2B)) + ((long long)bt << LOG2C);
            in_base = (long long)batch * p.in_bstride + off;
            if constexpr (C2R_IN) mbase = (long long)batch * p.in_bstride;
            out_base = (long long)(p.out_ring ? (batch & (p.out_ring - 1)) : batch) * p.out_bstride + off;
            in_rstride = 1LL << p.log2B;
            in_cstride = 1;
            out_kstride = in_rstride;
            kp0 = a & ((1u << p.log2Rprev) - 1u);
            bcol0 = (uint32_t)bt << LOG2C;
            if constexpr (XCH == 1) out_base = (long long)bcol0;   // no global output: the last stage wants the tile's first column
        } else if constexpr (KIND == KIND_TRANS) {
            // rows of the tile: a(c) = (k0 + c) * rest_n + rest, rest_n = A / R1
            const int log2restn = p.log2A - p.log2R1;
            const int tilesK = 1 << p.log2_ktn;
            const int kt = p.kt_base + (tile_index & (tilesK - 1));
            const int tmp = tile_index >> p.log2_ktn;
            const int rest = tmp & ((1 << log2restn) - 1);
            const int batch = tmp >> log2restn;
            const int k0 = kt << LOG2C;
            in_base = (long long)(p.in_ring ? (batch & (p.in_ring - 1)) : batch) * p.in_bstride + ((((long long)k0 << log2restn) + rest) << LOG2R);
            in_rstride = 1;
            in_cstride = 1LL << (log2restn + LOG2R);
            // out[(k0 + c) + R1*rest + A*kr]
            out_base = (long long)batch * p.out_bstride + k0 + ((long long)rest << p.log2R1);
            out_kstride = 1LL << p.log2A;
            const uint32_t rprev_mask = (1u << p.log2Rprev) - 1u;
            kp0 = (uint32_t)(((long long)k0 << log2restn) + rest) & rprev_mask;
            kp_cstep = (log2restn == 0) ? 1u : 0u;   // 2-pass plan: kp = k1 = k0 + c ; 3-pass: kp = k2
        } else {
            const long long first = (long long)tile_index * C;
            rows_valid = (int)min((long long)C, (long long)p.batch - first);
            in_base = first * p.in_bstride;
            out_base = first * p.out_bstride;
            in_rstride = 1;
            in_cstride = p.in_bstride;
            out_kstride = 1;
        }

        // ---- asynchronous tile input: thread 0 puts the whole tile in flight --------------------------------------
        [[maybe_unused]] const unsigned mbar = (unsigned)__cvta_generic_to_shared(smem_raw + MBAR_OFF);
        if constexpr (ASYNC_IN) {
            if (tid == 0) {
                mbar_init(mbar, 1);
                if (p.pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
                mbar_expect_tx(mbar, XCH == MODE_ROW_BULK ? (unsigned)(2 * rows_valid * R * sizeof(T)) : (unsigned)(TILE_ELEMS * sizeof(cx<T>)));
                const unsigned tile_s = (unsigned)__cvta_generic_to_shared(tile);
                if constexpr (XCH == MODE_TMA_IN) {
                    // boxes of at most 256 rows.  Planar input: re plane [R][C] then im plane [R][C].  Interleaved input (the
                    // workspace of a 3-pass plan): one map over the pairs, the landing zone is the tile itself, [R][C] complex.
                    constexpr int BOX_ROWS = R < 256 ? R : 256;
                    const int blkq = (int)(tile_index + (unsigned)p.blk_offset);
                    const int col0 = (blkq & ((1 << (p.log2B - LOG2C)) - 1)) << LOG2C;
                    const int bz = blkq >> (p.log2B - LOG2C);          // = a + A * batch: the map's third dimension
                    if (p.in_interleaved) {
#pragma unroll
                        for (int r0 = 0; r0 < R; r0 += BOX_ROWS)
                            tma_load_3d(tile_s + (unsigned)(r0 * C * sizeof(cx<T>)), &p.tmap_re, 2 * col0, r0, bz, mbar);
                    } else {
#pragma unroll
                        for (int r0 = 0; r0 < R; r0 += BOX_ROWS) {
                            tma_load_3d(tile_s + (unsigned)(r0 * C * sizeof(T)), &p.tmap_re, col0, r0, bz, mbar);
                            tma_load_3d(tile_s + (unsigned)((R + r0) * C * sizeof(T)), &p.tmap_im, col0, r0, bz, mbar);
                        }
                    }
                } else if constexpr (XCH == MODE_ROW_BULK) {
                    const unsigned bytes = (unsigned)(rows_valid * R * sizeof(T));
                    bulk_load_1d(tile_s, p.in_re + in_base, bytes, mbar);
                    bulk_load_1d(tile_s + (unsigned)(C * R * sizeof(T)), p.in_im + in_base, bytes, mbar);
                } else {
                    const cx<T>* src = reinterpret_cast<const cx<T>*>(p.in_re) + in_base;
#pragma unroll
                    for (int c = 0; c < C; ++c)
                        bulk_load_1d(tile_s + (unsigned)(c * R * sizeof(cx<T>)), src + (long long)c * in_cstride, (unsigned)(R * sizeof(cx<T>)), mbar);
                }
            }
        }

        // ---- PRELOAD: when every thread owns exactly one stage-1 task, issue its global loads NOW so
        // they are in flight while the twiddle tables below are built (their two-level lookups are two
        // dependent L2 round trips that would otherwise sit in front of the first data load).
        constexpr bool PRELOAD = (M * C <= NT);
        static_assert((XCH != 2 && !ASYNC_IN) || PRELOAD, "a pass that reads its input out of its own tile must do stage 1 in a single trip (every thread holds its task's inputs across the barrier)");
        cx<T> pre[PRELOAD ? R1 : 1];
        if constexpr (PRELOAD) {
            const int t = tid;
            if (t < M * C) {
                int c, mp;
                if constexpr (KIND == KIND_COL) { c = t % C; mp = t / C; } else { mp = t % M; c = t / M; }
                if constexpr (ASYNC_IN) {
                    // filled in below, once the tile has landed
                } else if constexpr (XCH == 2) {
                    // the previous pass's CTAs left this tile as [c][t], t = mp + i*M (what the global loads would have read)
                    const cx<T>* src = tile + c * R + mp;
#pragma unroll
                    for (int i = 0; i < R1; ++i) pre[i] = src[i * M];
                } else if ((KIND != KIND_ROW) || (c < rows_valid)) {
                    const long long a0 = in_base + (long long)c * in_cstride + (long long)mp * in_rstride;
                    gload_n<R1>(p, a0, (long long)M * in_rstride, pre, mbase);
                } else {
#pragma unroll
                    for (int i = 0; i < R1; ++i) pre[i] = make_cx<T>(T(0), T(0));
                }
            }
        }

        // ---- per-CTA inter-pass twiddle factors (two-level lookups, f64, once per CTA) ----------
        // tw(r, c) = W_L^( kp(c) * (r*B + bcol(c)) ),  r = m' + i*M
        //          = W_L^(kp*B*m') * W_L^(kp*bcol) * W_L^(kp*M*B*i)  =  Um[m'] * V[c] * G[c][i]
        cx<T> vreg = make_cx<T>(T(1), T(0));
        const bool has_tw = (KIND != KIND_ROW) && p.has_tw;
        if (has_tw) {
            const int log2B = (KIND == KIND_COL) ? p.log2B : 0;
            for (int mp = tid; mp < M; mp += NT) {
                uint32_t e = (kp0 * (uint32_t)mp) << log2B;
                s_um[mp] = to_cx<T>(p.tw2.get(e << p.tw_shift));
            }
            constexpr int LOG2M = ilog2_c(M);
            for (int q = tid; q < G_ELEMS; q += NT) {
                const int i = q % R1;
                const int c = q / R1;
                uint32_t kp = kp0 + kp_cstep * (uint32_t)c;
                uint32_t e = (kp * (uint32_t)i) << (LOG2M + log2B);
                s_g[q] = to_cx<T>(p.tw2.get(e << p.tw_shift));
            }
            if constexpr (KIND == KIND_COL) {
                const int c = tid % C;   // NT % C == 0: a thread keeps its column for the whole kernel
                uint32_t e = kp0 * (bcol0 + (uint32_t)c);
                vreg = to_cx<T>(p.tw2.get(e << p.tw_shift));
            }
            __syncthreads();
        } else if constexpr (XCH == 2 || ASYNC_IN) {
            __syncthreads();     // every thread has read its inputs out of the exchanged tile before stage 1 overwrites it
        }                        // (asynchronous input: thread 0's mbarrier init is visible to all)
        if constexpr (ASYNC_IN) {
            mbar_wait(mbar, 0);
            const int t = tid;
            if (t < M * C) {
                int c, mp;
                if constexpr (KIND == KIND_COL) { c = t % C; mp = t / C; } else { mp = t % M; c = t / M; }
                if constexpr (XCH == MODE_ROW_BULK) {
                    const T* re_pl = reinterpret_cast<const T*>(tile) + c * R + mp;
                    const T* im_pl = re_pl + C * R;
                    if (c < rows_valid) {
#pragma unroll
                        for (int i = 0; i < R1; ++i) pre[i] = make_cx<T>(re_pl[i * M], im_pl[i * M]);
                    } else {
#pragma unroll
                        for (int i = 0; i < R1; ++i) pre[i] = make_cx<T>(T(0), T(0));
                    }
                } else if constexpr (XCH == MODE_TMA_IN) {
                    if (p.in_interleaved) {
                        const cx<T>* src = tile + mp * C + c;
#pragma unroll
                        for (int i = 0; i < R1; ++i) pre[i] = src[i * M * C];
                    } else {
                        const T* re_pl = reinterpret_cast<const T*>(tile) + mp * C + c;
                        const T* im_pl = re_pl + R * C;
#pragma unroll
                        for (int i = 0; i < R1; ++i) pre[i] = make_cx<T>(re_pl[i * M * C], im_pl[i * M * C]);
                    }
                } else {
                    const cx<T>* src = tile + c * R + mp;
#pragma unroll
                    for (int i = 0; i < R1; ++i) pre[i] = src[i * M];
                }
            }
            __syncthreads();     // the landing zone is free: stage 1 may overwrite it
        }

        // ---- stage 1: global -> registers -> (twiddle, DFT) -> tile (or global when S == 1) ------
        // The input layout is tested once, outside the task loop (see gload_n).
        auto stage1 = [&](auto il_tag) {
            [[maybe_unused]] constexpr int IL = decltype(il_tag)::value;
            constexpr int NTASK = M * C;
            constexpr int TRIPS1 = (NTASK + NT - 1) / NT;
#pragma unroll((VARIANT & 4) ? TRIPS1 : 1)
            for (int t = tid; t < NTASK; t += NT) {
                int c, mp;
                if constexpr (KIND == KIND_COL) { c = t % C; mp = t / C; } else { mp = t % M; c = t / M; }
                cx<T> x[R1];
                [[maybe_unused]] const bool valid = (KIND != KIND_ROW) || (c < rows_valid);
                if constexpr (PRELOAD) {
#pragma unroll
                    for (int i = 0; i < R1; ++i) x[i] = pre[i];
                } else if (valid) {
                    const long long a0 = in_base + (long long)c * in_cstride + (long long)mp * in_rstride;
                    gload_n<R1, IL>(p, a0, (long long)M * in_rstride, x, mbase);
                } else {
#pragma unroll
                    for (int i = 0; i < R1; ++i) x[i] = make_cx<T>(T(0), T(0));
                }
                if (has_tw) {
                    cx<T> pt = s_um[mp];
                    if constexpr (KIND == KIND_COL) {
                        pt = ctwid<T>(pt, vreg);
                    } else {
                        if (kp_cstep) pt = ctwid<T>(pt, __ldg(p.tw_wc + c * M + mp));
                    }
                    const cx<T>* g = (KIND == KIND_TRANS) ? (s_g + c * R1) : s_g;
                    x[0] = ctwid<T>(x[0], pt);
#pragma unroll
                    for (int i = 1; i < R1; ++i) x[i] = ctwid<T>(x[i], ctwid<T>(pt, g[i]));
                }
                DftC<T, R1>::run(x);
                if constexpr (S >= 2) {
                    const int j = rev_tail<RL>(mp);
#pragma unroll
                    for (int k = 0; k < R1; ++k) tile[Addr::at(j * R1 + k, c)] = x[k];
                } else {
                    if (valid) {
                        if constexpr (KIND == KIND_ROW) gstore_n<R1>(p, out_base + (long long)c * p.out_bstride, 1LL, x);
                        else gstore_n<R1>(p, out_base + c, out_kstride, x);
                    }
                }
                // A preloaded task is the thread's only one, but the compiler cannot prove the loop runs once: pre[] then has to
                // outlive x[] across the back edge, and in the 32 x 32 tiles the two 32-value arrays do not fit the registers.
                if constexpr (PRELOAD && STAGE32) break;
            }
        };
        if constexpr (PRELOAD || C2R_IN) stage1(std::integral_constant<int, 0>{});
        else if (p.in_interleaved == 0) stage1(std::integral_constant<int, 0>{});
        else if (p.in_interleaved == 1) stage1(std::integral_constant<int, 1>{});
        else stage1(std::integral_constant<int, 2>{});
        // ---- stages 2..S -------------------------------------------------------------------------
        run_stages<1>(p, tile, out_base, out_kstride, rows_valid, tid);
        if constexpr (XCH == MODE_ROW_BULK) {
            // the staging area was written through the generic proxy: make it visible to the asynchronous proxy, then one thread
            // copies the two planes out and waits until the copies have READ shared memory before the CTA may exit
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
            if (tid == 0) {
                const unsigned stage_s = (unsigned)__cvta_generic_to_shared(smem_raw + OUT_OFF);
                const unsigned bytes = (unsigned)(rows_valid * R * sizeof(T));
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(p.out_re + out_base), "r"(stage_s), "r"(bytes) : "memory");
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(p.out_im + out_base), "r"(stage_s + (unsigned)(C * R * sizeof(T))), "r"(bytes) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            }
        }
    }

};

template <typename T, class RL, int C, int NT, int KIND, int VARIANT = 0, int MINB = 0>
__global__ void __launch_bounds__(NT, MINB) fft_pass_kernel(const __grid_constant__ PassParams<T> p) {
    PassKernel<T, RL, C, NT, KIND, 0, VARIANT>::body(p, blockIdx.x);
}
// the same pass with an asynchronous tile input (MODE_TMA_IN / MODE_BULK_IN)
template <typename T, class RL, int C, int NT, int KIND, int MODE, int VARIANT = 0, int MINB = 0>
__global__ void __launch_bounds__(NT, MINB) fft_pass_async_kernel(const __grid_constant__ PassParams<T> p) {
    PassKernel<T, RL, C, NT, KIND, MODE, VARIANT>::body(p, blockIdx.x);
}

// The table a strided tile's radix-32 last stage reads (stage_from_tile): out[m * 32 + i] = W_R^(m*i), m < R / 32, i < 32, out of
// the pass's W_R table by the product chain that stage computed in registers -- W^(m*i) loaded for i = 1, 2, 4, 8, 16, every other
// i the product of two earlier ones (i = hi + lo, hi its top bit) -- so each entry is bit for bit what the stage used to multiply by.
template <typename T>
__global__ void __launch_bounds__(256) stage32_table_kernel(const cx<T>* __restrict__ tw_stage, cx<T>* __restrict__ out, int ns) {
    const int m = (int)(blockIdx.x * blockDim.x + threadIdx.x);
    if (m >= ns) return;
    cx<T> w[32];
    w[0] = __ldg(tw_stage);
#pragma unroll
    for (int i = 1; i < 32; ++i) {
        const int hi = 1 << (31 - __builtin_clz((unsigned)i));
        if (i == hi) w[i] = __ldg(tw_stage + m * i);
        else w[i] = ctwid<T>(w[hi], w[i - hi]);
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) out[m * 32 + i] = w[i];
}

// ---------------------------------------------------------------------------------------------
// One HBM pass for transforms that fit the shared memory of a thread-block cluster (2^13..2^17 points): the K CTAs of a
// cluster run pass 1 (PK1, KIND_COL, each CTA P2/K adjacent columns of the P1 x P2 view of the signal) out of global
// memory, exchange the intermediate through distributed shared memory (every CTA scatters its results into the tiles of
// the CTAs that own those rows in pass 2 -- the transpose that a two-launch plan does through a global workspace), and
// run pass 2 (PK2, KIND_TRANS, P1/K rows each) out of shared memory into global memory.  HBM sees the signal once in
// and once out; grid = transforms x K, cluster dimension K (launch attribute).
// Replaces, for these sizes, the L1-resident leaf of the reference's recursion (algorithms/dit.rs:27-93).
// ---------------------------------------------------------------------------------------------
template <class PK1, class PK2, typename T, int NT, int MINB>
__global__ void __launch_bounds__(NT, MINB) fft_cluster2_kernel(const __grid_constant__ PassParams<T> p1,
                                                                const __grid_constant__ PassParams<T> p2) {
    PK1::body(p1, blockIdx.x);      // ends with: cluster barrier, scatter into the cluster's tiles
    cluster_sync();                 // every CTA's scatter has landed; nobody writes another CTA's tile after this
    PK2::body(p2, blockIdx.x);
}

// ---------------------------------------------------------------------------------------------
// Both passes of a two-pass plan in ONE persistent launch with the intermediates in an L2-resident ring.
//
// A two-launch plan writes the whole batch's intermediate to HBM and reads it back: 2x the compulsory traffic, which
// caps it at half the roofline however good each pass is (round 1: 4096 x 2^16 f32 at 0.47 with both passes at
// 0.92-0.96).  Here one grid runs both passes at once, its CTAs drawing pass-1 and pass-2 tiles from one ordered ticket queue.
// Pass 1 of transform b writes slot b % ring of a workspace of `ring` transforms (sized to stay in L2, PHASTFT_PIPE_RING_MB),
// pass 2 of transform b reads it back while it is still in L2, and the slot is rewritten (or discarded) before its dirty
// lines are evicted, so HBM sees the batch once in and once out.  Dependencies are per-transform counters:
//     a pass-2 tile of transform b waits for done1[b] == tiles1   (all of its rows have been produced)
//     a pass-1 tile of transform b waits for done2[b - ring] == tiles2   (its slot has been drained)
// released with red.release.gpu after a block barrier and acquired with ld.acquire.gpu by thread 0 before a block barrier.
// With batch == 1 this is a fused two-pass launch of a lone transform (replaces round 1's cooperative-launch + grid-barrier
// experiment).
// ---------------------------------------------------------------------------------------------
struct PipeCtl {
    unsigned* ticket;              // next work item (zeroed before the launch, like done1 / done2)
    unsigned* done1;               // [batch] pass-1 tiles finished per transform
    unsigned* done2;               // [batch] pass-2 tiles finished per transform
    unsigned tiles1, tiles2;       // tiles per transform in pass 1 / pass 2
    unsigned batch, ring, delay;   // ring: workspace slots (transforms), a power of two; pass 2 runs `delay` < ring transforms behind
    int discard;                   // pass 2 tells L2 to drop its input lines once read (discard.global.L2): no write-back of the ring
};
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_gpu(unsigned* p, unsigned v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void wait_count(const unsigned* p, unsigned want) {
    if (threadIdx.x == 0)
        while (ld_acquire_gpu(p) < want) __nanosleep(64);
    __syncthreads();
}

// One CTA = one tile.  The tile is NOT derived from blockIdx: the CTA draws a ticket when it starts running, so tickets are
// held by resident CTAs only and every wait below is for a smaller ticket -- forward progress without assuming anything about
// the order in which the hardware dispatches CTAs (the decoupled-look-back argument).  Ticket order:
//     step s  =  [pass-1 tiles of transform s]  then  [pass-2 tiles of transform s - delay]
// so pass 1 runs `delay` transforms ahead of pass 2 and both kinds of tile are in flight on every SM.  No loop around the
// pass bodies: each keeps (about) the register allocation it has as a kernel of its own.
template <class PK, typename T>
__device__ __forceinline__ void pipe_discard_rows(const PassParams<T>& p, unsigned bq, unsigned kt) {
    // this tile's input rows (C rows of R contiguous interleaved elements each) will not be read again: let L2 drop them
    constexpr int LINES_PER_ROW = (int)(PK::R * sizeof(cx<T>) / 128);
    const char* rows = reinterpret_cast<const char*>(reinterpret_cast<const cx<T>*>(p.in_re) + (long long)bq * p.in_bstride +
                                                     (long long)kt * PK::TILE_C * PK::R);
    for (int q = threadIdx.x; q < PK::TILE_C * LINES_PER_ROW; q += blockDim.x)
        asm volatile("discard.global.L2 [%0], 128;" ::"l"(rows + (size_t)q * 128) : "memory");
}

template <class PK1, class PK2, typename T, int NTF, int MINB>
__global__ void __launch_bounds__(NTF, MINB) fft_pipe2_kernel(const __grid_constant__ PassParams<T> p1,
                                                             const __grid_constant__ PassParams<T> p2,
                                                             const __grid_constant__ PipeCtl c) {
    __shared__ unsigned s_ticket;
    if (threadIdx.x == 0) s_ticket = atomicAdd(c.ticket, 1u);
    __syncthreads();
    const unsigned t = s_ticket;
    const unsigned L = c.tiles1 + c.tiles2;
    const unsigned step = t / L, j = t - step * L;
    if (j < c.tiles1) {
        if (step >= c.batch) return;
        if (step >= c.ring) wait_count(c.done2 + (step - c.ring), c.tiles2);          // the slot has been drained
        PK1::body(p1, step * c.tiles1 + j);
        __syncthreads();
        if (threadIdx.x == 0) red_release_gpu(c.done1 + step, 1u);
    } else {
        if (step < c.delay || step - c.delay >= c.batch) return;
        const unsigned b = step - c.delay, kt = j - c.tiles1;
        wait_count(c.done1 + b, c.tiles1);                                             // all rows of the transform have been produced
        PK2::body(p2, b * c.tiles2 + kt);
        __syncthreads();
        if (c.discard) { pipe_discard_rows<PK2, T>(p2, b & (c.ring - 1), kt); __syncthreads(); }
        if (threadIdx.x == 0) red_release_gpu(c.done2 + b, 1u);
    }
}

// ---------------------------------------------------------------------------------------------
// r2c post-processing (reference: simd_untangle_inplace_*, algorithms/r2c.rs:150-242) and c2r
// pre-processing (simd_c2r_preprocess_*, r2c.rs:263-432).  Elementwise over bin pairs (k, half-k).
// The planner's w[k] = 0.5 * W_N^k table (planner.rs:120-162, an O(N) rotation recurrence on the
// CPU) is replaced by a two-level lookup: consecutive k hit consecutive `lo` entries (coalesced)
// and one broadcast `hi` entry.
// ---------------------------------------------------------------------------------------------
// A member's spectrum bins: planar (re[k], im[k]), or SIL: Complex<T> values at re (im unused), as the interleaved real
// transforms (phastft_{r2c,c2r}_interleaved_any_*) hold them.  One complex value per access: an interleaved f32 member may start
// at an odd complex offset, so it is only 8-byte aligned.
template <typename T, bool SIL>
struct SpecBins {
    T* re;
    T* im;
    __device__ __forceinline__ cx<T> get(long long k) const {
        if constexpr (SIL) return reinterpret_cast<const cx<T>*>(re)[k];
        else return make_cx<T>(re[k], im[k]);
    }
    __device__ __forceinline__ void put(long long k, T x, T y) const {
        if constexpr (SIL) reinterpret_cast<cx<T>*>(re)[k] = make_cx<T>(x, y);
        else { re[k] = x; im[k] = y; }
    }
};
// the bins of the member `off` bins in (planar: elements of each array; SIL: complex values)
template <typename T, bool SIL>
__device__ __forceinline__ SpecBins<T, SIL> spec_at(const T* re, const T* im, long long off) {
    if constexpr (SIL) return {const_cast<T*>(reinterpret_cast<const T*>(reinterpret_cast<const cx<T>*>(re) + off)), nullptr};
    else return {const_cast<T*>(re + off), const_cast<T*>(im + off)};
}

template <typename T>
struct RealParams {
    T* __restrict__ re;         // untangle: in/out (length half+1).  preprocess: z_re out (length half)
    T* __restrict__ im;
    const T* __restrict__ in_re;  // preprocess only: spectrum (length half+1)
    const T* __restrict__ in_im;
    long long bstride;          // elements between batch members in re/im (the interleaved untangle: complex values)
    long long in_bstride;       // (the interleaved preprocess: complex values)
    int log2half;
    unsigned blocks_per_member; // the grid is members x blocks_per_member blocks, member-major
    Tw2 tw2;                    // two-level table for W_N, N = 2*half
};

// SIL: the bins are interleaved (R2C-UNTANGLE-IL)
template <typename T, bool SIL = false>
__global__ void __launch_bounds__(256) r2c_untangle_kernel(const __grid_constant__ RealParams<T> p) {
    const long long half = 1LL << p.log2half;
    const long long q = half >> 1;
    const unsigned mb = blockIdx.x / p.blocks_per_member;
    const long long k = (long long)(blockIdx.x - mb * p.blocks_per_member) * blockDim.x + threadIdx.x;
    const SpecBins<T, SIL> y = spec_at<T, SIL>(p.re, p.im, (long long)mb * p.bstride);
    if (k > q) return;
    if (k == 0) {
        // r2c.rs:161-166
        const cx<T> z0 = y.get(0);
        T a0 = z0.x, b0 = z0.y;
        y.put(0, a0 + b0, T(0));
        y.put(half, a0 - b0, T(0));
        return;
    }
    double2 wd = p.tw2.get((uint32_t)k);
    const T wkr = T(0.5 * wd.x), wki = T(0.5 * wd.y);
    if (k == q) {
        // r2c.rs:233-236 (self pair)
        const cx<T> zq = y.get(q);
        T a = zq.x, b = zq.y;
        y.put(q, a + T(2) * wkr * b, T(2) * wki * b);
        return;
    }
    const long long m = half - k;
    const cx<T> zk = y.get(k), zm = y.get(m);
    T a = zk.x, b = zk.y, c = zm.x, d = zm.y;
    T s_re = T(0.5) * (a + c), s_im = T(0.5) * (b - d);
    T t_re = b + d, t_im = c - a;
    T wzr = wkr * t_re - wki * t_im;
    T wzi = wkr * t_im + wki * t_re;
    y.put(k, s_re + wzr, s_im + wzi);
    y.put(m, s_re - wzr, wzi - s_im);
}

// SIL: the spectrum is interleaved (C2R-PRE-IL); z stays planar
template <typename T, bool SIL = false>
__global__ void __launch_bounds__(256) c2r_preprocess_kernel(const __grid_constant__ RealParams<T> p) {
    const long long half = 1LL << p.log2half;
    const unsigned mb = blockIdx.x / p.blocks_per_member;
    const long long k = (long long)(blockIdx.x - mb * p.blocks_per_member) * blockDim.x + threadIdx.x;
    if (k >= half) return;
    const SpecBins<T, SIL> x = spec_at<T, SIL>(p.in_re, p.in_im, (long long)mb * p.in_bstride);
    T* zre = p.re + (long long)mb * p.bstride;
    T* zim = p.im + (long long)mb * p.bstride;
    const long long m = half - k;
    double2 wd = p.tw2.get((uint32_t)k);
    const T c_h = T(0.5 * wd.x), s_h = T(0.5 * wd.y);
    // r2c.rs:263-347
    const cx<T> xf = x.get(k), xs = x.get(m);
    T re_f = xf.x, im_f = xf.y;
    T re_s = xs.x, im_s = -xs.y;
    T zx_re = T(0.5) * (re_f + re_s), zx_im = T(0.5) * (im_f + im_s);
    T dr = re_f - re_s, di = im_f - im_s;
    T zy_re = c_h * dr + s_h * di;
    T zy_im = c_h * di - s_h * dr;
    zre[k] = zx_re - zy_im;
    zim[k] = zx_im + zy_re;
}

// ---------------------------------------------------------------------------------------------
// Bluestein's chirp-z algorithm (any N, phastft_fft_any_*): X[k] = w[k] sum_n (x[n] w[n]) conj(w[k-n]), w[j] =
// exp(-pi i (j^2 mod 2N) / N), a circular convolution of length M = 2^ceil(log2(2N - 1)) done with two forward M-point
// transforms in place on an interleaved workspace of M complex values per member:
//   CHIRP-PRE   a[m] = x[m] w[m] (m < N), 0 (N <= m < M)
//   CHIRP-MUL   A[k] <- conj(A[k] Bh[k]),  Bh = FFT_M(b) / M,  b[m] = conj(w[|m|]) on the circle
//   CHIRP-POST  X[k] = scale * w[k] conj(C[k]) (k < N)
// (the conjugation makes the second forward transform an inverse one: ifft(Y) = conj(fft(conj Y)) / M).  Each thread moves 16
// bytes of the interleaved side (one complex f64, two complex f32) in one access; grids are member-major like the r2c ones.
// ---------------------------------------------------------------------------------------------
template <typename T> struct Cx16;
template <> struct Cx16<double> {
    static constexpr int V = 1;
    using vec = double2;
    __device__ static void unpack(const double2& q, double2* c) { c[0] = q; }
    __device__ static double2 pack(const double2* c) { return c[0]; }
};
template <> struct Cx16<float> {
    static constexpr int V = 2;
    using vec = float4;
    __device__ static void unpack(const float4& q, float2* c) { c[0] = make_float2(q.x, q.y); c[1] = make_float2(q.z, q.w); }
    __device__ static float4 pack(const float2* c) { return make_float4(c[0].x, c[0].y, c[1].x, c[1].y); }
};

template <typename T>
struct ChirpParams {
    const T* in_re;                // CHIRP-PRE: the caller's planar input (re / im swapped for the reverse direction); the
    const T* in_im;                // interleaved modes read Complex<T> values from in_re (in_im unused)
    T* out_re;                     // CHIRP-POST: the caller's planar output (swapped like the input), or interleaved as in_re
    T* out_im;
    cx<T>* ws;                     // members x M interleaved complex
    const cx<T>* chirp;            // w[0 .. N), padded with zeros to a multiple of Cx16<T>::V
    const cx<T>* bhat;             // FFT_M(b) / M
    long long bstride;             // elements between members of the caller's arrays
    long long n;
    int log2m;
    unsigned blocks_per_member;    // the grid is members x blocks_per_member blocks, member-major
    T scale;                       // CHIRP-POST: 1 forward, 1/N reverse
    long long out_bstride;         // real modes: elements between members of the output arrays (bstride is the input's)
    const cx<T>* wn;               // halved modes: W_(2n)^k for k = 0 .. n/2
};

// What CHIRP-PRE reads and CHIRP-POST writes around the convolution (n above is the Bluestein length L):
//   C2C          planar complex in, planar complex out (phastft_fft_any_*)
//   R2C_HALVED   even N = 2L: z[m] = x[2m] + i x[2m+1] in; the untangle of Z = DFT_L(z) with W_N^k out, bins 0 .. L
//   R2C_DIRECT   odd N = L: real x in; bins 0 .. floor(N/2) out
//   C2R_HALVED   bins 0 .. L in, the c2r pre-processing with W_N^m (swapped); the pairs (y[2k], y[2k+1]) out
//   C2R_DIRECT   bins 0 .. floor(N/2) in, the Hermitian extension (swapped); the real part of the inverse out
//   C2C_IL       interleaved complex in and out (phastft_fft_interleaved_any_*), the forward direction
//   C2C_IL_SWAP  the same for the reverse direction: re / im swapped on load and on store, as the planar call swaps its pointers
//   R2C_HALVED_IL, R2C_DIRECT_IL, C2R_HALVED_IL, C2R_DIRECT_IL  the real modes with the spectrum as interleaved Complex<T> bins
//                (phastft_{r2c,c2r}_interleaved_any_*): only the spectrum's end runs them (CHIRP-POST of r2c, CHIRP-PRE of c2r);
//                the real side runs the planar mode's kernel
enum ChirpMode { CHIRP_C2C, CHIRP_R2C_HALVED, CHIRP_R2C_DIRECT, CHIRP_C2R_HALVED, CHIRP_C2R_DIRECT, CHIRP_C2C_IL, CHIRP_C2C_IL_SWAP,
                 CHIRP_R2C_HALVED_IL, CHIRP_R2C_DIRECT_IL, CHIRP_C2R_HALVED_IL, CHIRP_C2R_DIRECT_IL };

// a real mode with an interleaved spectrum, and the planar mode whose arithmetic it runs (the mode itself for the others)
template <int MODE>
__host__ __device__ constexpr bool chirp_spec_il() { return MODE >= CHIRP_R2C_HALVED_IL; }
template <int MODE>
__host__ __device__ constexpr int chirp_planar() {
    return MODE == CHIRP_R2C_HALVED_IL ? CHIRP_R2C_HALVED : MODE == CHIRP_R2C_DIRECT_IL ? CHIRP_R2C_DIRECT
         : MODE == CHIRP_C2R_HALVED_IL ? CHIRP_C2R_HALVED : MODE == CHIRP_C2R_DIRECT_IL ? CHIRP_C2R_DIRECT : MODE;
}

// The interleaved modes' ends.  The swap is part of the mode, so no kernel carries a runtime test for it.  The caller's array is
// accessed one complex value at a time: a member starts at any complex offset, so f32 members are only 8-byte aligned.
template <int MODE>
__host__ __device__ constexpr bool chirp_il() { return MODE == CHIRP_C2C_IL || MODE == CHIRP_C2C_IL_SWAP; }
template <typename T, int MODE>
__device__ __forceinline__ cx<T> il_load(const cx<T>& v) {
    if constexpr (MODE == CHIRP_C2C_IL_SWAP) return make_cx<T>(v.y, v.x);
    else return v;
}
// the planar call's two stores re = v.x * scale, im = v.y * scale (swapped pointers for the reverse direction) as one
template <typename T, int MODE>
__device__ __forceinline__ cx<T> il_store(const cx<T>& v, T scale) {
    if constexpr (MODE == CHIRP_C2C_IL_SWAP) return make_cx<T>(v.y * scale, v.x * scale);
    else return make_cx<T>(v.x * scale, v.y * scale);
}

// CHIRP-POST's items per member: values, or bin pairs (k, L - k) for R2C_HALVED
template <int MODE>
__host__ __device__ constexpr long long chirp_post_count(long long n) {
    return chirp_planar<MODE>() == CHIRP_R2C_HALVED || chirp_planar<MODE>() == CHIRP_R2C_DIRECT ? n / 2 + 1 : n;
}

// W_N^k for 0 <= k < L, N = 2L, from the table of k <= L/2: W_N^k = -conj(W_N^(L-k))
template <typename T>
__device__ __forceinline__ cx<T> chirp_wn(const ChirpParams<T>& p, long long k) {
    if (2 * k <= p.n) return p.wn[k];
    const cx<T> w = p.wn[p.n - k];
    return make_cx<T>(-w.x, w.y);
}

// The real modes' arithmetic at the two ends, shared by the Bluestein (CHIRP-*) and mixed-radix (SMOOTH-* / ODD) kernels.
// c2r_preprocess_kernel's formula with w = W_N^m, L = N/2 bins x: z = (X[m] + conj X[L-m]) / 2 +
// i conj(w) (X[m] - conj X[L-m]) / 2, swapped for the inverse
template <typename T, bool SIL>
__device__ __forceinline__ cx<T> c2r_halved_in(const SpecBins<T, SIL>& x, long long l, long long m, cx<T> w) {
    const long long s = l - m;
    const T c_h = T(0.5) * w.x, s_h = T(0.5) * w.y;
    const cx<T> xf = x.get(m), xs = x.get(s);
    const T re_f = xf.x, im_f = xf.y, re_s = xs.x, im_s = -xs.y;
    const T zx_re = T(0.5) * (re_f + re_s), zx_im = T(0.5) * (im_f + im_s);
    const T dr = re_f - re_s, di = im_f - im_s;
    const T zy_re = c_h * dr + s_h * di;
    const T zy_im = c_h * di - s_h * dr;
    return make_cx<T>(zx_im + zy_re, zx_re - zy_im);
}
// odd N: the Hermitian extension Y[m] = X[m] (m <= N/2) or conj X[N - m], swapped
template <typename T, bool SIL>
__device__ __forceinline__ cx<T> c2r_direct_in(const SpecBins<T, SIL>& x, long long n, long long m) {
    if constexpr (SIL) {
        const cx<T> v = x.get(2 * m <= n ? m : n - m);
        return 2 * m <= n ? make_cx<T>(v.y, v.x) : make_cx<T>(-v.y, v.x);
    } else {
        return 2 * m <= n ? make_cx<T>(x.im[m], x.re[m]) : make_cx<T>(-x.im[n - m], x.re[n - m]);
    }
}
// r2c_untangle_kernel's formula for the bin pair (k, L - k) of Z = DFT_L(z), w = W_N^k: X[k] and X[L - k]
template <typename T>
__device__ __forceinline__ void r2c_untangle(cx<T> zk, cx<T> zm, cx<T> w, cx<T>& xk, cx<T>& xm) {
    const T wkr = T(0.5) * w.x, wki = T(0.5) * w.y;
    const T a = zk.x, b = zk.y, cc = zm.x, d = zm.y;
    const T s_re = T(0.5) * (a + cc), s_im = T(0.5) * (b - d);
    const T t_re = b + d, t_im = cc - a;
    const T wzr = wkr * t_re - wki * t_im;
    const T wzi = wkr * t_im + wki * t_re;
    xk = make_cx<T>(s_re + wzr, s_im + wzi);
    xm = make_cx<T>(s_re - wzr, wzi - s_im);
}

// CHIRP-PRE's value before the chirp product, real modes: member mb's element m < L
template <typename T, int MODE>
__device__ __forceinline__ cx<T> chirp_real_in(const ChirpParams<T>& p, unsigned mb, long long m) {
    constexpr int PM = chirp_planar<MODE>();
    const T* re = p.in_re + (long long)mb * p.bstride;
    if constexpr (PM == CHIRP_R2C_HALVED) {
        return reinterpret_cast<const cx<T>*>(re)[m];                   // (x[2m], x[2m+1]): base and stride keep pairs aligned
    } else {
        // bstride counts T either way: the interleaved spectrum's member starts at re
        const SpecBins<T, chirp_spec_il<MODE>()> x = spec_at<T, chirp_spec_il<MODE>()>(re, p.in_im + (long long)mb * p.bstride, 0);
        if constexpr (PM == CHIRP_C2R_HALVED) return c2r_halved_in<T>(x, p.n, m, chirp_wn(p, m));
        else return c2r_direct_in<T>(x, p.n, m);
    }
}

// index of this thread's first complex value in its member, and the member
template <typename T>
__device__ __forceinline__ long long chirp_index(const ChirpParams<T>& p, unsigned& mb) {
    mb = blockIdx.x / p.blocks_per_member;
    return ((long long)(blockIdx.x - mb * p.blocks_per_member) * blockDim.x + threadIdx.x) * Cx16<T>::V;
}

template <typename T, int MODE = CHIRP_C2C>
__global__ void __launch_bounds__(256) chirp_pre_kernel(const __grid_constant__ ChirpParams<T> p) {
    using P = Cx16<T>;
    unsigned mb;
    const long long m0 = chirp_index(p, mb);
    const long long M = 1LL << p.log2m;
    if (m0 >= M) return;
    cx<T> a[P::V];
    if (m0 < p.n) {
        cx<T> w[P::V];
        P::unpack(reinterpret_cast<const typename P::vec*>(p.chirp)[m0 / P::V], w);
        if constexpr (MODE == CHIRP_C2C) {
            const T* re = p.in_re + (long long)mb * p.bstride;
            const T* im = p.in_im + (long long)mb * p.bstride;
#pragma unroll
            for (int j = 0; j < P::V; ++j)
                a[j] = m0 + j < p.n ? cmul<T>(make_cx<T>(re[m0 + j], im[m0 + j]), w[j]) : make_cx<T>(T(0), T(0));
        } else if constexpr (chirp_planar<MODE>() == CHIRP_R2C_DIRECT) {
            const T* re = p.in_re + (long long)mb * p.bstride;            // real x complex: any element offset is legal
#pragma unroll
            for (int j = 0; j < P::V; ++j) {
                const T x = m0 + j < p.n ? re[m0 + j] : T(0);
                a[j] = make_cx<T>(x * w[j].x, x * w[j].y);
            }
        } else if constexpr (chirp_il<MODE>()) {
            const cx<T>* x = reinterpret_cast<const cx<T>*>(p.in_re + (long long)mb * p.bstride);
#pragma unroll
            for (int j = 0; j < P::V; ++j)
                a[j] = m0 + j < p.n ? cmul<T>(il_load<T, MODE>(x[m0 + j]), w[j]) : make_cx<T>(T(0), T(0));
        } else {
#pragma unroll
            for (int j = 0; j < P::V; ++j)
                a[j] = m0 + j < p.n ? cmul<T>(chirp_real_in<T, MODE>(p, mb, m0 + j), w[j]) : make_cx<T>(T(0), T(0));
        }
    } else {
#pragma unroll
        for (int j = 0; j < P::V; ++j) a[j] = make_cx<T>(T(0), T(0));
    }
    reinterpret_cast<typename P::vec*>(p.ws + ((long long)mb << p.log2m))[m0 / P::V] = P::pack(a);
}

template <typename T>
__global__ void __launch_bounds__(256) chirp_mul_kernel(const __grid_constant__ ChirpParams<T> p) {
    using P = Cx16<T>;
    unsigned mb;
    const long long k0 = chirp_index(p, mb);
    if (k0 >= (1LL << p.log2m)) return;
    typename P::vec* ws = reinterpret_cast<typename P::vec*>(p.ws + ((long long)mb << p.log2m)) + k0 / P::V;
    cx<T> a[P::V], b[P::V];
    P::unpack(*ws, a);
    P::unpack(reinterpret_cast<const typename P::vec*>(p.bhat)[k0 / P::V], b);
#pragma unroll
    for (int j = 0; j < P::V; ++j) {
        const cx<T> y = cmul<T>(a[j], b[j]);
        a[j] = make_cx<T>(y.x, -y.y);
    }
    *ws = P::pack(a);
}

template <typename T, int MODE = CHIRP_C2C>
__global__ void __launch_bounds__(256) chirp_post_kernel(const __grid_constant__ ChirpParams<T> p) {
    using P = Cx16<T>;
    unsigned mb;
    const long long k0 = chirp_index(p, mb);
    const long long count = chirp_post_count<MODE>(p.n);
    if (k0 >= count) return;
    const cx<T>* ws = p.ws + ((long long)mb << p.log2m);
    cx<T> c[P::V], w[P::V];
    P::unpack(reinterpret_cast<const typename P::vec*>(ws)[k0 / P::V], c);
    P::unpack(reinterpret_cast<const typename P::vec*>(p.chirp)[k0 / P::V], w);
    if constexpr (MODE == CHIRP_C2C) {
        T* re = p.out_re + (long long)mb * p.bstride;
        T* im = p.out_im + (long long)mb * p.bstride;
#pragma unroll
        for (int j = 0; j < P::V; ++j) {
            if (k0 + j >= p.n) break;
            const cx<T> x = cmul<T>(w[j], make_cx<T>(c[j].x, -c[j].y));
            re[k0 + j] = x.x * p.scale;
            im[k0 + j] = x.y * p.scale;
        }
    } else if constexpr (chirp_il<MODE>()) {
        cx<T>* y = reinterpret_cast<cx<T>*>(p.out_re + (long long)mb * p.out_bstride);
#pragma unroll
        for (int j = 0; j < P::V; ++j) {
            if (k0 + j >= p.n) break;
            y[k0 + j] = il_store<T, MODE>(cmul<T>(w[j], make_cx<T>(c[j].x, -c[j].y)), p.scale);
        }
    } else if constexpr (chirp_planar<MODE>() == CHIRP_R2C_HALVED) {
        // bin pair (k, L - k): Z[k] = w[k] conj C[k] and Z[L - k] (Z[L] = Z[0]), then r2c_untangle_kernel's formula with W_N^k;
        // k = 0 gives X[0] and X[L] = X[N/2], k = L/2 (L even) is the self pair.  The mirrored reads are one value each.
        // out_bstride counts T either way.
        const SpecBins<T, chirp_spec_il<MODE>()> y =
            spec_at<T, chirp_spec_il<MODE>()>(p.out_re + (long long)mb * p.out_bstride, p.out_im + (long long)mb * p.out_bstride, 0);
#pragma unroll
        for (int j = 0; j < P::V; ++j) {
            const long long k = k0 + j;
            if (k >= count) break;
            const long long m = p.n - k, mm = k ? m : 0;
            const cx<T> zk = cmul<T>(w[j], make_cx<T>(c[j].x, -c[j].y));
            const cx<T> cm = ws[mm], wm = p.chirp[mm];
            const cx<T> zm = cmul<T>(wm, make_cx<T>(cm.x, -cm.y));
            cx<T> xk, xm;
            r2c_untangle<T>(zk, zm, p.wn[k], xk, xm);
            y.put(k, xk.x, xk.y);
            if (m != k) y.put(m, xm.x, xm.y);
        }
    } else if constexpr (chirp_planar<MODE>() == CHIRP_R2C_DIRECT) {
        const SpecBins<T, chirp_spec_il<MODE>()> y =
            spec_at<T, chirp_spec_il<MODE>()>(p.out_re + (long long)mb * p.out_bstride, p.out_im + (long long)mb * p.out_bstride, 0);
#pragma unroll
        for (int j = 0; j < P::V; ++j) {
            if (k0 + j >= count) break;
            const cx<T> x = cmul<T>(w[j], make_cx<T>(c[j].x, -c[j].y));
            y.put(k0 + j, x.x, x.y);
        }
    } else if constexpr (MODE == CHIRP_C2R_HALVED) {
        // y = swap(w conj C) / L, the pair (y[2k], y[2k+1]): one aligned 2 * sizeof(T) store
        cx<T>* y = reinterpret_cast<cx<T>*>(p.out_re + (long long)mb * p.out_bstride);
#pragma unroll
        for (int j = 0; j < P::V; ++j) {
            if (k0 + j >= count) break;
            const cx<T> x = cmul<T>(w[j], make_cx<T>(c[j].x, -c[j].y));
            y[k0 + j] = make_cx<T>(x.y * p.scale, x.x * p.scale);
        }
    } else {
        // the real part of the inverse: the imaginary part of w conj C before the swap, / N
        T* y = p.out_re + (long long)mb * p.out_bstride;
#pragma unroll
        for (int j = 0; j < P::V; ++j) {
            if (k0 + j >= count) break;
            const cx<T> x = cmul<T>(w[j], make_cx<T>(c[j].x, -c[j].y));
            y[k0 + j] = x.y * p.scale;
        }
    }
}

// Plan time, f32 plans: Bh rounded to T from its f64 transform.
template <typename T>
__global__ void __launch_bounds__(256) chirp_narrow_kernel(const double2* __restrict__ in, cx<T>* __restrict__ out, long long count) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (long long)gridDim.x * blockDim.x)
        out[i] = make_cx<T>((T)in[i].x, (T)in[i].y);
}

// ---------------------------------------------------------------------------------------------
// Mixed radix (N = P * Q, P = 2^a, Q = 3^b 5^c 7^d > 1; phastft_fft_any_* with PHASTFT_ANY_MIXED): with n = n_o + Q n_2 and
// k = k_2 + P k_o,  X[k_2 + P k_o] = sum_(n_o) W_Q^(n_o k_o) W_N^(n_o k_2) Y_(n_o)[k_2],  Y_(n_o) = DFT_P(x[n_o + Q n_2]).
//   SMOOTH-PRE  planar x -> workspace member n_o (P interleaved points), a tiled transpose by Q
//   the P-point plan on Q * batch interleaved members in place
//   ODD         Q <= ODD_MAX_ROWS: one pass, W_N^(n_o k_2) on load, the Q-point DFT down the member axis, planar store.
//               Otherwise Q = Q_a Q_b, n_o = n_a Q_b + n_b, k_o = k_a + Q_a k_b: pass A (W_N^(n_o k_2) on load, n_a -> k_a in place
//               in the workspace, rows Q_b P apart), pass B (W_Q^(n_b k_a) on load, n_b -> k_b, planar store of row k_a + Q_a k_b).
// Every pass is "R rows, N / R columns per member": column c of member m reads rows r at in0 + r * in_rs, multiplies by
// W_N^(e0 + r * de) and writes row k at c + k * out_rs.
// The real any-length plan runs the same kernels with a ChirpMode at both ends (N below is the mixed length: L = N_real / 2
// for the halved modes, N_real for the direct ones): SMOOTH-PRE loads what CHIRP-PRE would (the pairs, the real data, the c2r
// pre-processing with W_(2L)^m, the Hermitian extension), the last ODD pass stores the pairs, the real part or the bins up to
// floor(N/2), and the halved r2c untangles the bins in place afterwards (SMOOTH-POST-R2C).  The interleaved complex modes
// (C2C_IL, C2C_IL_SWAP) load and store Complex<T> values of the caller's array instead of planar ones.  Pass A is always C2C.
// ---------------------------------------------------------------------------------------------
enum OddRole { ODD_SINGLE, ODD_A, ODD_B };
constexpr int ODD_MAX_STAGES = 6;      // 3^6 = 729
constexpr int ODD_MAX_ROWS = 729;      // the largest tile: 729 rows x 128 bytes = 91 KiB, two CTAs per SM
constexpr int ODD_NT = 256;

template <typename T>
struct OddParams {
    const cx<T>* ws;               // batch x N interleaved: every pass reads it, pass A writes it
    cx<T>* ws_out;
    T* out_re;                     // the last pass: the caller's planar arrays (re / im swapped for the reverse direction), or
    T* out_im;                     // its interleaved array in out_re
    const cx<T>* wn_hi;            // W_N^(j << lo_bits)
    const cx<T>* wn_lo;            // W_N^j, j < 2^lo_bits
    const cx<T>* wr;               // W_R^j, j < R: the twiddles between the stages of this pass
    const unsigned short* perm;    // tile kernel: where stage 1 puts the butterfly of row r < R / rad[0] (digit reversal)
    long long n, p, cols, total;   // N, P, columns per member (N / R), batch * cols
    long long in_rs, out_rs;       // elements between rows
    long long bstride;             // elements between members of the caller's arrays (complex values for C2R_HALVED, C2C_IL* and
                                   // R2C_DIRECT_IL)
    int role, r, qb, lo_bits;
    int nstages, rad[ODD_MAX_STAGES];
    int cw;                        // tile kernel: columns per CTA
    T scale;                       // the last pass: 1 forward, 1/N reverse
};

// One column of a pass: where its rows are, its twiddle exponents and where its output rows go.  MODE: how the last pass
// stores (C2C for pass A).
template <typename T, int MODE = CHIRP_C2C>
struct OddCol {
    const cx<T>* in;
    cx<T>* out_c;
    T* out_re;
    T* out_im;
    cx<T>* out_y;                      // C2R_HALVED: the caller's real array as pairs (bstride counts pairs); C2C_IL*: its
                                       // interleaved array; R2C_DIRECT_IL: its interleaved bins
    int kmax;                          // R2C_DIRECT: the last row whose output index c + k out_rs is a stored bin (<= N/2)
    unsigned long long e0, de;
    __device__ __forceinline__ OddCol(const OddParams<T>& p, long long g) {
        const long long m = g / p.cols, c = g - m * p.cols;
        const long long hi = p.role == ODD_SINGLE ? 0 : c / p.p, lo = c - hi * p.p;
        in = p.ws + m * p.n + (p.role == ODD_B ? hi * p.qb * p.p + lo : c);
        e0 = p.role == ODD_A ? hi * lo : 0;
        de = p.role == ODD_SINGLE ? lo : p.role == ODD_A ? p.qb * lo : hi * p.p;
        out_c = p.ws_out + m * p.n + c;
        out_re = p.out_re + m * p.bstride + c;
        out_im = p.out_im + m * p.bstride + c;
        if constexpr (MODE == CHIRP_C2R_HALVED || chirp_il<MODE>() || MODE == CHIRP_R2C_DIRECT_IL)
            out_y = reinterpret_cast<cx<T>*>(p.out_re) + m * p.bstride + c;
        if constexpr (chirp_planar<MODE>() == CHIRP_R2C_DIRECT) kmax = (int)((p.n / 2 - c) / p.out_rs);      // c < N / 3 on the last pass
    }
    // row r, times W_N^(e0 + r de)
    __device__ __forceinline__ cx<T> load(const OddParams<T>& p, int r) const {
        const cx<T> v = in[r * p.in_rs];
        const unsigned long long e = e0 + r * de;
        if (e == 0) return v;
        const cx<T> w = cmul<T>(__ldg(p.wn_hi + (e >> p.lo_bits)), __ldg(p.wn_lo + (e & ((1ull << p.lo_bits) - 1))));
        return ctwid<T>(v, w);
    }
    __device__ __forceinline__ void store(const OddParams<T>& p, int k, const cx<T>& v) const {
        if (p.role == ODD_A) {
            out_c[k * p.out_rs] = v;
        } else if constexpr (MODE == CHIRP_C2R_HALVED) {
            out_y[k * p.out_rs] = make_cx<T>(v.y * p.scale, v.x * p.scale);      // (y[2K], y[2K+1]) = swap(v) / L
        } else if constexpr (MODE == CHIRP_C2R_DIRECT) {
            out_re[k * p.out_rs] = v.y * p.scale;                               // the real part of the inverse, / N
        } else if constexpr (chirp_il<MODE>()) {
            out_y[k * p.out_rs] = il_store<T, MODE>(v, p.scale);
        } else if constexpr (MODE == CHIRP_R2C_DIRECT_IL) {
            if (k > kmax) return;                                               // bins 0 .. floor(N/2) only, as R2C_DIRECT
            out_y[k * p.out_rs] = il_store<T, MODE>(v, p.scale);
        } else {
            // R2C_DIRECT: the caller holds bins 0 .. floor(N/2) only
            if (MODE == CHIRP_R2C_DIRECT && k > kmax) return;
            out_re[k * p.out_rs] = v.x * p.scale;
            out_im[k * p.out_rs] = v.y * p.scale;
        }
    }
};

// R = RA * RB rows (RB = 1: one register DFT) held by one thread: no shared memory, a block covers ODD_NT adjacent columns.
template <typename T, int RA, int RB, int MODE = CHIRP_C2C>
__global__ void __launch_bounds__(ODD_NT, MODE == CHIRP_C2R_DIRECT ? 1 : 0) odd_reg_kernel(const __grid_constant__ OddParams<T> p) {
    constexpr int R = RA * RB;
    const long long g = (long long)blockIdx.x * ODD_NT + threadIdx.x;
    if (g >= p.total) return;
    const OddCol<T, MODE> col(p, g);
    cx<T> x[R];
#pragma unroll
    for (int r = 0; r < R; ++r) x[r] = col.load(p, r);
    if constexpr (RB == 1) {
        DftC<T, RA>::run(x);
#pragma unroll
        for (int k = 0; k < R; ++k) col.store(p, k, x[k]);
    } else {
        // n = n_a RB + n_b, k = k_a + RA k_b: DFT_RA over n_a, W_R^(n_b k_a), DFT_RB over n_b
#pragma unroll
        for (int nb = 0; nb < RB; ++nb) {
            cx<T> a[RA];
#pragma unroll
            for (int na = 0; na < RA; ++na) a[na] = x[na * RB + nb];
            DftC<T, RA>::run(a);
#pragma unroll
            for (int ka = 0; ka < RA; ++ka) x[ka * RB + nb] = nb * ka ? ctwid<T>(a[ka], __ldg(p.wr + nb * ka)) : a[ka];
        }
#pragma unroll
        for (int ka = 0; ka < RA; ++ka) {
            cx<T> b[RB];
#pragma unroll
            for (int nb = 0; nb < RB; ++nb) b[nb] = x[ka * RB + nb];
            DftC<T, RB>::run(b);
#pragma unroll
            for (int kb = 0; kb < RB; ++kb) col.store(p, ka + RA * kb, b[kb]);
        }
    }
}

// One stage of the tile kernel over the butterflies row0, row0 + step, ...: FIRST reads the column's rows from global memory
// (digit-reversed placement in the tile), LAST stores the output rows; the stages between work in place in shared memory.
enum OddStage { ODD_FIRST, ODD_MID, ODD_LAST };
template <typename T, int RAD, int STAGE, int MODE>
__device__ __forceinline__ void odd_tile_stage(const OddParams<T>& p, const OddCol<T, MODE>& col, cx<T>* sm, int L, int row0, int step,
                                               bool live) {
    const int nb = p.r / RAD;
    for (int b = row0; b < nb; b += step) {
        cx<T> x[RAD];
        int base;
        if constexpr (STAGE == ODD_FIRST) {
            base = p.perm[b] * RAD;
#pragma unroll
            for (int q = 0; q < RAD; ++q) x[q] = col.load(p, b + q * nb);
        } else {
            const int t = b % L;
            base = (b / L) * L * RAD + t;
            const int ts = t * (nb / L);                               // W_(L RAD)^(q t) = W_R^(q t R / (L RAD))
#pragma unroll
            for (int q = 0; q < RAD; ++q) {
                const cx<T> v = sm[(base + q * L) * p.cw];
                x[q] = q && t ? ctwid<T>(v, __ldg(p.wr + q * ts)) : v;
            }
        }
        DftC<T, RAD>::run(x);
        if constexpr (STAGE == ODD_LAST) {
            if (live) {
#pragma unroll
                for (int q = 0; q < RAD; ++q) col.store(p, base + q * L, x[q]);
            }
        } else {
#pragma unroll
            for (int q = 0; q < RAD; ++q) sm[(base + q * L) * p.cw] = x[q];
        }
    }
}
template <typename T, int STAGE, int MODE>
__device__ __forceinline__ void odd_tile_stage_of(int rad, const OddParams<T>& p, const OddCol<T, MODE>& col, cx<T>* sm, int L,
                                                  int row0, int step, bool live) {
    if (rad == 3) odd_tile_stage<T, 3, STAGE, MODE>(p, col, sm, L, row0, step, live);
    else if (rad == 5) odd_tile_stage<T, 5, STAGE, MODE>(p, col, sm, L, row0, step, live);
    else odd_tile_stage<T, 7, STAGE, MODE>(p, col, sm, L, row0, step, live);
}

// R rows x cw adjacent columns in shared memory (cw * sizeof(cx<T>) >= 128 bytes, so the interleaved loads and the planar
// stores both move in runs of 64 bytes or more), radix-3/5/7 stages between __syncthreads().  Thread t owns column t % cw
// and every (ODD_NT / cw)-th butterfly of it.
template <typename T, int MODE = CHIRP_C2C>
__global__ void __launch_bounds__(ODD_NT, 2) odd_tile_kernel(const __grid_constant__ OddParams<T> p) {
    extern __shared__ __align__(16) unsigned char odd_smem[];
    const int c = threadIdx.x % p.cw, row0 = threadIdx.x / p.cw, step = ODD_NT / p.cw;
    cx<T>* sm = reinterpret_cast<cx<T>*>(odd_smem) + c;
    const long long g = (long long)blockIdx.x * p.cw + c;
    const bool live = g < p.total;
    const OddCol<T, MODE> col(p, live ? g : p.total - 1);              // a dead column computes its neighbour's and stores nothing
    odd_tile_stage_of<T, ODD_FIRST>(p.rad[0], p, col, sm, 1, row0, step, live);
    int L = p.rad[0];
    for (int s = 1; s + 1 < p.nstages; ++s) {
        __syncthreads();
        odd_tile_stage_of<T, ODD_MID>(p.rad[s], p, col, sm, L, row0, step, live);
        L *= p.rad[s];
    }
    __syncthreads();
    odd_tile_stage_of<T, ODD_LAST>(p.rad[p.nstages - 1], p, col, sm, L, row0, step, live);
}

// One ODD pass of r rows over `grid` blocks: the tile kernel when smem > 0, else the register kernel of r rows (false: none).
template <typename T, int MODE>
bool launch_odd_kernel(const OddParams<T>& q, int r, size_t smem, unsigned grid, cudaStream_t stream) {
    if (smem) {
        odd_tile_kernel<T, MODE><<<grid, ODD_NT, smem, stream>>>(q);
        return true;
    }
    switch (r) {
        case 3: odd_reg_kernel<T, 3, 1, MODE><<<grid, ODD_NT, 0, stream>>>(q); return true;
        case 5: odd_reg_kernel<T, 5, 1, MODE><<<grid, ODD_NT, 0, stream>>>(q); return true;
        case 7: odd_reg_kernel<T, 7, 1, MODE><<<grid, ODD_NT, 0, stream>>>(q); return true;
        case 9: odd_reg_kernel<T, 3, 3, MODE><<<grid, ODD_NT, 0, stream>>>(q); return true;
        case 15: odd_reg_kernel<T, 5, 3, MODE><<<grid, ODD_NT, 0, stream>>>(q); return true;
        case 21: odd_reg_kernel<T, 7, 3, MODE><<<grid, ODD_NT, 0, stream>>>(q); return true;
        case 25: odd_reg_kernel<T, 5, 5, MODE><<<grid, ODD_NT, 0, stream>>>(q); return true;
        case 35: odd_reg_kernel<T, 7, 5, MODE><<<grid, ODD_NT, 0, stream>>>(q); return true;
        default: return false;
    }
}

// SMOOTH-PRE: ws[m N + n_o P + n_2] = (re, im)[m bstride + n_o + Q n_2].  A block transposes a tile of tq values of n_o by
// tp values of n_2 through shared memory: it reads runs of tq adjacent elements and writes runs of tp adjacent complex values
// (the plan picks tq * tp <= 1024 with the runs as long as Q and P allow).  The real modes load element n of z instead, the
// interleaved ones complex value n of in_re (bstride is the input's member stride in T either way; the c2r modes with an
// interleaved spectrum read its bins from in_re).
constexpr int SMOOTH_TILE = 1024;
template <typename T>
struct SmoothParams {
    const T* in_re;                // swapped for the reverse direction; C2C_IL*: the caller's interleaved array (in_im unused)
    const T* in_im;
    cx<T>* ws;
    long long n, p, q, bstride;
    int tq, tp;
    unsigned tiles_q, tiles_per_member;
    const cx<T>* wn_hi;            // C2R_HALVED: W_(2N)^e = wn_hi[e >> lo_bits] wn_lo[e & (2^lo_bits - 1)]
    const cx<T>* wn_lo;
    int lo_bits;
};

// W^e from a two-level table (hi[e >> lo_bits] lo[e & (2^lo_bits - 1)])
template <typename T>
__device__ __forceinline__ cx<T> two_level_root(const cx<T>* hi, const cx<T>* lo, int lo_bits, unsigned long long e) {
    return cmul<T>(__ldg(hi + (e >> lo_bits)), __ldg(lo + (e & ((1ull << lo_bits) - 1))));
}

// SMOOTH-PRE's element n of a real mode's z, from the member's input re / im
template <typename T, int MODE>
__device__ __forceinline__ cx<T> smooth_real_in(const SmoothParams<T>& p, const T* re, const T* im, long long n) {
    constexpr int PM = chirp_planar<MODE>();
    constexpr bool SIL = chirp_spec_il<MODE>();
    if constexpr (PM == CHIRP_R2C_HALVED) return reinterpret_cast<const cx<T>*>(re)[n];     // (x[2n], x[2n+1]), pair-aligned
    else if constexpr (PM == CHIRP_R2C_DIRECT) return make_cx<T>(re[n], T(0));
    else if constexpr (PM == CHIRP_C2R_HALVED)
        return c2r_halved_in<T>(spec_at<T, SIL>(re, im, 0), p.n, n, two_level_root<T>(p.wn_hi, p.wn_lo, p.lo_bits, n));
    else return c2r_direct_in<T>(spec_at<T, SIL>(re, im, 0), p.n, n);
}

template <typename T, int MODE = CHIRP_C2C>
__global__ void __launch_bounds__(256) smooth_pre_kernel(const __grid_constant__ SmoothParams<T> p) {
    __shared__ cx<T> sm[2 * SMOOTH_TILE];
    const unsigned m = blockIdx.x / p.tiles_per_member, tile = blockIdx.x - m * p.tiles_per_member;
    const long long o = (long long)(tile % p.tiles_q) * p.tq, a = (long long)(tile / p.tiles_q) * p.tp;
    const T* re = p.in_re + (long long)m * p.bstride;
    const T* im = p.in_im + (long long)m * p.bstride;
    const int count = p.tq * p.tp, pitch = p.tp + 1;
    for (int i = threadIdx.x; i < count; i += 256) {
        const int j2 = i / p.tq, jo = i - j2 * p.tq;
        if (o + jo < p.q) {
            const long long src = o + jo + p.q * (a + j2);
            if constexpr (MODE == CHIRP_C2C) sm[jo * pitch + j2] = make_cx<T>(re[src], im[src]);
            else if constexpr (chirp_il<MODE>()) sm[jo * pitch + j2] = il_load<T, MODE>(reinterpret_cast<const cx<T>*>(re)[src]);
            else sm[jo * pitch + j2] = smooth_real_in<T, MODE>(p, re, im, src);
        }
    }
    __syncthreads();
    cx<T>* ws = p.ws + (long long)m * p.n;
    for (int i = threadIdx.x; i < count; i += 256) {
        const int jo = i / p.tp, j2 = i - jo * p.tp;
        if (o + jo < p.q) ws[(o + jo) * p.p + a + j2] = sm[jo * pitch + j2];
    }
}

// SMOOTH-POST-R2C, the halved r2c's untangle in place: the last ODD pass stored Z = DFT_L(z) in bins 0 .. L-1 of the caller's
// arrays; the thread of pair (k, L - k), k <= L/2, replaces Z[k] and Z[L - k] with X[k] and X[L - k] (k = 0: X[0] and X[L];
// L even: k = L/2 is the self pair).  A member-major grid of 256-thread blocks.  SIL: the bins are interleaved at re
// (SMOOTH-POST-R2C-IL).
template <typename T>
struct SmoothPostParams {
    T* re;
    T* im;
    const cx<T>* wn_hi;            // W_(2L) two-level, as SmoothParams
    const cx<T>* wn_lo;
    long long l, bstride;          // bstride: elements of each array between members (interleaved: complex values)
    int lo_bits;
    unsigned blocks_per_member;
};
template <typename T, bool SIL = false>
__global__ void __launch_bounds__(256) smooth_post_r2c_kernel(const __grid_constant__ SmoothPostParams<T> p) {
    const unsigned mb = blockIdx.x / p.blocks_per_member;
    const long long k = (long long)(blockIdx.x - mb * p.blocks_per_member) * 256 + threadIdx.x;
    if (2 * k > p.l) return;
    const SpecBins<T, SIL> y = spec_at<T, SIL>(p.re, p.im, (long long)mb * p.bstride);
    const long long m = p.l - k, mm = k ? m : 0;
    cx<T> xk, xm;
    r2c_untangle<T>(y.get(k), y.get(mm), two_level_root<T>(p.wn_hi, p.wn_lo, p.lo_bits, k), xk, xm);
    y.put(k, xk.x, xk.y);
    if (m != k) y.put(m, xm.x, xm.y);
}

// ---------------------------------------------------------------------------------------------
// DCT-PRE / DCT-POST: the two elementwise ends of the DCT / DST types 2 and 3 over an N-point real FFT (Makhoul 1980), with
// W = W_(4N) from a two-level table.  DCT-II: v[n] = x[2n], v[N-1-n] = x[2n+1]; V = rfft(v); u = W^k V[k],
// y[k] = 2 Re u, y[N-k] = -2 Im u.  DCT-III: bin k = W^-k (x[k] - i x[N-k]) (x[N] = 0); v = irfft(bins) * N;
// y[2n] = v[n], y[2n+1] = v[N-1-n].  DST-II is DCT-II of (-1)^n x[n] with the output reversed, DST-III (-1)^k DCT-III of x
// reversed: the DST kinds negate the odd-indexed side of the permutation and reverse the caller's side of the twiddle.  The
// norm is folded into `scale` (and the ortho factor into `scale0`, for output 0 of DCT-II / input 0 of DCT-III, i.e. element
// N-1 of a DST), the c2r's 1/N into DCT-III's scale.  The caller's arrays (`re`, any stride and offset) are read or written with
// scalar accesses only; the workspace's reals `v` (even stride) and bins (one complex access each) belong to the plan.
// One thread per (n, N-1-n) pair (the permutations) or per bin k <= N/2 (the twiddles); a member-major grid of 256-thread
// blocks.
enum DctKind { DCT_KIND_DCT2 = 0, DCT_KIND_DCT3 = 1, DCT_KIND_DST2 = 2, DCT_KIND_DST3 = 3 };
template <typename T>
struct DctParams {
    const T* in;                   // the caller's input (PRE) or the workspace reals (type 3's POST)
    T* out;                        // the workspace reals (type 2's PRE) or the caller's output (POST)
    cx<T>* bins;                   // the workspace bins, floor(N/2) + 1 per member
    const cx<T>* w_hi;             // W_(4N)^e = w_hi[e >> lo_bits] w_lo[e & (2^lo_bits - 1)]
    const cx<T>* w_lo;
    long long n, in_stride, out_stride, bin_stride;   // member strides: T, T, complex values
    T scale, scale0;
    int lo_bits;
    unsigned blocks_per_member;
};

// v[n] = x[2n], v[N-1-n] = +-x[2n+1] (type 2's PRE), or its inverse y[2n] = v[n], y[2n+1] = +-v[N-1-n] (type 3's POST)
template <typename T, bool DST, bool INVERSE>
__device__ __forceinline__ void dct_permute(const DctParams<T>& p, long long mb, long long j) {
    if (2 * j >= p.n) return;
    const T* x = p.in + mb * p.in_stride;
    T* y = p.out + mb * p.out_stride;
    const long long r = p.n - 1 - j;
    if constexpr (INVERSE) {
        y[2 * j] = x[j];
        if (2 * j + 1 < p.n) y[2 * j + 1] = DST ? -x[r] : x[r];
    } else {
        y[j] = x[2 * j];
        if (2 * j + 1 < p.n) y[r] = DST ? -x[2 * j + 1] : x[2 * j + 1];
    }
}

template <typename T, int KIND>
__global__ void __launch_bounds__(256) dct_pre_kernel(const __grid_constant__ DctParams<T> p) {
    constexpr bool DST = KIND == DCT_KIND_DST2 || KIND == DCT_KIND_DST3;
    const unsigned mb = blockIdx.x / p.blocks_per_member;
    const long long j = (long long)(blockIdx.x - mb * p.blocks_per_member) * 256 + threadIdx.x;
    if constexpr (KIND == DCT_KIND_DCT2 || KIND == DCT_KIND_DST2) {
        dct_permute<T, DST, false>(p, mb, j);
    } else {
        if (2 * j > p.n) return;
        const T* x = p.in + (long long)mb * p.in_stride;
        // x[k] and x[N-k] of the DCT-III input, x reversed for DST-III
        const T a = x[DST ? p.n - 1 - j : j] * (j ? p.scale : p.scale0);
        const T b = j ? x[DST ? j - 1 : p.n - j] * p.scale : T(0);
        const cx<T> w = two_level_root<T>(p.w_hi, p.w_lo, p.lo_bits, (unsigned long long)j);
        p.bins[(long long)mb * p.bin_stride + j] = cmul<T>(make_cx<T>(w.x, -w.y), make_cx<T>(a, -b));
    }
}

template <typename T, int KIND>
__global__ void __launch_bounds__(256) dct_post_kernel(const __grid_constant__ DctParams<T> p) {
    constexpr bool DST = KIND == DCT_KIND_DST2 || KIND == DCT_KIND_DST3;
    const unsigned mb = blockIdx.x / p.blocks_per_member;
    const long long k = (long long)(blockIdx.x - mb * p.blocks_per_member) * 256 + threadIdx.x;
    if constexpr (KIND == DCT_KIND_DCT3 || KIND == DCT_KIND_DST3) {
        dct_permute<T, DST, true>(p, mb, k);
    } else {
        if (2 * k > p.n) return;
        const cx<T> u = cmul<T>(two_level_root<T>(p.w_hi, p.w_lo, p.lo_bits, (unsigned long long)k), p.bins[(long long)mb * p.bin_stride + k]);
        T* y = p.out + (long long)mb * p.out_stride;
        // DCT-II outputs k and N-k; DST-II stores output j of the DCT at N-1-j
        y[DST ? p.n - 1 - k : k] = u.x * (k ? p.scale : p.scale0);
        if (k && 2 * k != p.n) y[DST ? k - 1 : p.n - k] = -u.y * p.scale;
    }
}

// ---------------------------------------------------------------------------------------------
// CONV-PRE / CONV-MUL / CONV-POST: the three elementwise kernels of linear convolution and correlation over an L-point
// transform (L a power of two >= n_x + n_h - 1, so the circular convolution at L is the linear one).  Workspace members are
// L apart in the signal region (reals or complex values) and `spec_stride` bins apart in the spectrum region (the same memory
// for complex signals).  PRE pads member m < n_xm (x) or m - n_xm (h; reversed and conjugated for correlation) to L; MUL forms
// X_b H_b in place over `bins` bins, or X_b H_0 when h_bcast; POST copies the window [start, start + out_len) of member b to
// the caller.  The caller's arrays (any stride and offset, complex ones as pairs aligned to 2 * sizeof(T)) are accessed one
// element at a time.  A member-major grid of 256-thread blocks, member m0 + blockIdx.x / blocks_per_member.
template <typename T>
struct ConvParams {
    const T* x;                    // the caller's signals (PRE)
    const T* h;                    // the caller's filters (PRE)
    T* y;                          // the caller's output (POST)
    T* sig;                        // the workspace signal region: member m at sig + m * L values
    cx<T>* spec;                   // the workspace spectra: member m at spec + m * spec_stride
    long long n_x, n_h, L, x_stride, h_stride, y_stride;   // strides in values (complex ones for complex signals)
    long long n_xm;                // PRE: members below it are signals, the rest filters
    long long start, out_len;      // POST's window
    long long spec_stride, bins;   // MUL
    long long m0;                  // the first member of this launch
    int h_bcast;                   // MUL: one filter spectrum for every member
    unsigned blocks_per_member;
};

template <typename T, bool CPLX>
using conv_value_t = typename std::conditional<CPLX, cx<T>, T>::type;

template <typename T, bool CPLX, bool CORR>
__global__ void __launch_bounds__(256) conv_pre_kernel(const __grid_constant__ ConvParams<T> p) {
    using E = conv_value_t<T, CPLX>;
    const long long m = p.m0 + blockIdx.x / p.blocks_per_member;
    const long long j = (long long)(blockIdx.x % p.blocks_per_member) * 256 + threadIdx.x;
    if (j >= p.L) return;
    E v;
    if constexpr (CPLX) v = make_cx<T>(T(0), T(0)); else v = T(0);
    if (m < p.n_xm) {
        if (j < p.n_x) v = reinterpret_cast<const E*>(p.x)[m * p.x_stride + j];
    } else if (j < p.n_h) {
        v = reinterpret_cast<const E*>(p.h)[(m - p.n_xm) * p.h_stride + (CORR ? p.n_h - 1 - j : j)];
        if constexpr (CPLX && CORR) v.y = -v.y;
    }
    reinterpret_cast<E*>(p.sig)[m * p.L + j] = v;
}

template <typename T>
__global__ void __launch_bounds__(256) conv_mul_kernel(const __grid_constant__ ConvParams<T> p) {
    const long long b = p.m0 + blockIdx.x / p.blocks_per_member;
    const long long k = (long long)(blockIdx.x % p.blocks_per_member) * 256 + threadIdx.x;
    if (k >= p.bins) return;
    cx<T>* xb = p.spec + b * p.spec_stride + k;
    const cx<T> hb = p.spec[(p.n_xm + (p.h_bcast ? 0 : b)) * p.spec_stride + k];
    *xb = cmul<T>(*xb, hb);
}

template <typename T, bool CPLX>
__global__ void __launch_bounds__(256) conv_post_kernel(const __grid_constant__ ConvParams<T> p) {
    using E = conv_value_t<T, CPLX>;
    const long long b = p.m0 + blockIdx.x / p.blocks_per_member;
    const long long j = (long long)(blockIdx.x % p.blocks_per_member) * 256 + threadIdx.x;
    if (j >= p.out_len) return;
    reinterpret_cast<E*>(p.y)[b * p.y_stride + j] = reinterpret_cast<const E*>(p.sig)[b * p.L + p.start + j];
}

// ---------------------------------------------------------------------------------------------
// STFT-FRAME / ISTFT-OLA: the two elementwise kernels of the short-time Fourier transform (torch.stft / torch.istft) around
// the n_fft-point real or complex plan.  Frame f of member b is global frame m = b * n_frames + f; it covers the samples
// t = f * hop + j - pad (0 <= j < n_fft) of the member's signal, read with reflect or zero padding.  FRAME writes frame m at
// frames + m * fstride (reals for real signals, (re, im) pairs for complex ones), each sample times win[j] (the window,
// pre-scaled by n_fft^(-1/2) when normalized).  OLA writes output sample t of member b as
//   sum_f win[j] v_f[j] / sum_f win[j]^2 * scale,   j = t + pad - f * hop,
// over the frames that cover t + pad in ascending f (no atomics: bit-reproducible), zero where no frame does.  With EVEN_FIX
// (real signals, even n_fft) it first removes from each frame sample what the c2r adds for the imaginary parts of bin 0 (a)
// and bin n_fft / 2 (b), which numpy.fft.irfft and torch drop: -(a + b) / n_fft at even j, (a - b) / n_fft at odd j.  The
// caller's arrays are accessed one element at a time.  A member-major grid of 256-thread blocks, member m0 + blockIdx.x /
// blocks_per_member.
template <typename T>
struct StftParams {
    const T* x;                    // FRAME: the caller's signals
    T* frames;                     // FRAME: out, OLA: in; frame m at frames + m * fstride values (complex ones for CPLX)
    const cx<T>* spec;             // OLA with EVEN_FIX: the caller's bins, frame m at spec + m * spec_stride
    T* y;                          // OLA: the caller's output
    const T* win;                  // n_fft window values
    long long n, n_fft, hop, pad, n_frames;
    long long x_stride, fstride, spec_stride, y_stride;   // in values (complex ones for complex signals)
    long long m0;                  // the first member (FRAME: frame) of this launch
    T scale;                       // OLA: sqrt(n_fft) when normalized, else 1
    T inv_n;                       // OLA with EVEN_FIX: 1 / n_fft
    int reflect;                   // FRAME: reflect padding, else zeros
    unsigned blocks_per_member;
};

template <typename T, bool CPLX>
__global__ void __launch_bounds__(256) stft_frame_kernel(const __grid_constant__ StftParams<T> p) {
    using E = conv_value_t<T, CPLX>;
    const long long m = p.m0 + blockIdx.x / p.blocks_per_member;
    const long long j = (long long)(blockIdx.x % p.blocks_per_member) * 256 + threadIdx.x;
    if (j >= p.n_fft) return;
    const long long b = m / p.n_frames;
    long long t = (m - b * p.n_frames) * p.hop + j - p.pad;
    bool inside = true;
    if (t < 0 || t >= p.n) {
        if (p.reflect) t = t < 0 ? -t : 2 * (p.n - 1) - t;   // pad < n: one reflection lands inside
        else inside = false;
    }
    const T w = p.win[j];
    if constexpr (CPLX) {
        cx<T> v = make_cx<T>(T(0), T(0));
        if (inside) v = reinterpret_cast<const cx<T>*>(p.x)[b * p.x_stride + t];
        reinterpret_cast<cx<T>*>(p.frames)[m * p.fstride + j] = make_cx<T>(v.x * w, v.y * w);
    } else {
        const T v = inside ? p.x[b * p.x_stride + t] : T(0);
        p.frames[m * p.fstride + j] = v * w;
    }
}

template <typename T, bool CPLX, bool EVEN_FIX>
__global__ void __launch_bounds__(256) istft_ola_kernel(const __grid_constant__ StftParams<T> p) {
    using E = conv_value_t<T, CPLX>;
    const long long b = p.m0 + blockIdx.x / p.blocks_per_member;
    const long long t = (long long)(blockIdx.x % p.blocks_per_member) * 256 + threadIdx.x;
    if (t >= p.n) return;
    const long long u = t + p.pad;
    const long long f_hi = min(u / p.hop, p.n_frames - 1);
    const long long f_lo = u >= p.n_fft ? (u - p.n_fft) / p.hop + 1 : 0;   // the first frame with u - f * hop < n_fft
    T nre = T(0), nim = T(0), den = T(0);
    for (long long f = f_lo; f <= f_hi; ++f) {
        const long long j = u - f * p.hop, m = b * p.n_frames + f;
        const T w = p.win[j];
        if constexpr (CPLX) {
            const cx<T> v = reinterpret_cast<const cx<T>*>(p.frames)[m * p.fstride + j];
            nre += w * v.x;
            nim += w * v.y;
        } else {
            T v = p.frames[m * p.fstride + j];
            if constexpr (EVEN_FIX) {
                const T* im = reinterpret_cast<const T*>(p.spec + m * p.spec_stride) + 1;   // Im X[0], Im X[n_fft / 2]
                const T a = im[0], c = im[p.n_fft];
                v -= ((j & 1) ? a - c : -(a + c)) * p.inv_n;
            }
            nre += w * v;
        }
        den += w * w;
    }
    E* y = reinterpret_cast<E*>(p.y) + b * p.y_stride + t;
    const bool covered = f_lo <= f_hi;
    if constexpr (CPLX) *y = covered ? make_cx<T>(nre / den * p.scale, nim / den * p.scale) : make_cx<T>(T(0), T(0));
    else *y = covered ? nre / den * p.scale : T(0);
}

}  // namespace phast
