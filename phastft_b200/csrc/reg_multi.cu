// reg_multi.cu -- instantiates the launches that run BOTH passes of a two-pass plan:
//   fft_cluster2_kernel  a K-CTA thread-block cluster per transform, intermediate through distributed shared memory
//   fft_pipe2_kernel     one persistent grid per call, intermediates in an L2-resident ring, per-transform counters
// Compiled per precision: -DPHAST_T=double|float.
#include "registry.h"

#ifndef PHAST_T
#error "compile with -DPHAST_T=double|float"
#endif

namespace phast {

namespace {

template <typename T, class RL, int C, int NT, int KIND>
KernelEntry<T> body_desc() {
    KernelEntry<T> e;
    e.kind = KIND; e.R = RL::R(); e.C = C; e.NT = NT; e.first_radix = RL::rad(0); e.stages = RL::S; e.variant = 0;
    e.smem = 0; e.fn = nullptr; e.radices = radix_string<RL>();
    return e;
}

// N = P1 * P2 points per cluster of K CTAs; CTA q owns columns [q*P2/K, (q+1)*P2/K) in pass 1 and rows
// [q*P1/K, (q+1)*P1/K) in pass 2; E = N / K points (one tile) per CTA.
template <typename T, class RL1, class RL2, int K, int NT, int MINB, int ID>
ClusterEntry<T> make_cluster() {
    constexpr int P1 = RL1::R(), P2 = RL2::R();
    constexpr int C1 = P2 / K, C2 = P1 / K;
    static_assert(P2 % K == 0 && P1 % K == 0 && C1 >= 1 && C2 >= 1, "both passes split evenly over the cluster");
    using PK1 = PassKernel<T, RL1, C1, NT, KIND_COL, 1, 0>;
    using PK2 = PassKernel<T, RL2, C2, NT, KIND_TRANS, 2, 0>;
    static_assert(PK1::TILE_ELEMS == PK2::TILE_ELEMS, "both passes use the same tile");
    static_assert(!PK1::STAGE32 && !PK2::STAGE32, "the planner builds no radix-32 stage table for cluster launches");
    static_assert(NT % C1 == 0, "a COL thread keeps its column");
    constexpr size_t SMEM = PK1::SMEM_BYTES > PK2::SMEM_BYTES ? PK1::SMEM_BYTES : PK2::SMEM_BYTES;
    static_assert(SMEM <= 227 * 1024, "tile exceeds the 227 KB shared memory of an sm_90 CTA");
    ClusterEntry<T> e;
    e.log2n = ilog2_c(P1) + ilog2_c(P2); e.K = K; e.NT = NT; e.minb = MINB; e.variant = ID;
    e.k1 = body_desc<T, RL1, C1, NT, KIND_COL>();
    e.k2 = body_desc<T, RL2, C2, NT, KIND_TRANS>();
    e.fn = reinterpret_cast<const void*>(&fft_cluster2_kernel<PK1, PK2, T, NT, MINB>);
    e.smem = SMEM;
    return e;
}

template <typename T, class RL1, int C1, int NT1, int V1, class RL2, int C2, int NT2, int V2, int MINB, int ASYNC = 0>
PipeEntry<T> make_pipe() {
    using PK1 = PassKernel<T, RL1, C1, NT1, KIND_COL, ASYNC ? MODE_TMA_IN : MODE_PLAIN, V1>;
    using PK2 = PassKernel<T, RL2, C2, NT2, KIND_TRANS, ASYNC ? MODE_BULK_IN : MODE_PLAIN, V2>;
    constexpr int NTF = NT1 > NT2 ? NT1 : NT2;
    static_assert(!ASYNC || NT1 == NT2, "asynchronous bodies: thread 0 issues the copies, every thread is a worker");
    PipeEntry<T> e;
    e.mode = ASYNC;
    e.R1 = RL1::R(); e.C1 = C1; e.NT1 = NT1; e.R2 = RL2::R(); e.C2 = C2; e.NT2 = NT2;
    e.rad1 = radix_string<RL1>(); e.rad2 = radix_string<RL2>();
    e.fn = reinterpret_cast<const void*>(&fft_pipe2_kernel<PK1, PK2, T, NTF, MINB>);
    e.NT = NTF;
    e.smem = PK1::SMEM_BYTES > PK2::SMEM_BYTES ? PK1::SMEM_BYTES : PK2::SMEM_BYTES;
    return e;
}

}  // namespace

// Cluster launches.  The stage on either side of the exchange is a single trip (one task per thread: the
// producer holds its results in registers across the cluster barrier, the consumer its inputs across a block
// barrier), so NT = E / radix there.  64 KB tiles (E = 8192 f32 / 4096 f64 points) hold two CTAs per SM so one CTA's
// exchange overlaps the other's HBM traffic; the 128 KB builds (ids 1xx) have half the share of remote traffic.
template <>
const std::vector<ClusterEntry<PHAST_T>>& cluster_registry<PHAST_T>() {
    using T = PHAST_T;
    static const std::vector<ClusterEntry<T>> reg = [] {
        std::vector<ClusterEntry<T>> v;
        using R64 = RadixList<4, 16>; using R128a = RadixList<8, 16>; using R128b = RadixList<16, 8>;
        using R256 = RadixList<16, 16>;
        if constexpr (sizeof(T) == 4) {
            v.push_back(make_cluster<T, R128a, R128b, 2, 512, 2, 0>());     // 2^14
            v.push_back(make_cluster<T, R128a, R256, 4, 512, 2, 0>());      // 2^15
            v.push_back(make_cluster<T, R256, R256, 8, 512, 2, 0>());       // 2^16
            v.push_back(make_cluster<T, R256, R256, 8, 512, 1, 1>());       // 2^16, register budget of one CTA per SM
            v.push_back(make_cluster<T, R256, R256, 4, 1024, 1, 100>());    // 2^16, 128 KB tiles
            v.push_back(make_cluster<T, R128a, R256, 2, 1024, 1, 100>());   // 2^15, 128 KB tiles
        } else {
            v.push_back(make_cluster<T, R64, R128b, 2, 256, 2, 0>());       // 2^13
            v.push_back(make_cluster<T, R128a, R128b, 4, 256, 2, 0>());     // 2^14
            v.push_back(make_cluster<T, R128a, R256, 8, 256, 2, 0>());      // 2^15
            v.push_back(make_cluster<T, R256, R256, 16, 256, 2, 0>());      // 2^16 (cluster of 16: non-portable size)
            v.push_back(make_cluster<T, R128a, R128b, 2, 512, 1, 100>());   // 2^14, 128 KB tiles
            v.push_back(make_cluster<T, R128a, R256, 4, 512, 1, 100>());    // 2^15, 128 KB tiles
            v.push_back(make_cluster<T, R256, R256, 8, 512, 1, 100>());     // 2^16, 128 KB tiles
        }
        return v;
    }();
    return reg;
}

// Pipelined two-pass launches.  The pairs are the plans the planner makes for BATCHES of 2^13..2^20-point transforms
// (PassDesc::kb: 64-byte-run tiles) and for a lone 2^20; the knob values (V) repeat the ones of the registry entries so
// pipelined and two-launch results are bit-identical.
template <>
const std::vector<PipeEntry<PHAST_T>>& pipe_registry<PHAST_T>() {
    using T = PHAST_T;
    static const std::vector<PipeEntry<T>> reg = [] {
        std::vector<PipeEntry<T>> v;
        constexpr int CN = TileC<T>::CN, CH = TileC<T>::CH;
        constexpr bool F64 = sizeof(T) == 8;
        using R64 = RadixList<8, 8>; using R128 = RadixList<16, 8>; using R256 = RadixList<16, 16>; using R512 = RadixList<8, 8, 8>;
        using R1024 = typename std::conditional<F64, RadixList<32, 32>, RadixList<16, 8, 8>>::type;
        constexpr int NT256 = F64 ? 128 : 256, NT1024 = F64 ? 256 : 512;
        // MINB: the register budget of the merged kernel is pinned to the occupancy its two passes have as separate kernels
        // (left alone ptxas gives the loop 128 registers: 2 CTAs/SM instead of 3-4, measured much slower on 4096 x 2^16 f32)
        constexpr int M64 = F64 ? 8 : 10, M128 = F64 ? 4 : 6, M256 = F64 ? 4 : 4, M512 = 2, M1024 = 1;
        v.push_back(make_pipe<T, R64, CN, 64, 0, R128, CN, 128, 0, M128>());         // 2^13 = {6,7}
        v.push_back(make_pipe<T, R128, CN, 128, 0, R128, CN, 128, 0, M128>());       // 2^14
        v.push_back(make_pipe<T, R128, CN, 128, 0, R256, CN, NT256, 0, M256>());     // 2^15 = {7,8}
        v.push_back(make_pipe<T, R256, CN, NT256, 0, R256, CN, NT256, 0, M256>());   // 2^16
        v.push_back(make_pipe<T, R512, CN, 256, 3, R256, CN, NT256, 0, M512>());     // 2^17 = {9,8}
        v.push_back(make_pipe<T, R512, CN, 256, 3, R512, CN, 256, 3, M512>());       // 2^18
        v.push_back(make_pipe<T, R1024, CN, NT1024, 0, R512, CN, 256, 3, M1024>());  // 2^19 = {10,9}
        v.push_back(make_pipe<T, R1024, CN, NT1024, 0, R1024, CN, NT1024, 0, M1024>());  // 2^20
        // the same 2^16 pair with asynchronous tile input (both stages a single trip: NT = 16 * C)
        v.push_back(make_pipe<T, R256, CN, 16 * CN, 0, R256, CN, 16 * CN, 0, M256, 1>());
        (void)M64; (void)CH;
        return v;
    }();
    return reg;
}

}  // namespace phast
