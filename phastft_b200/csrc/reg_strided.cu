// reg_strided.cu -- instantiates the first / middle (KIND_COL) and last (KIND_TRANS) pass kernels.
// Compiled four times: -DPHAST_T=double|float -DPHAST_KIND=KIND_COL|KIND_TRANS (see __graft_entry__.build()).
#include "registry.h"

#ifndef PHAST_T
#error "compile with -DPHAST_T=double|float -DPHAST_KIND=KIND_COL|KIND_TRANS"
#endif

namespace phast {

// Every (kind, R, C) the planner can ask for has a DEFAULT entry (variant id 0) whose code-generation knobs
// (task-loop unrolling, twiddle derivation, register budget, thread count) are the ones that measured fastest for
// that tile when it was tuned (not re-tuned on H100); push_entry also adds, for COL tiles, the MODE_C2R_IN build of the same kernel
// (the first pass of the half-length inverse transform inside c2r, pre-processing folded into its loads) -- used on the tiles
// the planner picks as the FIRST pass of a lone transform (a plan whose first pass has no such build keeps the separate sweep);
// push_entry_batch does the same for the first-pass tiles of batched calls (PassDesc::kb) of the inner plans of N = 2^13..2^31,
// whose c2r build only batched c2r uses (PassDesc::kcb); variant 62 is the half-width 1024-row middle tile the planner asks
// for by id.  The losing alternates of round 1 are no longer compiled.
//   knob bits: 1 = unroll the task loops of the shared-memory stages, 2 = stage twiddles from 3 table loads +
//   products, 4 = unroll the stage-1 task loop;  MINB = CTAs/SM the register budget is sized for.
template <>
void add_strided_kernels<PHAST_T, PHAST_KIND>(std::vector<KernelEntry<PHAST_T>>& v) {
    using T = PHAST_T;
    constexpr int KIND = PHAST_KIND;
    constexpr int CH = TileC<T>::CH, CN = TileC<T>::CN, CW = TileC<T>::CW;
    constexpr bool F64 = sizeof(T) == 8;
    push_entry<T, KIND, CH, 32, 0, 0, 0, 8, 8>(v);
    push_entry<T, KIND, CH, 64, 0, 0, 0, 16, 8>(v);
    push_entry<T, KIND, CH, F64 ? 64 : 128, 0, 0, 0, 16, 16>(v);
    push_entry<T, KIND, CN, 32, 0, 0, 0, 4, 8>(v);
    v.push_back(make_entry_v<T, KIND, CW, 64, 0, 0, 0, 4, 8>());
    v.push_back(make_entry_v<T, KIND, CN, 64, 0, 0, 0, 8, 8>());
    v.push_back(make_entry_v<T, KIND, CW, 128, 0, 0, 0, 8, 8>());
    v.push_back(make_entry_v<T, KIND, 2 * CW, 256, 0, 0, 0, 8, 8>());
    push_entry_batch<T, KIND, CN, 128, 0, 0, 0, 16, 8>(v);
    push_entry<T, KIND, CW, 256, 0, 0, 0, 16, 8>(v);
    v.push_back(make_entry_v<T, KIND, 2 * CW, 256, 0, 0, 0, 16, 8>());
    // R = 256 as two radix-16 stages (one shared-memory exchange): faster as a first pass than
    // 4x8x8; 128 threads for the 64-byte-run f64 tile (128 tasks per stage)
    if constexpr (F64) {
        push_entry_batch<T, KIND, CN, 128, 0, 0, 0, 16, 16>(v);
        push_entry<T, KIND, CW, 256, 0, 0, 0, 16, 16>(v);
        push_entry<T, KIND, CN, 256, 3, 2, 0, 8, 8, 8>(v);      // +20% over the plain build
        v.push_back(make_entry_v<T, KIND, CW, 256, 3, 2, 0, 8, 8, 8>());
        push_entry<T, KIND, CH, 256, 3, 2, 0, 8, 8, 8>(v);
        // two radix-32 stages: faster at 2^20 (no c2r build: at 255 registers it spills, as the plain build does)
        v.push_back(make_entry_v<T, KIND, CN, 256, 0, 0, 0, 32, 32>());
        push_entry<T, KIND, CH, 512, 0, 1, 0, 16, 8, 8>(v);
    } else {
        push_entry_batch<T, KIND, CN, 256, 0, 0, 0, 16, 16>(v);
        push_entry<T, KIND, CW, 256, 0, 0, 0, 16, 16>(v);
        push_entry<T, KIND, CN, 256, 3, 2, 0, 8, 8, 8>(v);
        v.push_back(make_entry_v<T, KIND, CW, 256, 3, 2, 0, 8, 8, 8>());
        push_entry<T, KIND, CH, 256, 3, 2, 0, 8, 8, 8>(v);
        push_entry_batch<T, KIND, CN, 512, 0, 1, 0, 16, 8, 8>(v);
        push_entry<T, KIND, CH, 256, 0, 0, 0, 32, 32>(v);       // two radix-32 stages: faster at 2^20
    }
    // id 62: the 1024-row tile at half width (64 KB f64 / 32 KB f32) for interleaved intermediates, register budget
    // pinned to 2 CTAs/SM (150 registers and 1 CTA/SM otherwise: much slower on the 2^26 middle pass)
    v.push_back(make_entry_v<T, KIND, CH, 256, 7, 2, 62, 16, 8, 8>());
    // Asynchronous tile input (variant ids 3xx): the tile arrives by TMA (first pass: cp.async.bulk.tensor boxes of the
    // planar arrays; last pass: cp.async.bulk copies of the contiguous rows of the interleaved workspace).  32-byte runs
    // cost the LSU nothing this way, so a 1024-row tile can be 64 KB (CH columns) and three CTAs share an SM.
    constexpr int MODE = KIND == KIND_COL ? MODE_TMA_IN : MODE_BULK_IN;
    v.push_back(make_entry_async<T, KIND, CH, 32 * CH, MODE, 0, 3, 300, 32, 32>());      // 1024 rows, 64 KB tile
    v.push_back(make_entry_async<T, KIND, CN, 32 * CN, MODE, 0, 1, 301, 32, 32>());      // 1024 rows, 128 KB tile
    v.push_back(make_entry_async<T, KIND, CH, 32 * CH, MODE, 0, 3, 300, 16, 32>());      // 512 rows, 32 KB tile
    v.push_back(make_entry_async<T, KIND, CN, 32 * CN, MODE, 0, 1, 301, 16, 32>());      // 512 rows, 64 KB tile
    // half-width 256- and 128-row tiles: the middle pass of the 3-pass plans of 2^21..2^24 points (COL only)
    if constexpr (KIND == KIND_COL) {
        v.push_back(make_entry_async<T, KIND, CH, 16 * CH, MODE, 0, 0, 310, 16, 16>());  // 256 rows x CH   (id 310: middle passes only,
        v.push_back(make_entry_async<T, KIND, CH, 8 * CH, MODE, 0, 0, 310, 16, 8>());    // 128 rows x CH    never half of a 2-pass pair)
    }
    // the 256-row end passes of 3-pass plans (128-byte runs) and the batch tiles (64-byte runs), one task per thread per stage
    v.push_back(make_entry_async<T, KIND, CW, 16 * CW, MODE, 0, 0, 300, 16, 16>());      // 256 rows x CW
    v.push_back(make_entry_async<T, KIND, CN, 16 * CN, MODE, 0, 0, 300, 16, 16>());      // 256 rows x CN
}

}  // namespace phast
