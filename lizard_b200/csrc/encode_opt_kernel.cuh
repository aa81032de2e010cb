// encode_opt_kernel.cuh -- lizard_encode_optimal_kernel (levels 18, 19, 39), the device kernel around encode_opt.cuh: one
// warp per unit, with the persistent grid, atomic unit queue, Progress hand-shake and fused frame packing of encode.cuh, in a
// kernel of its own so that the existing encode instances and the lowestPrice kernel keep their code.
//
// Scratch (carved from the encoder's workspace, which does not grow):
//   [LpPool: busy flags + kLpBigSlots big slots of 48 MiB][grid warps x OptWork (~4.1 MiB: LpWork, whose 2^17-entry chain is
//   the binary tree, plus opt[] and the match list)]
// A unit of several inner blocks takes a big slot of the lowestPrice pool for its hash table (4 * 2^hashLog bytes), under the
// same rules: an atomic acquisition, a holder waits on nothing else, the slot is left zero.
#pragma once
#include "encode_lp_kernel.cuh"
#include "encode_opt.cuh"

namespace lzb {

constexpr int kOptWarpsPerCta = 4;
constexpr int kOptMaxRegs = 96;

__global__ void __maxnreg__(kOptMaxRegs)
lizard_encode_optimal_kernel(EncodeBatch b, size_t per_warp_bytes)
{
    __shared__ u32 seg_hist[kOptWarpsPerCta][4][256];
    __shared__ OptStats stats[kOptWarpsPerCta];
    const u32 lane = WarpLanes::lane(), wic = threadIdx.x >> 5;
    u8* const pool = b.scratch;
    u32* const busy = reinterpret_cast<u32*>(pool);
    OptWork* const work = reinterpret_cast<OptWork*>(pool + kLpPoolBytes + ((size_t)blockIdx.x * kOptWarpsPerCta + wic) * per_warp_bytes);
    if (lane == 0) work->lp.huf.seg_count = seg_hist[wic];
    __syncwarp();
    u32 epoch = kLpEpochMax;                              // the map is cleared before the warp's first unit
    for (;;) {
        u32 unit = 0;
        if (lane == 0) unit = atomicAdd(b.counter, 1u);
        unit = __shfl_sync(0xffffffffu, unit, 0);
        if (unit >= b.n_units) break;
        progress_wait(b.progress, unit, lane);
        const u32 len = b.src_len[unit];
        int r;
        if (len <= kBlockSize) {
            if (epoch == kLpEpochMax) {
                ulonglong2* m = reinterpret_cast<ulonglong2*>(work->lp.map);
                for (u32 i = lane; i < (1u << kLpMapLog) / 2; i += 32) m[i] = make_ulonglong2(0, 0);
                __syncwarp();
                epoch = 0;
            }
            ++epoch;
            r = encode_unit_opt<WarpLanes>(b.src_base + b.src_off[unit], len, b.dst_base + b.dst_off[unit], b.dst_cap[unit],
                                           b.level, work, epoch, nullptr, &stats[wic]);
        } else {
            const u32 slot = lp_slot_acquire(busy, lane);
            r = encode_unit_opt<WarpLanes>(b.src_base + b.src_off[unit], len, b.dst_base + b.dst_off[unit], b.dst_cap[unit],
                                           b.level, work, 0, pool + kLpPoolHead + (size_t)slot * kLpBigSlotBytes, &stats[wic]);
            lp_slot_release(busy, slot, lane);
        }
        if (lane == 0) b.result[unit] = r;
        __syncwarp();
        if (b.pack.out) { pack_unit(b, unit, len, r, lane); __syncwarp(); pack_done(b, unit, lane); }
        else progress_done(b.progress, unit, lane);
    }
}

// Launch shape: CTAs of kOptWarpsPerCta warps, as many per SM as registers allow, and no more warps than the workspace holds an
// OptWork for (DESIGN.md 3.1b).
inline LpShape opt_shape()
{
    LpShape sh;
    sh.warps = kOptWarpsPerCta;
    sh.ctas_per_sm = 65536 / (kOptMaxRegs * 32 * kOptWarpsPerCta);
    sh.per_warp = (sizeof(OptWork) + 255) / 256 * 256;
    return sh;
}

// Launches the kernel.  `big_units`: the batch may hold a unit of several inner blocks (the device call cannot tell); then the
// big slots and their busy flags are zeroed first, as for the lowestPrice kernel.
inline cudaError_t opt_encode_launch(const EncodeConfig& c, const EncodeBatch& b, cudaStream_t s, int* launches, bool big_units)
{
    const LpShape sh = opt_shape();
    int per_sm = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lizard_encode_optimal_kernel, 32 * sh.warps, 0);
    if (e != cudaSuccess) return e;
    if (per_sm < 1) per_sm = 1;
    if (per_sm > sh.ctas_per_sm) per_sm = sh.ctas_per_sm;
    size_t grid = (size_t)c.sm_count * per_sm;
    const size_t need = (b.n_units + sh.warps - 1) / sh.warps;
    if (grid > need) grid = need;
    if (c.scratch_bytes < kLpPoolBytes + sh.per_warp * sh.warps) return cudaErrorMemoryAllocation;
    const size_t fit = (c.scratch_bytes - kLpPoolBytes) / (sh.per_warp * sh.warps);
    if (grid > fit) grid = fit;
    if (big_units && (e = cudaMemsetAsync(b.scratch, 0, kLpPoolBytes, s)) != cudaSuccess) return e;
    lizard_encode_optimal_kernel<<<(unsigned)grid, 32 * sh.warps, 0, s>>>(b, sh.per_warp);
    *launches = 1;
    return cudaGetLastError();
}

}  // namespace lzb
