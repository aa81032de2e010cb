// encode_lp_kernel.cuh -- lizard_encode_lowest_price_kernel (levels 23-25 / 43-45), the device kernel
// around encode_lp.cuh: one warp per unit, with the persistent grid, atomic unit queue, Progress hand-shake and fused frame
// packing of encode.cuh, in a kernel of its own so that the existing encode instances keep their code.
//
// Scratch (carved from the encoder's workspace, which does not grow):
//   [LpPool: busy flags + kLpBigSlots big slots of 48 MiB][grid warps x LpWork (~4 MiB: sequence list, 2^17 chain, streams,
//   Huffman scratch, 2 MiB map)]
// A unit of several inner blocks needs the reference's full tables (4 * 2^hashLog + 4 * 2^22 bytes).  Its warp takes a big slot
// with an atomic and waits while none is free; a holder waits on nothing else (the frame path's progress_wait comes before the
// acquisition), so the pool cannot deadlock.  The slots are zeroed before each launch and every unit leaves its slot zero.
#pragma once
#include "encode.cuh"
#include "encode_lp.cuh"

namespace lzb {

constexpr int kLpWarpsPerCta = 4;
// 96 registers at 128 threads: 5 CTAs (20 warps) per SM.  The parser is a call of its own with no stack; the kernel's 496-byte
// frame belongs to the entropy stage it inlines (512 bytes in the Generic encode instance).
constexpr int kLpMaxRegs = 96;
constexpr u32 kLpBigSlots = 8;
constexpr size_t kLpPoolHead = 256;                      // busy flags
constexpr size_t kLpPoolBytes = kLpPoolHead + (size_t)kLpBigSlots * kLpBigSlotBytes;

__device__ __forceinline__ u32 lp_slot_acquire(u32* busy, u32 lane)
{
    u32 got = 0;
    if (lane == 0) {
        for (u32 i = 0;; i = (i + 1) % kLpBigSlots) {
            if (atomicCAS(&busy[i], 0u, 1u) == 0u) { got = i; break; }
            if (i == kLpBigSlots - 1) __nanosleep(1000);
        }
        __threadfence();
    }
    got = __shfl_sync(0xffffffffu, got, 0);
    __syncwarp();                                         // the slot's contents are read by every lane from here on
    return got;
}
__device__ __forceinline__ void lp_slot_release(u32* busy, u32 slot, u32 lane)
{
    __syncwarp();
    if (lane == 0) { __threadfence(); atomicExch(&busy[slot], 0u); }
}

__global__ void __maxnreg__(kLpMaxRegs)
lizard_encode_lowest_price_kernel(EncodeBatch b, size_t per_warp_bytes)
{
    __shared__ u32 seg_hist[kLpWarpsPerCta][4][256];
    const u32 lane = WarpLanes::lane(), wic = threadIdx.x >> 5;
    u8* const pool = b.scratch;
    u32* const busy = reinterpret_cast<u32*>(pool);
    LpWork* const work = reinterpret_cast<LpWork*>(pool + kLpPoolBytes + ((size_t)blockIdx.x * kLpWarpsPerCta + wic) * per_warp_bytes);
    if (lane == 0) work->huf.seg_count = seg_hist[wic];
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
                ulonglong2* m = reinterpret_cast<ulonglong2*>(work->map);
                for (u32 i = lane; i < (1u << kLpMapLog) / 2; i += 32) m[i] = make_ulonglong2(0, 0);
                __syncwarp();
                epoch = 0;
            }
            ++epoch;
            r = encode_unit_lp<WarpLanes>(b.src_base + b.src_off[unit], len, b.dst_base + b.dst_off[unit], b.dst_cap[unit],
                                          b.level, work, epoch, nullptr);
        } else {
            const u32 slot = lp_slot_acquire(busy, lane);
            r = encode_unit_lp<WarpLanes>(b.src_base + b.src_off[unit], len, b.dst_base + b.dst_off[unit], b.dst_cap[unit],
                                          b.level, work, 0, pool + kLpPoolHead + (size_t)slot * kLpBigSlotBytes);
            lp_slot_release(busy, slot, lane);
        }
        if (lane == 0) b.result[unit] = r;
        __syncwarp();
        if (b.pack.out) { pack_unit(b, unit, len, r, lane); __syncwarp(); pack_done(b, unit, lane); }
        else progress_done(b.progress, unit, lane);
    }
}

// Launch shape: CTAs of kLpWarpsPerCta warps, as many per SM as registers allow (5), and no more warps than the workspace holds
// an LpWork for.  The workspace is the other encoder's (28 warps per SM x 2.1 MB): with the pool and 4.07 MB per LpWork it holds
// 453 CTAs of 4 warps on 132 SMs, i.e. 1812 resident warps (13.7 per SM), below the 5 CTAs per SM that registers allow.
struct LpShape { int warps, ctas_per_sm; size_t per_warp; };
inline LpShape lp_shape()
{
    LpShape sh;
    sh.warps = kLpWarpsPerCta;
    sh.ctas_per_sm = 65536 / (kLpMaxRegs * 32 * kLpWarpsPerCta);
    sh.per_warp = (sizeof(LpWork) + 255) / 256 * 256;
    return sh;
}

// Launches the kernel.  `big_units`: the batch may hold a unit of several inner blocks (the device call cannot tell); then the
// big slots and their busy flags are zeroed first, because the pool overlaps the other encoder's per-warp scratch (384 MiB:
// about 0.15 ms at HBM3 rates).
inline cudaError_t lp_encode_launch(const EncodeConfig& c, const EncodeBatch& b, cudaStream_t s, int* launches, bool big_units)
{
    const LpShape sh = lp_shape();
    int per_sm = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lizard_encode_lowest_price_kernel, 32 * sh.warps, 0);
    if (e != cudaSuccess) return e;
    if (per_sm < 1) per_sm = 1;
    if (per_sm > sh.ctas_per_sm) per_sm = sh.ctas_per_sm;
    size_t grid = (size_t)c.sm_count * per_sm;
    const size_t need = (b.n_units + sh.warps - 1) / sh.warps;
    if (grid > need) grid = need;
    if (c.scratch_bytes < kLpPoolBytes + sh.per_warp * sh.warps) return cudaErrorMemoryAllocation;
    const size_t fit = (c.scratch_bytes - kLpPoolBytes) / (sh.per_warp * sh.warps);
    if (grid > fit) grid = fit;
    // the big slots and their busy flags start zero; units leave them zero
    if (big_units && (e = cudaMemsetAsync(b.scratch, 0, kLpPoolBytes, s)) != cudaSuccess) return e;
    lizard_encode_lowest_price_kernel<<<(unsigned)grid, 32 * sh.warps, 0, s>>>(b, sh.per_warp);
    *launches = 1;
    return cudaGetLastError();
}

}  // namespace lzb
