// frame_async_kernels.cuh -- the kernels of LizardB200_decompressFramesAsync (DESIGN.md 3.4b): frame planning, the decode
// unit table, settling and verdicts on the device, so that the call enqueues a fixed sequence of launches and reads nothing
// back.  Included by api.cu after frame_device_kernels.cuh; the serial rules they run are in frame_device.cuh.
#pragma once
#include "frame_device_kernels.cuh"

namespace lzb {

// The call's device tables (frame.inl: decompress_frames_async lays them out in one workspace buffer).
struct FrameAsync {
    const u8* src; const u64* src_off; const u64* src_size;     // the caller's frames
    const u64* dst_off; const u64* dst_cap; size_t* result;     // the caller's output ranges and results
    u32 n; u32 max_blocks; u64 stage_bytes; u32 tiles;
    FrameInfoRec* info;                                         // [n] index pass 1, then pass 2 (admitted frames)
    u64* base;                                                  // [n] the frame's first block in the block tables
    u32* adm;                                                   // [n] 1: admitted (after step 1: passed the block bound)
    u64* size2;                                                 // [n] the frame's size for index pass 2 (0: not walked)
    u64* tsum;                                                  // [tiles] sums of the planning tiles
    u64* out;                                                   // [n] output bytes before the checksum
    u32* verdict;                                               // [n] kFwOk / error, kFaRefused, kFaHash
    u32* h_count; u64* h_off; u64* h_len; u32* h_frame; u32* hash;  // the frames whose verdict waits for their checksum
    FrameBlockRec* blocks;                                      // [max_blocks] block records (index pass 2)
    u64* u_src; u32* u_len; u64* u_stage; u32* u_cap; int* u_res;  // [max_blocks] decode units (length 0: none)
    FrameGather g;                                              // [max_blocks] gather entries
};
enum : u32 { kFaRefused = 0xFFFFFFFEu, kFaHash = 0xFFFFFFFFu };
constexpr u32 kPlanThreads = 1024;                              // frames per planning tile

// Exclusive scan of v over the CTA; *total = the CTA's sum.  Every thread of the CTA calls it.
__device__ __forceinline__ u64 plan_cta_scan(u64 v, u64* total)
{
    __shared__ u64 ws[kPlanThreads / 32];
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u64 inc = v;
    for (int o = 1; o < 32; o <<= 1) { const u64 t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= (u32)o) inc += t; }
    if (lane == 31) ws[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        u64 w = ws[lane];
        for (int o = 1; o < 32; o <<= 1) { const u64 t = __shfl_up_sync(0xffffffffu, w, o); if (lane >= (u32)o) w += t; }
        ws[lane] = w;
    }
    __syncthreads();
    const u64 before = warp ? ws[warp - 1] : 0;
    *total = ws[kPlanThreads / 32 - 1];
    __syncthreads();
    return before + inc - v;
}

// what frame i asks for in planning step `step` (0: blocks, 1: slot bytes, for a frame that passed step 0)
__device__ __forceinline__ u64 plan_demand(const FrameAsync& a, u32 i, u32 step)
{
    if (i >= a.n) return 0;
    const FrameInfoRec& fi = a.info[i];
    if (step == 0) return frame_plan_blocks(fi);
    return a.adm[i] ? frame_plan_slots(fi, a.blocks + a.base[i]) : 0;
}

// Planning, tile pass: the sum of each tile's demands.  Step 0 also clears the unit and gather tables and the checksum list
// left by the previous call, so that blocks no admitted frame owns decode and move nothing.
__global__ void __launch_bounds__(kPlanThreads) lizard_frames_async_tile_kernel(FrameAsync a, u32 step)
{
    if (step == 0) {
        for (u32 k = blockIdx.x * kPlanThreads + threadIdx.x; k < a.max_blocks; k += gridDim.x * kPlanThreads) {
            a.u_src[k] = 0; a.u_len[k] = 0; a.u_stage[k] = 0; a.u_cap[k] = 0;
            a.g.s_len[k] = 0; a.g.r_len[k] = 0;
        }
        if (blockIdx.x == 0 && threadIdx.x == 0) *a.h_count = 0;
    }
    u64 total;
    plan_cta_scan(plan_demand(a, blockIdx.x * kPlanThreads + threadIdx.x, step), &total);
    if (threadIdx.x == 0) a.tsum[blockIdx.x] = total;
}

// Planning, apply pass: each frame's exclusive sum (the tiles in front, summed by the CTA, plus its place in its own tile) and
// its admission.  Step 0: block bases, and the sizes index pass 2 walks (0 for a frame past the block bound).  Step 1: the
// final admission, and the decode units of the admitted frames' compressed blocks, each in a slot of its frame's maximum
// block size behind the slots of the frames in front.
__global__ void __launch_bounds__(kPlanThreads) lizard_frames_async_plan_kernel(FrameAsync a, u32 step)
{
    u64 front = 0, total;
    for (u32 t = threadIdx.x; t < blockIdx.x; t += kPlanThreads) front += a.tsum[t];
    plan_cta_scan(front, &total);
    front = total;
    const u32 i = blockIdx.x * kPlanThreads + threadIdx.x;
    const u64 v = plan_demand(a, i, step);
    const u64 before = front + plan_cta_scan(v, &total);
    if (i >= a.n) return;
    if (step == 0) {
        const bool ok = frame_admit_blocks(before, v, a.max_blocks);
        a.base[i] = before; a.adm[i] = ok; a.size2[i] = ok ? a.src_size[i] : 0;
        return;
    }
    const bool ok = a.adm[i] && frame_admit_slots(before, v, a.stage_bytes);
    a.adm[i] = ok;
    if (!ok) return;
    const FrameInfoRec& fi = a.info[i];
    const u64 b0 = a.base[i];
    const u32 nb = (u32)frame_plan_blocks(fi);
    u64 slot = before;
    for (u32 k = 0; k < nb; ++k) {
        const FrameBlockRec b = a.blocks[b0 + k];
        if (b.raw) continue;
        a.u_src[b0 + k] = a.src_off[i] + b.src; a.u_len[b0 + k] = b.csize; a.u_stage[b0 + k] = slot; a.u_cap[b0 + k] = fi.max_block;
        slot += fi.max_block;
    }
}

// Settling: one thread per frame replays frame_settle over its blocks' decode results and writes their gather entries; a frame
// whose verdict depends on its content checksum joins the checksum list.
__global__ void __launch_bounds__(128) lizard_frames_async_settle_kernel(FrameAsync a)
{
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    if (!a.adm[i]) { a.verdict[i] = kFaRefused; return; }
    const u64 b0 = a.base[i];
    FrameGather g = a.g;
    g.s_off += b0; g.s_dst += b0; g.s_len += b0; g.r_off += b0; g.r_dst += b0; g.r_len += b0;
    u64 out;
    u32 check;
    const u32 v = frame_settle_entries(a.info[i], a.blocks + b0, a.u_res + b0, a.u_stage + b0, a.src_off[i], a.dst_off[i],
                                       a.dst_cap[i], g, &out, &check);
    a.out[i] = out;
    a.verdict[i] = check ? kFaHash : v;
    if (check) {
        const u32 h = atomicAdd(a.h_count, 1u);
        a.h_off[h] = a.dst_off[i]; a.h_len[h] = out; a.h_frame[h] = i;
    }
}

// XXH32 of the frames on the checksum list, whose length the settle kernel left in device memory (lizard_frame_hash_kernel's
// loop); frame h_frame[k]'s hash goes to hash[h_frame[k]].
__global__ void __launch_bounds__(kHashWarps * 32) lizard_frames_async_hash_kernel(const u8* base, const u64* off, const u64* len,
                                                                                  const u32* count, u32* out, const u32* slot)
{
    __shared__ __align__(16) uint4 stage[kHashWarps][kHashWords + 1];
    frame_hash_buffers(stage, base, off, len, *count, out, slot);
}

// Verdicts: result[i] as LizardB200_decompressFrames reports it, LizardF_ERROR_allocation_failed for a frame not admitted.
__global__ void __launch_bounds__(128) lizard_frames_async_verdict_kernel(FrameAsync a)
{
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    u32 v = a.verdict[i];
    if (v == kFaRefused) v = kFwAllocation;
    else if (v == kFaHash) v = frame_settle_hash(a.info[i], a.hash[i]);
    a.result[i] = v != kFwOk ? (size_t)-(long long)v : a.info[i].skippable ? 0 : (size_t)a.out[i];
}

}  // namespace lzb
