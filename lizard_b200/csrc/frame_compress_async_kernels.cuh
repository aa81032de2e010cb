// frame_compress_async_kernels.cuh -- the kernels of LizardB200_compressFramesAsync (DESIGN.md 3.4c): frame planning and the
// block table on the device, so that the call enqueues a fixed sequence of launches and reads nothing back.  The encoder, the
// hash kernel and the frame assembly (frame_device_kernels.cuh) run unchanged over the tables these kernels write.  Included by
// api.cu after frame_async_kernels.cuh; the per-frame decisions they run are in frame_device.cuh.
#pragma once
#include "frame_async_kernels.cuh"

namespace lzb {

// The call's device tables (frame.inl: compress_frames_async lays them out in one workspace buffer).  The FrameAsm tables have
// one entry more than there are frames: frame n owns the padding blocks and is never live.
struct FrameCompressAsync {
    const u64* src_off; const u64* src_size;                    // the caller's frames
    const u64* dst_off; const u64* dst_cap; size_t* result;     // the caller's output ranges and results
    FramePrefs prefs; u32 level_ok;
    u32 n; u32 max_blocks; u64 stage_bytes;
    u64* tsum;                                                  // [2 * tiles] block and staging sums of the planning tiles
    u32* verdict;                                               // [n] frame_compress_plan's verdict, kFaRefused if not admitted
    u32* bsize; u64* sbase;                                     // [n] block size, first staging byte
    u64* h_len;                                                 // [n] bytes to hash: the source of a live checksummed frame, else 0
    u64* first; u32* nblk; u8* hdr; u32* hdr_len; u32* ccksum;  // [n + 1] FrameAsm's per-frame tables
    u32* live; u64* f_dst_off; u64* f_dst_cap;
    u64* b_src_off; u32* b_len; u32* b_cap; u64* b_enc_off; u32* b_frame;  // [max_blocks] FrameAsm's and the encoder's block tables
    const u64* total;                                           // [n] FrameAsm's frame sizes
};

// frame i's plan (its header bytes go to its slot of the header table) and what it asks for; nothing past the last frame
__device__ __forceinline__ void compress_plan_of(const FrameCompressAsync& a, u32 i, FrameCompressPlan* pl, u64* blocks, u64* stage)
{
    *blocks = 0; *stage = 0;
    if (i >= a.n) return;
    frame_compress_plan(a.prefs, a.level_ok != 0, a.src_size[i], a.dst_cap[i], a.hdr + 16 * (size_t)i, pl);
    *blocks = frame_compress_demand_blocks(*pl, a.max_blocks);
    *stage = frame_compress_demand_stage(*pl);
}

// Planning, tile pass: each tile's sums of blocks and staging bytes.  (The header bytes land in the table here and again, the
// same, in the apply pass.)
__global__ void __launch_bounds__(kPlanThreads) lizard_frames_compress_tile_kernel(FrameCompressAsync a)
{
    FrameCompressPlan pl;
    u64 b, s, tb, ts;
    compress_plan_of(a, blockIdx.x * kPlanThreads + threadIdx.x, &pl, &b, &s);
    plan_cta_scan(b, &tb);
    plan_cta_scan(s, &ts);
    if (threadIdx.x == 0) { a.tsum[2 * blockIdx.x] = tb; a.tsum[2 * blockIdx.x + 1] = ts; }
}

// Planning, apply pass: each frame's two exclusive sums (the tiles in front, summed by the CTA, plus its place in its own tile),
// its admission, and every per-frame entry of the tables.  A frame's blocks are known from its size, so one pass decides both
// bounds.
__global__ void __launch_bounds__(kPlanThreads) lizard_frames_compress_plan_kernel(FrameCompressAsync a)
{
    u64 fb = 0, fs = 0, total;
    for (u32 t = threadIdx.x; t < blockIdx.x; t += kPlanThreads) { fb += a.tsum[2 * t]; fs += a.tsum[2 * t + 1]; }
    plan_cta_scan(fb, &total);
    fb = total;
    plan_cta_scan(fs, &total);
    fs = total;
    const u32 i = blockIdx.x * kPlanThreads + threadIdx.x;
    FrameCompressPlan pl;
    u64 b, s;
    compress_plan_of(a, i, &pl, &b, &s);
    const u64 bb = fb + plan_cta_scan(b, &total);
    const u64 sb = fs + plan_cta_scan(s, &total);
    if (i >= a.n) return;
    const bool adm = frame_admit_blocks(bb, b, a.max_blocks) && frame_admit_slots(sb, s, a.stage_bytes);
    const bool live = adm && pl.verdict == kFwOk;
    a.verdict[i] = adm ? pl.verdict : kFaRefused;
    a.bsize[i] = pl.block_size; a.sbase[i] = sb;
    a.h_len[i] = live && pl.ccksum ? a.src_size[i] : 0;
    a.first[i] = bb; a.nblk[i] = live ? (u32)b : 0; a.hdr_len[i] = pl.hdr_len; a.ccksum[i] = pl.ccksum; a.live[i] = live;
    a.f_dst_off[i] = a.dst_off[i]; a.f_dst_cap[i] = a.dst_cap[i];
}

// Block table: entry k belongs to the last frame whose first block is at most k (a binary search over the block bases, which
// never decrease), if k lies within that frame's live blocks; every other entry is padding of length 0 and capacity 0, on
// which every encoder returns 0 without writing, owned by frame n.  Also writes frame n's entries.
__global__ void __launch_bounds__(256) lizard_frames_compress_blocks_kernel(FrameCompressAsync a)
{
    const u32 n = a.n;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        a.first[n] = 0; a.nblk[n] = 0; a.hdr_len[n] = 0; a.ccksum[n] = 0; a.live[n] = 0; a.f_dst_off[n] = 0; a.f_dst_cap[n] = 0;
    }
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < a.max_blocks; k += gridDim.x * blockDim.x) {
        u32 lo = 0, hi = n;                                     // first[0] = 0 <= k
        while (hi - lo > 1) {
            const u32 mid = lo + (hi - lo) / 2;
            if (a.first[mid] <= k) lo = mid; else hi = mid;
        }
        const u64 j = k - a.first[lo];
        u64 src = 0, enc = 0;
        u32 len = 0, f = n;
        if (j < a.nblk[lo]) {
            const u64 bs = a.bsize[lo], at = j * bs, left = a.src_size[lo] - at;
            len = (u32)(left < bs ? left : bs);
            src = a.src_off[lo] + at; enc = a.sbase[lo] + at; f = lo;
        }
        a.b_src_off[k] = src; a.b_len[k] = len; a.b_cap[k] = len ? len - 1 : 0;       // lizard_frame.c:459
        a.b_enc_off[k] = enc; a.b_frame[k] = f;
    }
}

// Verdicts: result[i] as LizardB200_compressFrames reports it, LizardF_ERROR_allocation_failed for a frame not admitted.
__global__ void __launch_bounds__(128) lizard_frames_compress_verdict_kernel(FrameCompressAsync a)
{
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    u32 v = a.verdict[i];
    if (v == kFaRefused) v = kFwAllocation;
    else if (v == kFwOk && a.total[i] == kFrameTooBig) v = kFwDstTooSmall;
    a.result[i] = v != kFwOk ? (size_t)-(long long)v : (size_t)a.total[i];
}

}  // namespace lzb
