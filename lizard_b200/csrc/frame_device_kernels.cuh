// frame_device_kernels.cuh -- the kernels of LizardB200_compressFrames / LizardB200_decompressFrames (DESIGN.md 3.4a).
// Included by api.cu after encode.cuh; the serial routines they run are in frame_device.cuh.
#pragma once
#include "frame_device.cuh"
#include "encode.cuh"

namespace lzb {

// Frame index: one thread per frame walks its header and block chain (frame_walk).  Count pass (block_base null): the
// frame's verdict and block count.  Fill pass: the same, plus its block records at blocks + block_base[i].
__global__ void __launch_bounds__(128) lizard_frame_index_kernel(const u8* src, const u64* off, const u64* size, u32 n,
                                                                 FrameInfoRec* info, const u64* block_base, FrameBlockRec* blocks)
{
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    FrameInfoRec fi;
    if (block_base) frame_walk(src + off[i], size[i], &fi, blocks + block_base[i], 0xFFFFFFFFu);
    else frame_walk(src + off[i], size[i], &fi, nullptr, 0);
    info[i] = fi;
}

// XXH32 of many buffers (seed 0): one warp per buffer.  The warp stages 4 KiB of the buffer at a time in shared memory with
// aligned 16-byte loads (the next piece is loaded into registers while the current one is hashed); lanes 0-3 each run one of
// the four accumulators over the piece's stripes, and lane 0 merges them and hashes the tail.  The recurrence stays serial:
// one buffer hashes at one warp's rate.  Buffer f's hash goes to out[slot[f]] (slot null: out[f]).
constexpr u32 kHashWarps = 4, kHashPiece = 4096, kHashWords = kHashPiece / 16 + 1;
// the loop of both hash kernels (n: the number of buffers, read by the caller)
__device__ __forceinline__ void frame_hash_buffers(uint4 (*stage)[kHashWords + 1], const u8* base, const u64* off, const u64* len,
                                                   u32 n, u32* out, const u32* slot)
{
    const u32 warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr u32 kPer = (kHashWords + 31) / 32;
    for (u32 f = blockIdx.x * kHashWarps + warp; f < n; f += gridDim.x * kHashWarps) {
        const u8* p = base + off[f];
        const u64 L = len[f];
        const u32 o = (u32)((size_t)p & 15);
        const uint4* a = (const uint4*)(p - o);
        const u64 words_total = (o + L + 15) / 16;                        // aligned words holding a byte of the buffer
        const u64 stripes = L / 16;
        const u64 pieces = L ? (L + kHashPiece - 1) / kHashPiece : 0;
        u32 v = lane < 4 ? xx_lane_init(0, lane) : 0;
        uint4 nx[kPer];
        auto load = [&](u64 pc) {
#pragma unroll
            for (u32 j = 0; j < kPer; ++j) {
                const u64 w = pc * (kHashPiece / 16) + lane + 32 * j;
                if (lane + 32 * j < kHashWords && w < words_total) nx[j] = a[w];
            }
        };
        auto store = [&]() {
#pragma unroll
            for (u32 j = 0; j < kPer; ++j) if (lane + 32 * j < kHashWords) stage[warp][lane + 32 * j] = nx[j];
        };
        if (pieces) load(0);
        for (u64 pc = 0; pc < pieces; ++pc) {
            __syncwarp();
            store();
            __syncwarp();
            if (pc + 1 < pieces) load(pc + 1);
            const u64 s0 = pc * (kHashPiece / 16);
            const u32 ns = (u32)(stripes > s0 ? (stripes - s0 < kHashPiece / 16 ? stripes - s0 : kHashPiece / 16) : 0);
            const u32* sw = (const u32*)stage[warp];
            const u32 sh = 8 * (o & 3);
            if (lane < 4) {
                u32 at = (o >> 2) + lane;
#pragma unroll 4
                for (u32 s = 0; s < ns; ++s, at += 4) v = xx_round(v, __funnelshift_r(sw[at], sw[at + 1], sh));
            }
            if (pc + 1 == pieces) {                                       // the tail lies in the last piece
                __syncwarp();
                u32 acc[4];
                for (int l = 0; l < 4; ++l) acc[l] = __shfl_sync(0xffffffffu, v, l);
                if (lane == 0)
                    out[slot ? slot[f] : f] = xx_finish(acc, L, (const u8*)stage[warp] + o + 16 * (stripes - s0), (u32)(L % 16), 0);
            }
        }
        if (!pieces && lane == 0) { const u32 z[4] = { 0, 0, 0, 0 }; out[slot ? slot[f] : f] = xx_finish(z, 0, nullptr, 0, 0); }
        __syncwarp();
    }
}
__global__ void __launch_bounds__(kHashWarps * 32) lizard_frame_hash_kernel(const u8* base, const u64* off, const u64* len, u32 n,
                                                                           u32* out, const u32* slot)
{
    __shared__ __align__(16) uint4 stage[kHashWarps][kHashWords + 1];
    frame_hash_buffers(stage, base, off, len, n, out, slot);
}

// Frame assembly, compressing.  Block k of the call belongs to frame frame_of[k]; blocks of one frame are consecutive,
// starting at first[i] (count nblk[i]).  Record k is 4 + frame_record_payload(len[k], res[k]) bytes.
struct FrameAsm {
    const u8* src; const u64* src_off; const u32* len;    // the blocks' source bytes (the encoder's tables)
    const u8* enc; const u64* enc_off; const int* res;     // their encoded bytes and Lizard_compress results
    const u32* frame_of;                                   // [n_blocks] the block's frame
    u32 n_blocks; int level;
    u64* rec_at;                                           // [n_blocks] record offset from the frame's first byte
    u32 n_frames;
    const u64* first; const u32* nblk;                     // [n_frames] the frame's block range (nblk 0: no blocks)
    const u8* hdr; const u32* hdr_len;                     // [n_frames] header bytes (16 per frame), prepared on the host
    const u32* ccksum; const u32* hash;                    // [n_frames] checksum flag and XXH32 of the frame's source
    u8* dst; const u64* dst_off; const u64* dst_cap;       // where frame i goes, and its room
    const u32* live;                                       // [n_frames] 0: the frame failed on the host, write nothing
    u64* total;                                            // [n_frames] frame size, kFrameTooBig if it does not fit
};
// A 1-byte block's record is 10 bytes, 5 more than the frame bound counts (frame_one_byte_record): a frame whose header
// carries the content size can outgrow a capacity that passed the bound check.  The host call then fails with
// ERROR_dstMaxSize_tooSmall (frame.inl: frame_compress_blocks) or writes its end mark past the capacity; here such a frame
// gets ERROR_dstMaxSize_tooSmall and the assembly writes nothing for it.
constexpr u64 kFrameTooBig = ~0ull;

// Segmented exclusive scan of the record sizes, one warp per frame, 32 records per step.
__global__ void __launch_bounds__(128) lizard_frame_scan_kernel(FrameAsm a)
{
    const u32 lane = threadIdx.x & 31;
    for (u32 f = blockIdx.x * 4 + (threadIdx.x >> 5); f < a.n_frames; f += gridDim.x * 4) {
        if (!a.live[f]) continue;
        u64 at = a.hdr_len[f];
        const u64 b0 = a.first[f];
        const u32 nb = a.nblk[f];
        for (u32 k0 = 0; k0 < nb; k0 += 32) {
            const u32 k = k0 + lane;
            const u64 rec = k < nb ? 4 + (u64)frame_record_payload(a.len[b0 + k], a.res[b0 + k]) : 0;
            u64 inc = rec;
            for (int o = 1; o < 32; o <<= 1) { const u64 t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= (u32)o) inc += t; }
            if (k < nb) a.rec_at[b0 + k] = at + inc - rec;
            at += __shfl_sync(0xffffffffu, inc, 31);
        }
        const u64 total = at + 4 + 4 * (u64)a.ccksum[f];
        if (lane == 0) a.total[f] = total <= a.dst_cap[f] ? total : kFrameTooBig;
    }
}

// Records to their places: CTA per block (its warps take 4 KiB tiles of the payload, as lizard_gather_segments_kernel), then
// per frame the header, the end mark and the checksum.
__global__ void __launch_bounds__(256) lizard_frame_assemble_kernel(FrameAsm a)
{
    const u32 warp = threadIdx.x >> 5;
    for (u32 k = blockIdx.x; k < a.n_blocks; k += gridDim.x) {
        const u32 f = a.frame_of[k];
        if (!a.live[f] || a.total[f] == kFrameTooBig) continue;
        const u32 len = a.len[k];
        const int r = a.res[k];
        const u8* s = a.src + a.src_off[k];
        u8* o = a.dst + a.dst_off[f] + a.rec_at[k];
        if (len == 1) {
            if (threadIdx.x == 0) frame_one_byte_record(o, a.level, s[0]);
            continue;
        }
        const u32 payload = frame_record_payload(len, r);
        if (threadIdx.x < 4) o[threadIdx.x] = (u8)((r > 0 ? (u32)r : (len | 0x80000000u)) >> (8 * threadIdx.x));
        const u8* from = r > 0 ? a.enc + a.enc_off[k] : s;
        for (u32 t = warp * 4096u; t < payload; t += 8u * 4096u) {
            const u32 part = payload - t < 4096u ? payload - t : 4096u;
            lanes_copy_wide<WarpLanes, true, true>(o + 4 + t, from + t, part, false);
        }
    }
    for (u32 f = blockIdx.x; f < a.n_frames; f += gridDim.x) {
        if (!a.live[f] || a.total[f] == kFrameTooBig) continue;
        u8* o = a.dst + a.dst_off[f];
        const u32 h = a.hdr_len[f];
        if (threadIdx.x < h) o[threadIdx.x] = a.hdr[16 * (size_t)f + threadIdx.x];
        const u64 end = a.total[f] - 4 - 4 * (u64)a.ccksum[f];
        if (threadIdx.x < 4) o[end + threadIdx.x] = 0;
        if (a.ccksum[f] && threadIdx.x < 4) o[end + 4 + threadIdx.x] = (u8)(a.hash[f] >> (8 * threadIdx.x));
    }
}

}  // namespace lzb
