// frame_cstream_kernels.cuh -- the kernels of LizardB200_compressStream* (DESIGN.md 3.4e).  Included by api.cu after encode.cuh
// and frame_stream_kernels.cuh; the decisions are in frame_cstream.h, the block records' rule in frame_device.cuh.
#pragma once
#include "frame_cstream.h"
#include "frame_stream_kernels.cuh"
#include "lanes.cuh"

namespace lzb {

// A stream's device-side state besides the carried block: the running checksum, and where the current call's next record goes
// (from the call's dDst; kCStreamTooBig once a record did not fit the call's capacity)
struct CStreamDev { StreamHashState hash; u64 off; };
constexpr u64 kCStreamTooBig = ~0ull;
// One round's block table (unit k: source address, length, encoder slot, capacity, result, record offset)
struct CStreamTab { u64* src; u32* len; u64* enc; u32* cap; int* res; u64* rec; };
// The frame header LizardF_compressBegin decided on the host, passed by value
struct CStreamHeader { u8 b[16]; u32 n; };

// Begin: the header to dst, the checksum reset, the header's length to *written
__global__ void __launch_bounds__(32) lizard_cstream_begin_kernel(CStreamHeader h, u8* dst, CStreamDev* st, size_t* written)
{
    if (threadIdx.x == 0) {
#pragma unroll
        for (u32 i = 0; i < 16; ++i) if (i < h.n) dst[i] = h.b[i];
        xx_stream_reset(&st->hash);
        st->off = 0;
        if (written) *written = h.n;
    }
}

// A round's block table from scalars (cstream_unit)
__global__ void __launch_bounds__(256) lizard_cstream_plan_kernel(u64 carry, u64 carry_len, u64 p, u64 n, u64 bs, u64 stride, u32 units,
                                                                  CStreamTab t)
{
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < units; k += gridDim.x * blockDim.x)
        cstream_unit(k, carry, carry_len, p, n, bs, stride, &t.src[k], &t.len[k], &t.enc[k], &t.cap[k]);
}

// The round's record offsets: an exclusive scan of the record sizes (4 + frame_record_payload) from where the call's previous
// round ended (first: from 0), in one CTA.  A round whose records would pass the call's capacity marks the call kCStreamTooBig.
constexpr u32 kCScanThreads = 1024;
__global__ void __launch_bounds__(kCScanThreads) lizard_cstream_scan_kernel(CStreamTab t, u32 units, u32 first, u64 cap, CStreamDev* st)
{
    __shared__ u64 warp_sum[kCScanThreads / 32];
    __shared__ u64 base;
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) base = first ? 0 : st->off;
    __syncthreads();
    if (base == kCStreamTooBig) return;
    for (u32 k0 = 0; k0 < units; k0 += kCScanThreads) {
        const u32 k = k0 + threadIdx.x;
        const u64 rec = k < units ? 4 + (u64)frame_record_payload(t.len[k], t.res[k]) : 0;
        u64 inc = rec;
        for (int o = 1; o < 32; o <<= 1) { const u64 v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= (u32)o) inc += v; }
        if (lane == 31) warp_sum[warp] = inc;
        __syncthreads();
        if (warp == 0) {
            u64 w = warp_sum[lane], wi = w;
            for (int o = 1; o < 32; o <<= 1) { const u64 v = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= (u32)o) wi += v; }
            warp_sum[lane] = wi - w;                                        // exclusive over the warps
        }
        __syncthreads();
        if (k < units) t.rec[k] = base + warp_sum[warp] + inc - rec;
        __syncthreads();
        if (threadIdx.x == kCScanThreads - 1) base += warp_sum[warp] + inc;
        __syncthreads();
    }
    if (threadIdx.x == 0) st->off = base <= cap ? base : kCStreamTooBig;
}

// Records to their places at dst + rec[k]: CTA per block, its warps take 4 KiB tiles of the payload (as
// lizard_frame_assemble_kernel); a block that did not shrink is stored raw, a 1-byte block is frame_one_byte_record
__global__ void __launch_bounds__(256) lizard_cstream_assemble_kernel(CStreamTab t, u32 units, const u8* enc, u8* dst, int level,
                                                                      const CStreamDev* st)
{
    if (st->off == kCStreamTooBig) return;
    const u32 warp = threadIdx.x >> 5;
    for (u32 k = blockIdx.x; k < units; k += gridDim.x) {
        const u32 len = t.len[k];
        const int r = t.res[k];
        const u8* s = (const u8*)(size_t)t.src[k];
        u8* o = dst + t.rec[k];
        if (len == 1) {
            if (threadIdx.x == 0) frame_one_byte_record(o, level, s[0]);
            continue;
        }
        const u32 payload = frame_record_payload(len, r);
        if (threadIdx.x < 4) o[threadIdx.x] = (u8)((r > 0 ? (u32)r : (len | 0x80000000u)) >> (8 * threadIdx.x));
        const u8* from = r > 0 ? enc + t.enc[k] : s;
        for (u32 q = warp * 4096u; q < payload; q += 8u * 4096u) {
            const u32 part = payload - q < 4096u ? payload - q : 4096u;
            lanes_copy_wide<WarpLanes, true, true>(o + 4 + q, from + q, part, false);
        }
    }
}

// The checksum over the chunk, on one warp (stream_hash_segments, as lizard_frame_stream_hash_kernel), the segment by value
__global__ void __launch_bounds__(32) lizard_cstream_hash_kernel(const u8* p, u64 n, CStreamDev* st)
{
    __shared__ __align__(16) u8 buf[kHashPiece + 16];
    stream_hash_segments([p, n](u32, const u8** q, u64* L) { *q = p; *L = n; }, 1, &st->hash, buf);
}

// The call's result: the bytes its rounds wrote (none ran: 0), with `end` the end mark and the checksum behind them; a host
// error replaces the size.  A call whose records passed its capacity gets ERROR_dstMaxSize_tooSmall and no end mark.
__global__ void __launch_bounds__(32) lizard_cstream_finish_kernel(u32 rounds, u8* dst, u32 end, u32 ccksum, u64 err, CStreamDev* st,
                                                                   size_t* written)
{
    if (threadIdx.x != 0) return;
    u64 o = rounds ? st->off : 0;
    if (o == kCStreamTooBig) { if (written) *written = (size_t)(0ull - (u64)kFwDstTooSmall); return; }
    if (end) {
        dst[o] = dst[o + 1] = dst[o + 2] = dst[o + 3] = 0;
        o += 4;
        if (ccksum) { wr_le32(dst + o, xx_stream_digest(&st->hash)); o += 4; }
    }
    if (written) *written = err ? (size_t)err : (size_t)o;
}

}  // namespace lzb
