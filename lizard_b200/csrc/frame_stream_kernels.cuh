// frame_stream_kernels.cuh -- the kernels of LizardB200_decompressStream (DESIGN.md 3.4d).  Included by api.cu; the serial
// routines they run are in frame_device.cuh, the decisions in frame_stream.h.
#pragma once
#include "frame_device.cuh"

namespace lzb {

// One round's walk: thread 0 walks the chunk from p (frame_stream_walk) and sets the carried block as unit 0; then every
// thread lays out the decode units' slots (unit k at k * max_block, room max_block) and gives the units the walk left
// without a block length 0.  hdr gets the walk's summary.
__global__ void __launch_bounds__(128) lizard_frame_stream_walk_kernel(const u8* p, u64 n, u32 max_block, const u8* carry,
                                                                       u32 carry_len, StreamWalkRec* rec, u32 max_recs,
                                                                       u32 slots, StreamWalk* hdr, u64* u_src, u32* u_len,
                                                                       u64* u_stage, u32* u_cap)
{
    __shared__ u32 units;
    if (threadIdx.x == 0) {
        const StreamWalk w = frame_stream_walk(p, n, max_block, rec, max_recs, slots, u_src, u_len);
        u_src[0] = (u64)(size_t)carry; u_len[0] = carry_len;
        *hdr = w;
        units = w.n_units;
    }
    __syncthreads();
    for (u32 k = threadIdx.x; k <= slots; k += blockDim.x) {
        u_stage[k] = (u64)k * max_block; u_cap[k] = max_block;
        if (k > units) { u_src[k] = 0; u_len[k] = 0; }
    }
}

// A stream's content checksum over n segments in order, on one warp: the warp stages up to kHashPiece bytes behind the
// bytes short of a stripe (aligned 16-byte loads), lanes 0-3 run the four accumulators over the whole stripes (as
// frame_hash_buffers), and what is left is moved to the front.  The recurrence is serial: one warp's rate.  seg(i, &p, &L)
// gives segment i; buf is the warp's kHashPiece + 16 bytes of shared memory.
template <class Seg> __device__ __forceinline__ void stream_hash_segments(Seg seg, u32 n, StreamHashState* st, u8* buf)
{
    const u32 lane = threadIdx.x;
    u32 v = lane < 4 ? st->v[lane] : 0;
    u32 nb = st->nbuf;
    if (lane < nb) buf[lane] = st->buf[lane];
    u64 total = st->total;
    __syncwarp();
    for (u32 i = 0; i < n; ++i) {
        const u8* p;
        u64 L;
        seg(i, &p, &L);
        total += L;
        for (u64 done = 0; done < L;) {
            const u32 take = (u32)(L - done < kHashPiece - nb ? L - done : kHashPiece - nb);
            {   // aligned 16-byte loads of the words holding the piece (as frame_hash_buffers), bytes to their places
                const u8* from = p + done;
                const uint4* a = (const uint4*)((size_t)from & ~(size_t)15);
                const u32 head = (u32)((size_t)from & 15), words = (head + take + 15) / 16;
                for (u32 w = lane; w < words; w += 32) {
                    const uint4 q = a[w];
                    const u32 x[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
                    for (u32 j = 0; j < 16; ++j) {
                        const int k = (int)(16 * w + j) - (int)head;
                        if (k >= 0 && k < (int)take) buf[nb + k] = (u8)(x[j >> 2] >> (8 * (j & 3)));
                    }
                }
            }
            __syncwarp();
            nb += take; done += take;
            const u32 stripes = nb / 16;
            if (lane < 4)
                for (u32 s = 0; s < stripes; ++s) v = xx_round(v, *(const u32*)(buf + 16 * s + 4 * lane));
            const u32 left = nb - 16 * stripes;
            const u8 t = lane < left ? buf[16 * stripes + lane] : 0;
            __syncwarp();
            if (lane < left) buf[lane] = t;
            __syncwarp();
            nb = left;
        }
    }
    if (lane < 4) st->v[lane] = v;
    if (lane < nb) st->buf[lane] = buf[lane];
    if (lane == 0) { st->total = total; st->nbuf = nb; }
}
// LizardB200_decompressStream's pieces: a segment list in device memory
__global__ void __launch_bounds__(32) lizard_frame_stream_hash_kernel(const StreamSeg* seg, u32 n, StreamHashState* st)
{
    __shared__ __align__(16) u8 buf[kHashPiece + 16];
    stream_hash_segments([seg](u32 i, const u8** p, u64* L) { *p = (const u8*)(size_t)seg[i].src; *L = seg[i].len; }, n, st, buf);
}

}  // namespace lzb
