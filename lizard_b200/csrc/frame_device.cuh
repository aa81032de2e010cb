// frame_device.cuh -- LizardF frames held in device memory (LizardB200_compressFrames / LizardB200_decompressFrames,
// DESIGN.md 3.4a): the XXH32 routine, the header check and block walk of one frame, and the kernels that run them over
// many frames at once.  XXH32 and the walk are plain serial code that the host shim builds too (host_shim.cpp), so the
// CPU tests pin them against the reference's xxhash.c and frame layer; the kernels are device-only.
//
// Reference: lib/xxhash/xxhash.c (XXH32), lib/lizard_frame.c:756-857 (header), :980-1320 (block loop), format
// doc/lizard_Frame_format.md.
#pragma once
#include "common.cuh"

namespace lzb {

// ---- XXH32 (public algorithm) --------------------------------------------------------------------------------------
constexpr u32 kXxP1 = 2654435761u, kXxP2 = 2246822519u, kXxP3 = 3266489917u, kXxP4 = 668265263u, kXxP5 = 374761393u;
LZ_HD u32 xx_rotl(u32 v, int r) { return (v << r) | (v >> (32 - r)); }
LZ_HD u32 xx_round(u32 acc, u32 in) { return xx_rotl(acc + in * kXxP2, 13) * kXxP1; }
LZ_HD u32 xx_lane_init(u32 seed, u32 lane)
{
    return lane == 0 ? seed + kXxP1 + kXxP2 : lane == 1 ? seed + kXxP2 : lane == 2 ? seed : seed - kXxP1;
}
// the digest from the four lane accumulators (ignored below 16 bytes), the length and the last n % 16 bytes
LZ_HD u32 xx_finish(const u32 v[4], u64 total, const u8* tail, u32 ntail, u32 seed)
{
    u32 h = total >= 16 ? xx_rotl(v[0], 1) + xx_rotl(v[1], 7) + xx_rotl(v[2], 12) + xx_rotl(v[3], 18) : seed + kXxP5;
    h += (u32)total;
    u32 i = 0;
    for (; i + 4 <= ntail; i += 4) h = xx_rotl(h + rd_le32(tail + i) * kXxP3, 17) * kXxP4;
    for (; i < ntail; ++i) h = xx_rotl(h + tail[i] * kXxP5, 11) * kXxP1;
    h ^= h >> 15; h *= kXxP2; h ^= h >> 13; h *= kXxP3; h ^= h >> 16;
    return h;
}
// one thread, one buffer: the header checksum byte, and the host build's content checksum
LZ_HD u32 xxh32_serial(const u8* p, u64 n, u32 seed)
{
    u32 v[4] = { xx_lane_init(seed, 0), xx_lane_init(seed, 1), xx_lane_init(seed, 2), xx_lane_init(seed, 3) };
    const u64 stripes = n / 16;
    for (u64 s = 0; s < stripes; ++s)
        for (int l = 0; l < 4; ++l) v[l] = xx_round(v[l], rd_le32(p + 16 * s + 4 * l));
    return xx_finish(v, n, p + 16 * stripes, (u32)(n % 16), seed);
}

// ---- one frame's header and block chain ------------------------------------------------------------------------------
// Verdicts use the numbering of LizardF_errorCodes (lib/lizard_frame_static.h:56-67); frame.inl ties them to its own.
enum : u32 { kFwOk = 0, kFwGeneric = 1, kFwMaxBlockSize = 2, kFwBlockMode = 3, kFwHeaderVersion = 6, kFwBlockChecksum = 7,
             kFwReserved = 8, kFwDstTooSmall = 11, kFwFrameType = 13, kFwFrameSize = 14, kFwDecompressionFailed = 16,
             kFwHeaderChecksum = 17, kFwContentChecksum = 18 };
// How the bytes after the last complete block end (FrameInfoRec::tail)
enum : u32 { kTailEnd = 0,          // end mark, checksum if flagged, nothing behind
             kTailTrailing = 1,     // the same, followed by more bytes
             kTailTruncated = 2,    // the bytes stop inside a block header, a block or the checksum
             kTailGeneric = 3,      // a block header announces more than the maximum block size
             kTailSkippable = 4 };  // a complete skippable frame (trailing bytes give kTailTrailing with skippable = 1)
struct FrameInfoRec {
    u32 verdict;          // kFwOk, or the header's error (then nothing else is set)
    u32 tail;             // kTail*
    u32 skippable;
    u32 ccksum;           // content checksum flag
    u32 stored_cksum;     // the frame's content checksum word (tail == kTailEnd / kTailTrailing with ccksum)
    u32 max_block;
    u32 n_blocks;         // complete blocks in front of the tail (a truncated block is not counted)
    u32 trunc_block;      // tail kTailTruncated inside a block: 1 compressed, 2 raw (0: inside a header word or the checksum)
    u64 trunc_avail;      // the bytes of that block present
    u64 content_size;     // 0 = not given
};
struct FrameBlockRec {
    u64 src;              // offset of the payload from the frame's first byte
    u32 csize;            // payload bytes
    u32 raw;              // 1 = stored block
};

// A frame block record's payload size for a block of len bytes that compressed to r (0 = did not fit len - 1 bytes): the
// compressed bytes, or the raw block.  A 1-byte block becomes the 6-byte raw inner block the reference produces through its
// wrapped bound check (lizard_frame.c:459 capacity 0, lizard_compress.c:238), written by frame_one_byte_record.
LZ_HD u32 frame_record_payload(u32 len, int r) { return len == 1 ? 6u : (r > 0 ? (u32)r : len); }
LZ_HD void frame_one_byte_record(u8* o, int level, u8 byte)
{
    o[0] = 6; o[1] = 0; o[2] = 0; o[3] = 0;
    o[4] = (u8)level; o[5] = (u8)kFlagRaw; o[6] = 1; o[7] = 0; o[8] = 0; o[9] = byte;
}

// maximum block size of a block size ID (lib/lizard_frame.c:194), 0 for an invalid one; frame.inl's frame_block_size too
LZ_HD u32 frame_block_bytes(u32 bsid)
{
    return bsid == 1 ? 128u << 10 : bsid == 2 ? 256u << 10 : bsid >= 3 && bsid <= 7 ? 1u << (20 + 2 * (bsid - 3)) : 0u;
}

// Header check and block walk of the n bytes at p, as LizardF_decompress (frame.inl) sees them when handed all n bytes at
// once; blocks (if not null) gets the complete blocks, at most `cap` of them.  Serial: one thread per frame.
LZ_HD void frame_walk(const u8* p, u64 n, FrameInfoRec* fi, FrameBlockRec* blocks, u32 cap)
{
    fi->verdict = kFwOk; fi->tail = kTailTruncated; fi->skippable = 0; fi->ccksum = 0; fi->stored_cksum = 0;
    fi->max_block = 0; fi->n_blocks = 0; fi->trunc_block = 0; fi->trunc_avail = 0; fi->content_size = 0;
    if (n < 7) return;                                                      // frame.inl DS_storeHeader waits for 7 bytes
    const u32 magic = rd_le32(p);
    if ((magic & 0xFFFFFFF0u) == 0x184D2A50u) {
        fi->skippable = 1;
        if (n < 8) return;
        const u64 sf = rd_le32(p + 4);
        fi->tail = n - 8 < sf ? kTailTruncated : n - 8 > sf ? kTailTrailing : kTailSkippable;
        return;
    }
    if (magic != 0x184D2206u) { fi->verdict = kFwFrameType; return; }
    const u32 FLG = p[4];
    const u32 fh = ((FLG >> 3) & 1) ? 15u : 7u;
    if (n < fh) return;
    const u32 BD = p[5], bsid = (BD >> 4) & 7;
    if (((FLG >> 6) & 3) != 1) { fi->verdict = kFwHeaderVersion; return; }
    if ((FLG >> 4) & 1) { fi->verdict = kFwBlockChecksum; return; }
    if ((FLG & 3) || (BD & 0x80)) { fi->verdict = kFwReserved; return; }
    if (bsid < 1) { fi->verdict = kFwMaxBlockSize; return; }
    if (BD & 0x0F) { fi->verdict = kFwReserved; return; }
    if ((u8)(xxh32_serial(p + 4, fh - 5, 0) >> 8) != p[fh - 1]) { fi->verdict = kFwHeaderChecksum; return; }
    if (!((FLG >> 5) & 1)) { fi->verdict = kFwBlockMode; return; }             // linked blocks
    fi->ccksum = (FLG >> 2) & 1;
    fi->max_block = frame_block_bytes(bsid);
    if (fh == 15) fi->content_size = rd_le64(p + 6);
    u64 pos = fh;
    u32 nb = 0;
    for (;;) {
        if (n - pos < 4) { fi->tail = kTailTruncated; break; }
        const u32 word = rd_le32(p + pos);
        const u32 csz = word & 0x7FFFFFFFu;
        pos += 4;
        if (csz == 0) {                                                     // end mark (the raw flag does not matter)
            if (fi->ccksum) {
                if (n - pos < 4) { fi->tail = kTailTruncated; break; }
                fi->stored_cksum = rd_le32(p + pos);
                pos += 4;
            }
            fi->tail = pos < n ? kTailTrailing : kTailEnd;
            break;
        }
        if (csz > fi->max_block) { fi->tail = kTailGeneric; break; }
        if (n - pos < csz) { fi->tail = kTailTruncated; fi->trunc_block = 1 + (word >> 31); fi->trunc_avail = n - pos; break; }
        if (blocks && nb < cap) { blocks[nb].src = pos; blocks[nb].csize = csz; blocks[nb].raw = word >> 31; }
        ++nb;
        pos += csz;
    }
    fi->n_blocks = nb;
}

// Where a frame's decoded blocks go and what LizardF_decompress would say, block by block in frame order, given each
// compressed block's Lizard_decompress_safe result at capacity max_block (`r`, ignored for raw blocks) and cap bytes of room.
// Follows frame.inl's batch rule: a compressed block decoded straight into the output (room for a whole block at its
// max-block-spaced slot of the current batch) fails with ERROR_GENERIC, one decoded through the context's one-block buffer
// with ERROR_decompressionFailed.  The state lets the host settle a frame over several decode rounds.
struct FrameSettle {
    u64 dp;                // output bytes so far
    u64 batch_at, batch_k; // the current in-place batch: where it started, slots taken after its first
    u32 in_batch;
    u32 verdict;           // kFwOk so far, or the frame's error
    u32 open;              // 1 while blocks remain to be settled (verdict kFwOk)
};
LZ_HD void frame_settle_begin(const FrameInfoRec& fi, FrameSettle* st)
{
    st->dp = st->batch_at = st->batch_k = 0; st->in_batch = 0; st->verdict = fi.verdict; st->open = 0;
    if (fi.verdict != kFwOk) return;
    if (fi.skippable) { st->verdict = fi.tail == kTailSkippable ? kFwOk : kFwFrameSize; return; }
    st->open = 1;
}
// the next block: returns its offset in the output; on an error closes the frame with that verdict
LZ_HD u64 frame_settle_block(const FrameInfoRec& fi, const FrameBlockRec& b, int r, u64 cap, FrameSettle* st)
{
    const u64 mb = fi.max_block, at = st->dp;
    u32 v = kFwOk;
    if (b.raw) {
        st->in_batch = 0;
        if (b.csize > cap - at) v = kFwDstTooSmall;
        else st->dp += b.csize;
    } else {
        const u64 slot = st->batch_at + (st->batch_k + 1) * mb;
        if (st->in_batch && slot <= cap && cap - slot >= mb) {              // next slot of the same batch
            ++st->batch_k;
            if (r < 0) v = kFwGeneric; else st->dp += (u64)r;
        } else {
            st->in_batch = 0;
            const u64 room = cap - at;
            if (room == 0) v = kFwDstTooSmall;
            else if (room >= mb) {                                          // a new batch, decoded in place
                st->in_batch = 1; st->batch_at = at; st->batch_k = 0;
                if (r < 0) v = kFwGeneric; else st->dp += (u64)r;
            }
            else if (r < 0) v = kFwDecompressionFailed;                     // through the one-block buffer
            else if ((u64)r > room) v = kFwDstTooSmall;
            else st->dp += (u64)r;
        }
    }
    if (v != kFwOk) { st->verdict = v; st->open = 0; }
    return at;
}
// after the frame's last complete block: the verdict of its tail; *check_hash = 1 when the verdict still depends on the
// content checksum over the placed output (frame_settle_hash)
LZ_HD u32 frame_settle_end(const FrameInfoRec& fi, u64 cap, FrameSettle* st, u32* check_hash)
{
    *check_hash = 0;
    st->open = 0;
    const u64 dp = st->dp;
    u32 v = kFwOk;
    if (fi.tail == kTailGeneric) v = kFwGeneric;
    else if (fi.tail == kTailTruncated) {
        // LizardF_decompress stops in a truncated block with input left over when the output is full first: a raw block
        // copies what fits, a compressed one is not started when no room is left
        const u64 room = cap - dp;
        v = (fi.trunc_block == 2 ? fi.trunc_avail > room : fi.trunc_block == 1 && room == 0 && fi.trunc_avail > 0) ? kFwDstTooSmall
                                                                                                               : kFwFrameSize;
    }
    else if (fi.content_size && fi.content_size != dp) v = kFwFrameSize;
    else if (fi.ccksum) *check_hash = 1;
    else if (fi.tail == kTailTrailing) v = kFwFrameSize;
    st->verdict = v;
    return v;
}
// the whole frame at once (the host shim): place[k] for every block, *out = total size
LZ_HD u32 frame_settle(const FrameInfoRec& fi, const FrameBlockRec* blocks, const int* decoded, u64 cap, u64* place,
                       u64* out, u32* check_hash)
{
    FrameSettle st;
    frame_settle_begin(fi, &st);
    *out = 0; *check_hash = 0;
    for (u32 k = 0; st.open && k < fi.n_blocks; ++k) place[k] = frame_settle_block(fi, blocks[k], decoded[k], cap, &st);
    if (!st.open) return st.verdict;
    *out = st.dp;
    return frame_settle_end(fi, cap, &st, check_hash);
}
// the verdict once the content checksum is known (frame_settle gave kFwOk with check_hash)
LZ_HD u32 frame_settle_hash(const FrameInfoRec& fi, u32 hash)
{
    if (hash != fi.stored_cksum) return kFwContentChecksum;
    return fi.tail == kTailTrailing ? kFwFrameSize : kFwOk;
}

// ---- LizardB200_decompressFramesAsync (DESIGN.md 3.4b): admission and settling on the device-side layout -------------------
// Admission is a prefix over frames in index order.  Frame i is admitted while the inclusive sum of the blocks taken by frames
// 0..i stays within max_blocks and the inclusive sum of their slot bytes (one slot of the frame's maximum block size per
// compressed block) within stage_bytes.  A frame whose header fails, a skippable frame and an empty frame take nothing.  The
// kernels apply the two bounds one after the other (the slot bytes are only known once the admitted frames' blocks are
// indexed); both sums grow with i, so the two steps admit the same prefix as the rule above.
constexpr u32 kFwAllocation = 9;                                            // LizardF_ERROR_allocation_failed
LZ_HD u64 frame_plan_blocks(const FrameInfoRec& fi) { return fi.verdict == kFwOk && !fi.skippable ? fi.n_blocks : 0; }
LZ_HD u64 frame_plan_slots(const FrameInfoRec& fi, const FrameBlockRec* blocks)
{
    u64 s = 0;
    const u32 nb = (u32)frame_plan_blocks(fi);
    for (u32 k = 0; k < nb; ++k) s += blocks[k].raw ? 0 : fi.max_block;
    return s;
}
// step 1: blocks before the frame (exclusive sum) and its own; step 2: slot bytes likewise, for a frame that passed step 1
LZ_HD bool frame_admit_blocks(u64 before, u64 blocks, u32 max_blocks) { return before + blocks <= max_blocks; }
LZ_HD bool frame_admit_slots(u64 before, u64 slots, u64 stage_bytes) { return before + slots <= stage_bytes; }
// The staging bytes a call can ever use: max_blocks slots of the largest maximum block size (256 MiB).  A larger stageBytes,
// up to SIZE_MAX for "no bound", admits the same frames, so the call sizes its arena by this and never by more.
LZ_HD u64 frame_stage_limit(u32 max_blocks, u64 stage_bytes)
{
    const u64 most = (u64)max_blocks * frame_block_bytes(7);
    return stage_bytes < most ? stage_bytes : most;
}

// Per-block gather entries of one frame: staged (decoded bytes from the staging arena) and raw (stored bytes from the
// frame).  Length 0 where a block is not placed.
struct FrameGather {
    u64* s_off; u64* s_dst; int* s_len;
    u64* r_off; u64* r_dst; int* r_len;
};
// frame_settle over one admitted frame laid out as the device keeps it: blocks[k], the block's decode result res[k] and its
// staging slot stage[k] (both ignored for raw blocks).  Writes one staged and one raw entry per block, the frame's source at
// src_at and its output at dst_at; returns the verdict before the content checksum (frame_settle).
LZ_HD u32 frame_settle_entries(const FrameInfoRec& fi, const FrameBlockRec* blocks, const int* res, const u64* stage,
                               u64 src_at, u64 dst_at, u64 cap, const FrameGather& g, u64* out, u32* check_hash)
{
    FrameSettle st;
    frame_settle_begin(fi, &st);
    *out = 0; *check_hash = 0;
    const u32 nb = (u32)frame_plan_blocks(fi);
    for (u32 k = 0; k < nb; ++k) {
        const FrameBlockRec b = blocks[k];
        int sl = 0, rl = 0;
        u64 d = dst_at;
        if (st.open) {
            const int r = b.raw ? 0 : res[k];
            d += frame_settle_block(fi, b, r, cap, &st);
            if (st.open && b.raw) rl = (int)b.csize;
            else if (st.open && r > 0) sl = r;
        }
        g.s_off[k] = b.raw ? 0 : stage[k]; g.s_dst[k] = d; g.s_len[k] = sl;
        g.r_off[k] = src_at + b.src;        g.r_dst[k] = d; g.r_len[k] = rl;
    }
    if (!st.open) return st.verdict;
    *out = st.dp;
    return frame_settle_end(fi, cap, &st, check_hash);
}

// ---- LizardF_compressFrame's decisions for one frame --------------------------------------------------------------------------
// The one statement of the frame header and the compression bounds: the host frame API (frame.inl: LizardF_compressBound,
// LizardF_compressFrameBound, LizardF_compressBegin, LizardF_compressFrame, LizardB200_compressFrames) and the planning kernels
// of LizardB200_compressFramesAsync (DESIGN.md 3.4c) run these functions.  Reference: lib/lizard_frame.c:231-312, :363-451.
constexpr u32 kFwCompressionLevel = 5;                                      // LizardF_ERROR_compressionLevel_invalid
// The LizardF_preferences_t fields the header and the bounds read, with the caller's enum values as they are (the enums'
// underlying type is unsigned)
struct FramePrefs { u32 bsid, block_mode, ccksum, auto_flush; u64 content_size; };

// frame.inl's frame_block_size: the block size of an ID, 0 counting as 1; an invalid ID gives LizardF_ERROR_maxBlockSize_invalid
// as a size_t, which the bounds below use as a size like the host code always has
LZ_HD u64 frame_block_size_of(u32 bsid)
{
    const u32 b = frame_block_bytes(bsid == 0 ? 1u : bsid);
    return b ? (u64)b : 0ull - kFwMaxBlockSize;
}
// the smallest block size ID from 128 KiB up to the requested one whose blocks hold the whole input (lizard_frame.c:231-240)
LZ_HD u32 frame_optimal_bsid(u32 req, u64 src_size)
{
    int prop = 1;
    while ((int)req > prop) {
        if (src_size <= frame_block_size_of((u32)prop)) return (u32)prop;
        prop++;
    }
    return req;
}
// LizardF_compressBound (lizard_frame.c:436-451)
LZ_HD u64 frame_compress_bound(u64 src_size, const FramePrefs& p)
{
    const u64 bs = frame_block_size_of(p.bsid);
    const u32 nb = (u32)(src_size / bs) + 1;
    const u64 last = p.auto_flush ? src_size % bs : bs;
    return 4 * (u64)nb + bs * (nb - 1) + last + 4 + (u64)p.ccksum * 4;
}
// LizardF_compressFrameBound (lizard_frame.c:242-247): a header of at most 15 bytes in front
LZ_HD u64 frame_compress_frame_bound(u64 src_size, FramePrefs p)
{
    p.bsid = frame_optimal_bsid(p.bsid, src_size);
    p.auto_flush = 1;
    return 15 + frame_compress_bound(src_size, p);
}
// the preferences LizardF_compressFrame runs a frame of src_size bytes with (lizard_frame.c:260-290): the content size is the
// input's if any is asked for (so none on an empty input), the optimal block size, autoFlush, and a frame of one block
// independent whatever its preferences say
LZ_HD FramePrefs frame_one_shot(FramePrefs p, u64 src_size)
{
    if (p.content_size != 0) p.content_size = src_size;
    p.bsid = frame_optimal_bsid(p.bsid, src_size);
    p.auto_flush = 1;
    if (src_size <= frame_block_size_of(p.bsid)) p.block_mode = 1;
    return p;
}
// LizardF_compressBegin's checks, in its order, and the header it writes to hdr (at most 15 bytes; nothing on an error): block
// size ID (0 counts as 1), block mode, level (level_ok: the level the preferences give passes the GPU's level gate).  Returns
// kFwOk or the error; *block_size and *hdr_len as the host call sets them.
LZ_HD u32 frame_begin(const FramePrefs& p, bool level_ok, u8* hdr, u32* hdr_len, u64* block_size)
{
    const u32 bsid = p.bsid == 0 ? 1u : p.bsid;
    *hdr_len = 0;
    *block_size = frame_block_size_of(bsid);
    if (!frame_block_bytes(bsid)) return kFwMaxBlockSize;
    if (p.block_mode != 1) return kFwBlockMode;
    if (!level_ok) return kFwCompressionLevel;
    wr_le32(hdr, 0x184D2206u);
    hdr[4] = (u8)((1u << 6) + ((p.block_mode & 1) << 5) + ((p.ccksum & 1) << 2) + ((p.content_size > 0) << 3));
    hdr[5] = (u8)((bsid & 7) << 4);
    u32 n = 6;
    if (p.content_size) { wr_le32(hdr + 6, (u32)p.content_size); wr_le32(hdr + 10, (u32)(p.content_size >> 32)); n = 14; }
    hdr[n] = (u8)(xxh32_serial(hdr + 4, n - 4, 0) >> 8);
    *hdr_len = n + 1;
    return kFwOk;
}

// What LizardF_compressFrame decides about one frame before it compresses anything
struct FrameCompressPlan {
    u32 verdict;          // kFwOk; kFwDstTooSmall below LizardF_compressFrameBound; else LizardF_compressBegin's error
    u32 hdr_len;
    u32 ccksum;           // the frame ends with the content checksum
    u32 block_size;
    u64 n_blocks;         // blocks of block_size, the last one shorter
    u64 stage;            // the blocks' lengths, each rounded up to 16: the encoder's output slots
};
// The frame of src_size bytes with cap bytes of room, under the caller's preferences; the header goes to hdr (16 bytes of room).
LZ_HD void frame_compress_plan(const FramePrefs& prefs, bool level_ok, u64 src_size, u64 cap, u8* hdr, FrameCompressPlan* pl)
{
    pl->hdr_len = 0; pl->ccksum = 0; pl->block_size = 0; pl->n_blocks = 0; pl->stage = 0;
    const FramePrefs p = frame_one_shot(prefs, src_size);
    if (cap < frame_compress_frame_bound(src_size, p)) { pl->verdict = kFwDstTooSmall; return; }
    u64 bs;
    pl->verdict = frame_begin(p, level_ok, hdr, &pl->hdr_len, &bs);
    if (pl->verdict != kFwOk) return;
    pl->ccksum = p.ccksum == 1;
    pl->block_size = (u32)bs;
    pl->n_blocks = src_size / bs + (src_size % bs != 0);
    if (pl->n_blocks) pl->stage = (pl->n_blocks - 1) * bs + ((src_size - (pl->n_blocks - 1) * bs + 15) & ~15ull);
}

// LizardB200_compressFramesAsync's admission: a prefix over frames in index order.  Frame i is admitted while the blocks of
// frames 0..i number at most max_blocks and their staging bytes stay within stage_bytes (frame_admit_blocks and
// frame_admit_slots on the two exclusive sums).  A frame that fails its checks, and an empty one, take nothing.  A frame's
// blocks count as at most max_blocks + 1, which decides the same and keeps the sum over 2^32 frames from wrapping.
LZ_HD u64 frame_compress_demand_blocks(const FrameCompressPlan& pl, u32 max_blocks)
{
    if (pl.verdict != kFwOk) return 0;
    return pl.n_blocks <= max_blocks ? pl.n_blocks : (u64)max_blocks + 1;
}
LZ_HD u64 frame_compress_demand_stage(const FrameCompressPlan& pl) { return pl.verdict == kFwOk ? pl.stage : 0; }
// the largest block a frame of these preferences can have: the preferences' block size, 256 MiB for an invalid ID (which
// frame_optimal_bsid may map to any valid one)
LZ_HD u64 frame_compress_top_block(u32 bsid)
{
    const u32 b = frame_block_bytes(bsid == 0 ? 1u : bsid);
    return b ? b : frame_block_bytes(7);
}
// The staging bytes a call can ever use: max_blocks blocks of the top block size.  A larger stage_bytes, up to SIZE_MAX for
// "no bound", admits the same frames, so the call sizes its arena by this and never by more.
LZ_HD u64 frame_compress_stage_limit(u32 max_blocks, u32 bsid, u64 stage_bytes)
{
    const u64 most = (u64)max_blocks * frame_compress_top_block(bsid);
    return stage_bytes < most ? stage_bytes : most;
}

// ---- LizardB200_decompressStream (DESIGN.md 3.4d): the block walk of one chunk, and the running content checksum ------------
// One record per size word the walk reads: where it is (from the walk's first byte), the word, and the decode unit of a
// complete compressed block (-1: no unit).  The last record of a walk that stops on a word is that word.
struct StreamWalkRec { u64 pos; u32 word; int unit; };
enum : u32 { kWalkShort = 0,        // fewer than 4 bytes left for the next size word
             kWalkEnd = 1,          // the end mark (the last record)
             kWalkBadSize = 2,      // a size word above the maximum block size (the last record)
             kWalkPartial = 3,      // a block whose payload is not all there (the last record)
             kWalkRecords = 4,      // the record table is full
             kWalkSlots = 5 };      // a complete compressed block found no decode unit (the last record, unit -1)
// tail: up to 8 bytes behind the end mark (the content checksum), little-endian, tail_n of them present
struct StreamWalk { u32 n_recs, stop, n_units, tail_n; u64 tail; };
// `len` bytes at address src, placed at address dst (the checksum's pieces leave dst 0)
struct StreamSeg { u64 src, dst, len; };
// The records of the n bytes at p, which start on a size word, with frame_walk's checks: at most max_recs records, and
// compressed blocks take decode units 1..slots (unit 0 is the carried block's) with u_src the payload's address and u_len its
// size.  Serial: one thread.
LZ_HD StreamWalk frame_stream_walk(const u8* p, u64 n, u32 max_block, StreamWalkRec* rec, u32 max_recs, u32 slots, u64* u_src,
                                   u32* u_len)
{
    StreamWalk w = { 0, kWalkShort, 0, 0, 0 };
    u64 pos = 0;
    for (;;) {
        if (n - pos < 4) { w.stop = kWalkShort; break; }
        if (w.n_recs == max_recs) { w.stop = kWalkRecords; break; }
        const u32 word = rd_le32(p + pos), csz = word & 0x7FFFFFFFu;
        StreamWalkRec& r = rec[w.n_recs++];
        r.pos = pos; r.word = word; r.unit = -1;
        if (csz == 0) {
            w.stop = kWalkEnd;
            for (u64 k = pos + 4; k < n && w.tail_n < 8; ++k) w.tail |= (u64)p[k] << (8 * w.tail_n++);
            break;
        }
        if (csz > max_block) { w.stop = kWalkBadSize; break; }
        if (n - pos - 4 < csz) { w.stop = kWalkPartial; break; }
        if (!(word >> 31)) {
            if (w.n_units == slots) { w.stop = kWalkSlots; break; }
            r.unit = (int)++w.n_units;
            u_src[w.n_units] = (u64)(size_t)(p + pos + 4); u_len[w.n_units] = csz;
        }
        pos += 4 + csz;
    }
    return w;
}

// XXH32 (seed 0) over bytes that arrive in pieces: the four accumulators, the length so far and the bytes short of a stripe
struct StreamHashState { u32 v[4]; u64 total; u32 nbuf, pad; u8 buf[16]; };
LZ_HD void xx_stream_reset(StreamHashState* s)
{
    for (u32 l = 0; l < 4; ++l) s->v[l] = xx_lane_init(0, l);
    s->total = 0; s->nbuf = 0; s->pad = 0;
    for (u32 i = 0; i < 16; ++i) s->buf[i] = 0;
}
LZ_HD void xx_stream_update(StreamHashState* s, const u8* p, u64 n)
{
    s->total += n;
    while (n) {
        s->buf[s->nbuf++] = *p++; --n;
        if (s->nbuf == 16) { for (u32 l = 0; l < 4; ++l) s->v[l] = xx_round(s->v[l], rd_le32(s->buf + 4 * l)); s->nbuf = 0; }
    }
}
LZ_HD u32 xx_stream_digest(const StreamHashState* s) { return xx_finish(s->v, s->total, s->buf, s->nbuf, 0); }

}  // namespace lzb
