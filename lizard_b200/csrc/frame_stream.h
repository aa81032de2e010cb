// frame_stream.h -- LizardF_decompress's decisions, stated once over a memory backend (DESIGN.md 3.4d).
//
// frame.inl runs frame_decompress_run with host memory (LizardF_decompress: the bytes are read where they are, complete
// compressed blocks are decoded in pipelined batches) and with device memory (LizardB200_decompressStream: StreamIO below,
// whose device work -- walk, decode, placement, checksum -- an executor enqueues).  The host shim builds both with host
// memory and the one-lane decoder, so the CPU tests compare the state machine and StreamIO with the reference's frame layer.
//
// Reference: lib/lizard_frame.c:756-857 (header), :980-1320 (the state machine), format doc/lizard_Frame_format.md.
#pragma once
#include "frame_device.cuh"
#include "../../include/lizard_b200.h"
#include <algorithm>
#include <cstring>
#include <new>
#include <stdexcept>
#include <vector>

namespace lzb {

// ---- frame constants / errors (lib/lizard_frame_static.h:56-67) ----
enum : int { FE_OK = 0, FE_GENERIC, FE_maxBlockSize_invalid, FE_blockMode_invalid, FE_contentChecksumFlag_invalid,
             FE_compressionLevel_invalid, FE_headerVersion_wrong, FE_blockChecksum_unsupported, FE_reservedFlag_set,
             FE_allocation_failed, FE_srcSize_tooLarge, FE_dstMaxSize_tooSmall, FE_frameHeader_incomplete,
             FE_frameType_unknown, FE_frameSize_wrong, FE_srcPtr_wrong, FE_decompressionFailed,
             FE_headerChecksum_invalid, FE_contentChecksum_invalid, FE_maxCode };
inline size_t ferr(int e) { return (size_t)-(long)e; }
inline bool fe_is_error(size_t code) { return code > (size_t)-(long)FE_maxCode; }   // LizardF_isError
constexpr u32 kFrameMagic = 0x184D2206u, kSkippableMagic = 0x184D2A50u, kRawFlag = 0x80000000u;
constexpr size_t kMinFH = 7, kMaxFH = 15, kBH = 4;
enum { DS_getHeader = 0, DS_storeHeader, DS_getCBlockSize, DS_storeCBlockSize, DS_copyDirect, DS_getCBlock,
       DS_storeCBlock, DS_flushOut, DS_getSuffix, DS_storeSuffix, DS_getSFrameSize, DS_storeSFrameSize, DS_skipSkippable };

// a compressed block of a batch: its payload in the span, its size, and its slot in the output (max_block apart)
struct FrameBlockRef { size_t src_pos; u32 csize; size_t dst_pos; };

// What a decompression context keeps between calls besides its buffers (the carried block, the one-block output buffer and
// the content checksum, which the backend owns)
struct FrameDState {
    LizardF_frameInfo_t info;
    int stage;                              // DS_*
    u64 remaining;                          // frameRemainingSize
    size_t max_block;
    const u8* src_expect;
    size_t tmp_in_size, tmp_in_target;
    size_t tmp_out_size, tmp_out_start;
    u8 header[16];                          // a frame or skippable header arriving in pieces
    u8 word[4];                             // a size word or the content checksum arriving in pieces
    void reset()
    {
        memset(&info, 0, sizeof info);
        stage = DS_getHeader; remaining = 0; max_block = 0; src_expect = nullptr;
        tmp_in_size = tmp_in_target = tmp_out_size = tmp_out_start = 0;
    }
};

// The backend (IO) a run goes through.  Pointers into the input and the output are the caller's; p/n name source bytes.
//   const u8* view(p, n, buf)    the n <= 15 bytes at p, readable here (p itself, or buf filled)
//   void load(to, p, n)          n source bytes into the context's small buffers (header, word)
//   u32 word(p)                  the little-endian size word at p
//   bool ready()                 the device can take work (else ERROR_GENERIC)
//   void hash_reset()            start the content checksum
//   void frame_buffers(mb)       the carried block and the one-block buffer hold a block of mb bytes (may throw bad_alloc)
//   void copy(to, p, n)          stored bytes to the output
//   void hash(q, n)              the content checksum takes the n bytes at q (source or output)
//   int decode_batch(...)        a batch of complete compressed blocks at max_block spacing from dp, compacted in order at
//                                dp by place(); -1 on a failure of the batch, else 1 if the checksum was taken beside it
//   void place(w, from, i, n)    block i of the batch, decoded at `from`, to w
//   int decode_tmp(p, n)         the compressed block at p into the one-block buffer: its size, or -1
//   void hash_tmp(n)             the checksum takes the one-block buffer's first n bytes
//   void carry(at, p, n)         source bytes to the carried block at offset `at`
//   int decode_carry(p, to, n)   the carried block of n bytes to `to` (null: the one-block buffer); p: where the source is
//   void flush_out(to, at, n)    the one-block buffer's bytes [at, at + n) to the output
//   bool digest_ok(word)         the content checksum equals word
template <class IO> size_t frame_decode_header(FrameDState* d, IO& io, const u8* p, size_t n)
{   // lib/lizard_frame.c:756-857
    if (n < kMinFH) return ferr(FE_frameHeader_incomplete);
    memset(&d->info, 0, sizeof d->info);
    if ((rd_le32(p) & 0xFFFFFFF0u) == kSkippableMagic) {
        d->info.frameType = LizardF_skippableFrame;
        if (p == d->header) { d->tmp_in_size = n; d->tmp_in_target = 8; d->stage = DS_storeSFrameSize; return n; }
        d->stage = DS_getSFrameSize; return 4;
    }
    if (rd_le32(p) != kFrameMagic) return ferr(FE_frameType_unknown);
    d->info.frameType = LizardF_frame;
    const u8 FLG = p[4];
    const unsigned version = (FLG >> 6) & 3, block_mode = (FLG >> 5) & 1, block_cksum = (FLG >> 4) & 1,
                   csize_flag = (FLG >> 3) & 1, ccksum = (FLG >> 2) & 1;
    const size_t fh = csize_flag ? kMaxFH : kMinFH;
    if (n < fh) {
        if (p != d->header) memcpy(d->header, p, n);
        d->tmp_in_size = n; d->tmp_in_target = fh; d->stage = DS_storeHeader;
        return n;
    }
    const u8 BD = p[5];
    const unsigned bsid = (BD >> 4) & 7;
    if (version != 1) return ferr(FE_headerVersion_wrong);
    if (block_cksum) return ferr(FE_blockChecksum_unsupported);
    if (FLG & 3) return ferr(FE_reservedFlag_set);
    if (BD & 0x80) return ferr(FE_reservedFlag_set);
    if (bsid < 1) return ferr(FE_maxBlockSize_invalid);
    if (BD & 0x0F) return ferr(FE_reservedFlag_set);
    if ((u8)(xxh32_serial(p + 4, fh - 5, 0) >> 8) != p[fh - 1]) return ferr(FE_headerChecksum_invalid);
    d->info.blockMode = (LizardF_blockMode_t)block_mode;
    d->info.contentChecksumFlag = (LizardF_contentChecksum_t)ccksum;
    d->info.blockSizeID = (LizardF_blockSizeID_t)bsid;
    d->max_block = frame_block_size_of(bsid);
    d->remaining = 0;
    if (csize_flag) d->remaining = d->info.contentSize = rd_le64(p + 6);
    if (ccksum) io.hash_reset();
    if (block_mode != LizardF_blockIndependent) return ferr(FE_blockMode_invalid);      // linked blocks: out of scope
    io.frame_buffers(d->max_block);
    d->tmp_in_size = d->tmp_in_target = 0; d->tmp_out_size = d->tmp_out_start = 0;
    d->stage = DS_getCBlockSize;
    return fh;
}

// LizardF_decompress (lib/lizard_frame.c:980-1320) for independent blocks: whole runs of complete compressed blocks with room
// in the output are one batch.  *srcSizePtr / *dstSizePtr: the input and the room on entry, what was consumed and produced on
// return.
template <class IO>
size_t frame_decompress_run(FrameDState* d, IO& io, const u8* s0, size_t* srcSizePtr, u8* d0, size_t* dstSizePtr)
{
    const u8* const se = s0 + *srcSizePtr; const u8* sp = s0;
    u8* const de = d0 + *dstSizePtr; u8* dp = d0;
    u32 word = 0;
    bool again = true;
    size_t hint = 1;
    *srcSizePtr = 0; *dstSizePtr = 0;
    if (d->src_expect && s0 != d->src_expect) return ferr(FE_srcPtr_wrong);

    while (again) {
        switch (d->stage) {
        case DS_getHeader:
            if ((size_t)(se - sp) >= kMaxFH) {
                u8 buf[kMaxFH];
                size_t h = frame_decode_header(d, io, io.view(sp, kMaxFH, buf), (size_t)(se - sp));
                if (fe_is_error(h)) return h;
                sp += h;
                break;
            }
            d->tmp_in_size = 0; d->tmp_in_target = kMinFH; d->stage = DS_storeHeader;
            /* fallthrough */
        case DS_storeHeader: {
            size_t n = d->tmp_in_target - d->tmp_in_size;
            if (n > (size_t)(se - sp)) n = (size_t)(se - sp);
            io.load(d->header + d->tmp_in_size, sp, n);
            d->tmp_in_size += n; sp += n;
            if (d->tmp_in_size < d->tmp_in_target) { hint = (d->tmp_in_target - d->tmp_in_size) + kBH; again = false; break; }
            size_t h = frame_decode_header(d, io, d->header, d->tmp_in_target);
            if (fe_is_error(h)) return h;
            break; }
        case DS_getCBlockSize:
            if ((size_t)(se - sp) >= kBH) { word = io.word(sp); sp += kBH; }
            else { d->tmp_in_size = 0; d->stage = DS_storeCBlockSize; }
            if (d->stage == DS_storeCBlockSize)
        case DS_storeCBlockSize: {
                size_t n = kBH - d->tmp_in_size;
                if (n > (size_t)(se - sp)) n = (size_t)(se - sp);
                io.load(d->word + d->tmp_in_size, sp, n);
                sp += n; d->tmp_in_size += n;
                if (d->tmp_in_size < kBH) { hint = kBH - d->tmp_in_size; again = false; break; }
                word = rd_le32(d->word);
            }
            {   const size_t csz = word & 0x7FFFFFFFu;
                if (csz == 0) { d->stage = DS_getSuffix; break; }
                if (csz > d->max_block) return ferr(FE_GENERIC);
                d->tmp_in_target = csz;
                if (word & kRawFlag) { d->stage = DS_copyDirect; break; }
                d->stage = DS_getCBlock;
                if (dp == de) { hint = csz + kBH; again = false; }
                break; }
        case DS_copyDirect: {
            size_t n = d->tmp_in_target;
            if ((size_t)(se - sp) < n) n = (size_t)(se - sp);
            if ((size_t)(de - dp) < n) n = (size_t)(de - dp);
            io.copy(dp, sp, n);
            if (d->info.contentChecksumFlag) io.hash(sp, n);
            if (d->info.contentSize) d->remaining -= n;
            sp += n; dp += n;
            if (n == d->tmp_in_target) { d->stage = DS_getCBlockSize; break; }
            d->tmp_in_target -= n; hint = d->tmp_in_target + kBH; again = false;
            break; }
        case DS_getCBlock: {
            if ((size_t)(se - sp) < d->tmp_in_target) { d->tmp_in_size = 0; d->stage = DS_storeCBlock; break; }
            // ---- batch: this block and every following complete compressed block that has room in dst ----
            if (!io.ready()) return ferr(FE_GENERIC);
            std::vector<FrameBlockRef> blocks;
            const u8* scan = sp; size_t csz = d->tmp_in_target; u8* out = dp;
            const u8* span_begin = sp;
            if ((size_t)(de - out) >= d->max_block) {
                for (;;) {
                    blocks.push_back({ (size_t)(scan - span_begin), (u32)csz, (size_t)(out - dp) });
                    scan += csz; out += d->max_block;
                    if ((size_t)(se - scan) < kBH) break;                      // next size word not here yet
                    const u32 w = io.word(scan);
                    const size_t nx = w & 0x7FFFFFFFu;
                    if (nx == 0 || (w & kRawFlag) || nx > d->max_block || (size_t)(se - scan - kBH) < nx) break;
                    if ((size_t)(de - out) < d->max_block) break;              // that one needs the tmp-out path
                    scan += kBH; csz = nx;                                     // take it into this batch
                }
            }
            if (blocks.empty()) {                                          // not enough room in dst: decode via tmp_out
                const int r = io.decode_tmp(sp, d->tmp_in_target);
                if (r < 0) return ferr(FE_decompressionFailed);
                sp += d->tmp_in_target;
                if (d->info.contentChecksumFlag) io.hash_tmp((size_t)r);
                if (d->info.contentSize) d->remaining -= (u64)r;
                d->tmp_out_size = (size_t)r; d->tmp_out_start = 0; d->stage = DS_flushOut;
                break;
            }
            // blocks are decoded at max_block spacing, then compacted into dst in order: full blocks land exactly in place,
            // a short block (the last of a frame) only shifts what follows it
            std::vector<int> sz;
            const int hashed = io.decode_batch(span_begin, (size_t)(scan - span_begin), blocks, dp, d->max_block, sz,
                                               d->info.contentChecksumFlag != 0);
            if (hashed < 0) return ferr(FE_GENERIC);
            u8* w = dp;
            for (size_t i = 0; i < blocks.size(); ++i) {
                if (sz[i] < 0) return ferr(FE_GENERIC);
                io.place(w, dp + blocks[i].dst_pos, i, (size_t)sz[i]);
                if (d->info.contentChecksumFlag && !hashed) io.hash(w, (size_t)sz[i]);
                if (d->info.contentSize) d->remaining -= (u64)sz[i];
                w += sz[i];
            }
            dp = w; sp = scan;
            d->stage = DS_getCBlockSize;
            break; }
        case DS_storeCBlock: {
            size_t n = d->tmp_in_target - d->tmp_in_size;
            if (n > (size_t)(se - sp)) n = (size_t)(se - sp);
            io.carry(d->tmp_in_size, sp, n);
            d->tmp_in_size += n; sp += n;
            if (d->tmp_in_size < d->tmp_in_target) { hint = (d->tmp_in_target - d->tmp_in_size) + kBH; again = false; break; }
            if (!io.ready()) return ferr(FE_GENERIC);
            const bool direct = (size_t)(de - dp) >= d->max_block;
            const int r = io.decode_carry(sp, direct ? dp : nullptr, d->tmp_in_target);
            if (r < 0) return direct ? ferr(FE_GENERIC) : ferr(FE_decompressionFailed);
            if (d->info.contentChecksumFlag) { if (direct) io.hash(dp, (size_t)r); else io.hash_tmp((size_t)r); }
            if (d->info.contentSize) d->remaining -= (u64)r;
            if (direct) { dp += r; d->stage = DS_getCBlockSize; }
            else { d->tmp_out_size = (size_t)r; d->tmp_out_start = 0; d->stage = DS_flushOut; }
            break; }
        case DS_flushOut: {
            size_t n = d->tmp_out_size - d->tmp_out_start;
            if (n > (size_t)(de - dp)) n = (size_t)(de - dp);
            io.flush_out(dp, d->tmp_out_start, n);
            d->tmp_out_start += n; dp += n;
            if (d->tmp_out_start == d->tmp_out_size) { d->stage = DS_getCBlockSize; break; }
            hint = kBH; again = false;
            break; }
        case DS_getSuffix: {
            const size_t suffix = (size_t)d->info.contentChecksumFlag * 4;
            if (d->remaining) return ferr(FE_frameSize_wrong);
            if (suffix == 0) { hint = 0; d->stage = DS_getHeader; again = false; break; }
            if ((size_t)(se - sp) < 4) { d->tmp_in_size = 0; d->stage = DS_storeSuffix; }
            else { u8 b[4]; io.load(b, sp, 4); word = rd_le32(b); sp += 4; }
            }
            if (d->stage == DS_storeSuffix)
        case DS_storeSuffix: {
                size_t n = 4 - d->tmp_in_size;
                if (n > (size_t)(se - sp)) n = (size_t)(se - sp);
                io.load(d->word + d->tmp_in_size, sp, n);
                sp += n; d->tmp_in_size += n;
                if (d->tmp_in_size < 4) { hint = 4 - d->tmp_in_size; again = false; break; }
                word = rd_le32(d->word);
            }
            {   if (!io.digest_ok(word)) return ferr(FE_contentChecksum_invalid);
                hint = 0; d->stage = DS_getHeader; again = false;
                break; }
        case DS_getSFrameSize:
            if ((size_t)(se - sp) >= 4) { u8 b[4]; io.load(b, sp, 4); word = rd_le32(b); sp += 4; }
            else { d->tmp_in_size = 4; d->tmp_in_target = 8; d->stage = DS_storeSFrameSize; }
            if (d->stage == DS_storeSFrameSize)
        case DS_storeSFrameSize: {
                size_t n = d->tmp_in_target - d->tmp_in_size;
                if (n > (size_t)(se - sp)) n = (size_t)(se - sp);
                io.load(d->header + d->tmp_in_size, sp, n);
                sp += n; d->tmp_in_size += n;
                if (d->tmp_in_size < d->tmp_in_target) { hint = d->tmp_in_target - d->tmp_in_size; again = false; break; }
                word = rd_le32(d->header + 4);
            }
            {   const size_t sf = word;
                d->info.contentSize = sf; d->tmp_in_target = sf; d->stage = DS_skipSkippable;
                break; }
        case DS_skipSkippable: {
            size_t n = d->tmp_in_target;
            if (n > (size_t)(se - sp)) n = (size_t)(se - sp);
            sp += n; d->tmp_in_target -= n;
            again = false; hint = d->tmp_in_target;
            if (hint) break;
            d->stage = DS_getHeader;
            break; }
        }
    }
    d->src_expect = sp < se ? sp : nullptr;
    *srcSizePtr = (size_t)(sp - s0);
    *dstSizePtr = (size_t)(dp - d0);
    return hint;
}

// ---- LizardB200_decompressStream: the backend over device memory ---------------------------------------------------------------
// The stream's buffers, kept between calls: the carried block, the one-block buffer and the running checksum (device
// memory), and where the one-block buffer's bytes are (the buffer, or a staging slot of the current call)
struct StreamBuffers {
    u8* carry = nullptr; u8* tmp_out = nullptr; size_t block = 0;
    StreamHashState* hash = nullptr;
    const u8* tmp_at = nullptr;
};
// At most this many records per walk, and this many staging bytes per round; a call's decode units are fixed by the chunk
// length and the output's room (stream_round_shape), so its launch sequence does not depend on what the chunk holds.
constexpr u32 kStreamMaxRecords = 16384;
constexpr size_t kStreamStageBudget = (size_t)1 << 30;
// the records a walk of n bytes may find (a complete block takes at least 5 bytes) and the compressed blocks it may decode:
// no more than fit the stage budget, nor more than the output's room can take in one call plus the one-block buffer's.
// Rounds only run inside a frame's blocks, where max_block is set; 0 is taken as 1 so that the shape stays defined.
LZ_HD void stream_round_shape(u64 n, u64 room, u64 max_block, u32* max_recs, u32* slots)
{
    const u64 r = n / 5 + 2;
    *max_recs = (u32)(r < kStreamMaxRecords ? r : kStreamMaxRecords);
    if (max_block == 0) max_block = 1;
    u64 s = kStreamStageBudget / max_block;
    const u64 by_room = room / max_block + 2;
    if (by_room < s) s = by_room;
    if (*max_recs < s) s = *max_recs;
    *slots = (u32)(s ? s : 1);
}

// The device side of one call.  Source bytes are read through rounds: a round walks the chunk from a size word (the
// executor's walk), decodes every complete compressed block it found that has a unit, plus the carried block as unit 0, into
// staging slots of max_block, and brings back the records and the results in one read-back.  The state machine then asks
// for words and results by address.  Placements and checksum pieces are collected in order and enqueued when the staging
// is about to be reused and when the call ends (finish).  Exec (frame.inl: device kernels; host_shim.cpp: host memory):
//   void read(host, p, n)      n bytes at p to host memory, synchronously
//   void copy(to, from, n)     in stream order
//   void round(p, n, max_block, carry, carry_len, max_recs, slots, walk, recs, res, stage)
//                              the walk of the n bytes at p and the decode of its units; *stage = the staging arena (unit k
//                              at *stage + k * max_block)
//   void gather(segs)          the segments to their places (one launch; the destinations do not overlap)
//   void hash(segs, state)     the running checksum over the segments in order
//   void hash_reset(state)
//   u32 digest(state)          synchronises
//   void sync()
//   void buffers(sb, block)    the carried block and the one-block buffer hold `block` bytes
template <class Exec> struct StreamIO {
    Exec& x; StreamBuffers& sb; FrameDState* d;
    const u8* se; u64 room;
    const u8* r_at = nullptr;                               // the current round: where its walk started
    std::vector<StreamWalkRec> recs; std::vector<int> res; StreamWalk walk = {0, 0, 0, 0, 0};
    u8* stage = nullptr; size_t slot = 0;
    std::vector<StreamSeg> place_segs, hash_segs;
    bool check = false; u32 expect = 0;
    int check_stage = 0; size_t check_fill = 0;             // the state the host call keeps when the checksum fails
    StreamIO(Exec& x_, StreamBuffers& sb_, FrameDState* d_, const u8* se_, u64 room_) : x(x_), sb(sb_), d(d_), se(se_), room(room_) {}

    void flush()
    {
        if (!place_segs.empty()) { x.gather(place_segs); place_segs.clear(); }
        if (!hash_segs.empty()) { x.hash(hash_segs, sb.hash); hash_segs.clear(); }
    }
    void run_round(const u8* p, u32 carry_len)
    {
        flush();
        u32 max_recs, slots;
        stream_round_shape((u64)(se - p), room, d->max_block, &max_recs, &slots);
        recs.assign(max_recs, StreamWalkRec{0, 0, -1});
        res.assign((size_t)slots + 1, -1);
        x.round(p, (u64)(se - p), (u32)d->max_block, sb.carry, carry_len, max_recs, slots, &walk, recs.data(), res.data(), &stage);
        r_at = p; slot = d->max_block;
    }
    // the record of the size word at p, walking from p if the current round has none
    const StreamWalkRec* find(const u8* p)
    {
        if (r_at && p >= r_at) {
            const u64 at = (u64)(p - r_at);
            const StreamWalkRec* e = recs.data() + walk.n_recs;
            const StreamWalkRec* r = std::lower_bound((const StreamWalkRec*)recs.data(), e, at, [](const StreamWalkRec& a, u64 v) { return a.pos < v; });
            if (r != e && r->pos == at) return r;
        }
        return nullptr;
    }
    const StreamWalkRec& rec(const u8* p)
    {
        const StreamWalkRec* r = find(p);
        if (!r) { run_round(p, 0); r = find(p); }
        return *r;                                          // the walk records the word at its start: 4 bytes are there
    }
    // the decode result of the compressed block whose payload is at p, and where its bytes are
    int result(const u8* p, const u8** at)
    {
        const StreamWalkRec* r = find(p - kBH);
        if (!r || r->unit < 0) { run_round(p - kBH, 0); r = find(p - kBH); }
        *at = stage + (size_t)r->unit * slot;
        return res[(size_t)r->unit];
    }

    const u8* view(const u8* p, size_t n, u8* buf) { x.read(buf, p, n); return buf; }
    void load(u8* to, const u8* p, size_t n)
    {   // the bytes behind the current round's end mark came back with its records
        if (r_at && walk.stop == kWalkEnd && walk.n_recs) {
            const u8* t = r_at + recs[walk.n_recs - 1].pos + kBH;
            if (p >= t && p + n <= t + walk.tail_n) {
                for (size_t i = 0; i < n; ++i) to[i] = (u8)(walk.tail >> (8 * (p - t + i)));
                return;
            }
        }
        if (n) x.read(to, p, n);
    }
    u32 word(const u8* p) { return rec(p).word; }
    bool ready() { return true; }
    void hash_reset() { x.hash_reset(sb.hash); }
    void frame_buffers(size_t mb) { x.buffers(sb, mb); }
    void copy(u8* to, const u8* p, size_t n) { if (n) place_segs.push_back({ (u64)(size_t)p, (u64)(size_t)to, n }); }
    void hash(const u8* q, size_t n) { if (n) hash_segs.push_back({ (u64)(size_t)q, 0, n }); }
    int decode_batch(const u8* span_begin, size_t, const std::vector<FrameBlockRef>& blocks, u8* dp, size_t, std::vector<int>& sz, bool)
    {   // placed here, block by block, so that a round started for a later block of the batch finds the earlier ones placed
        sz.assign(blocks.size(), -1);
        u8* w = dp;
        for (size_t i = 0; i < blocks.size(); ++i) {
            const u8* at;
            const int r = result(span_begin + blocks[i].src_pos, &at);
            sz[i] = r;
            if (r < 0) break;
            if (r > 0) place_segs.push_back({ (u64)(size_t)at, (u64)(size_t)w, (u64)r });
            w += r;
        }
        return 0;
    }
    void place(u8*, u8*, size_t, size_t) {}
    int decode_tmp(const u8* p, size_t)
    {
        const u8* at;
        const int r = result(p, &at);
        if (r >= 0) sb.tmp_at = at;
        return r;
    }
    void hash_tmp(size_t n) { if (n) hash_segs.push_back({ (u64)(size_t)sb.tmp_at, 0, n }); }
    void carry(size_t at, const u8* p, size_t n) { if (n) x.copy(sb.carry + at, p, n); }
    int decode_carry(const u8* p, u8* to, size_t n)
    {
        run_round(p, (u32)n);
        const int r = res[0];
        if (r < 0) return r;
        if (to) { if (r > 0) place_segs.push_back({ (u64)(size_t)stage, (u64)(size_t)to, (u64)r }); }
        else sb.tmp_at = stage;
        return r;
    }
    void flush_out(u8* to, size_t at, size_t n) { if (n) place_segs.push_back({ (u64)(size_t)(sb.tmp_at + at), (u64)(size_t)to, n }); }
    bool digest_ok(u32 w)
    {   // decided in finish(), when the checksum is known
        check = true; expect = w; check_stage = d->stage; check_fill = d->tmp_in_size;
        return true;
    }

    // after the run: the collected work, the one-block buffer's bytes still to come out of the staging arena, then the
    // stream is synchronised.  Returns false when the content checksum the run deferred does not match.
    bool finish()
    {
        flush();
        if (d->stage == DS_flushOut && sb.tmp_at != sb.tmp_out) { x.copy(sb.tmp_out, sb.tmp_at, d->tmp_out_size); sb.tmp_at = sb.tmp_out; }
        if (check) return x.digest(sb.hash) == expect;
        x.sync();
        return true;
    }
};

// One LizardB200_decompressStream call over an executor: the run, then finish().  A content checksum that does not match
// returns ERROR_contentChecksum_invalid with nothing consumed or produced and the context as the host call leaves it when it
// returns that error from the suffix stage: the stage and the suffix bytes kept, the expected source pointer unchanged.
template <class Exec>
size_t frame_stream_call(Exec& x, StreamBuffers& sb, FrameDState* d, u8* dDst, size_t* dstSizePtr, const u8* dSrc, size_t* srcSizePtr)
{
    StreamIO<Exec> io(x, sb, d, dSrc + *srcSizePtr, *dstSizePtr);
    const u8* const expect_before = d->src_expect;
    const size_t r = frame_decompress_run(d, io, dSrc, srcSizePtr, dDst, dstSizePtr);
    if (!io.finish()) {
        d->stage = io.check_stage; d->tmp_in_size = io.check_fill; d->src_expect = expect_before;
        *srcSizePtr = 0; *dstSizePtr = 0;
        return ferr(FE_contentChecksum_invalid);
    }
    return r;
}

}  // namespace lzb
