// frame_cstream.h -- LizardF_compressBegin / Update / flush / End's decisions, stated once over a backend (DESIGN.md 3.4e).
//
// frame.inl runs these functions with host memory (the LizardF_* calls: blocks compressed by the pipelined batch path) and with
// device memory (LizardB200_compressStream*: the backend enqueues copies and kernels, frame_cstream_kernels.cuh).  The host shim
// builds them with host memory and the one-lane encoder, so the CPU tests compare them call for call with the reference's frame
// layer.  Every decision depends only on host values: the stage, the capacity, the carried length, the chunk's length, the
// preferences and the running total.  Only the sizes of the records depend on the data.
//
// Reference: lib/lizard_frame.c:363-429 (begin), :501-590 (update, independent blocks), :601-629 (flush), :641-670 (end).
#pragma once
#include "frame_stream.h"

namespace lzb {

// Lizard_verifyCompressionLevel
LZ_HD int frame_level(int lvl) { return lvl > (int)kMaxLevel ? (int)kMaxLevel : lvl < (int)kMinLevel ? (int)kDefaultLevel : lvl; }
// the preference fields the frame header and the bounds depend on (frame_device.cuh: frame_begin and the bounds)
inline FramePrefs frame_prefs(const LizardF_preferences_t& p)
{
    return FramePrefs{ (u32)p.frameInfo.blockSizeID, (u32)p.frameInfo.blockMode, (u32)p.frameInfo.contentChecksumFlag,
                       p.autoFlush, p.frameInfo.contentSize };
}

// What a compression context keeps between calls besides its buffers (the carried bytes and the content checksum, which the
// backend owns)
struct FrameCState {
    LizardF_preferences_t prefs;
    unsigned stage;                         // 0: idle, 1: header written
    size_t block_size;
    size_t carry;                           // bytes of a partial block waiting for more input (lizard_frame.c tmpIn)
    u64 total_in;
    void reset() { memset(&prefs, 0, sizeof prefs); stage = 0; block_size = 0; carry = 0; total_in = 0; }
};

// How an Update takes a chunk of n bytes, with `carry` bytes carried and blocks of bs bytes: `take` bytes go to the carried block
// first (carry_block: they complete it, and it is compressed), then `whole` bytes are compressed as blocks (autoFlush: all that is
// left, the last block shorter), then the `rest` is carried.
struct CUpdatePlan { u64 take, whole, rest; u32 carry_block; };
LZ_HD CUpdatePlan frame_cupdate_plan(u64 carry, u64 bs, u32 auto_flush, u64 n)
{
    CUpdatePlan p = { 0, 0, 0, 0 };
    if (carry) {
        const u64 need = bs - carry;
        if (need > n) p.take = n;
        else { p.take = need; p.carry_block = 1; }
    }
    const u64 left = n - p.take;
    p.whole = auto_flush ? left : left / bs * bs;
    p.rest = left - p.whole;
    return p;
}

// Unit k of a compression round: the carried block (carry_len > 0: unit 0, carry_len bytes at `carry`), then the blocks of bs
// bytes of the n bytes at p, the last one shorter.  Sources are addresses; each unit's encoder slot is `stride` bytes and its
// capacity len - 1 (lizard_frame.c:459: a block that does not shrink is stored raw).
LZ_HD void cstream_unit(u32 k, u64 carry, u64 carry_len, u64 p, u64 n, u64 bs, u64 stride, u64* src, u32* len, u64* enc, u32* cap)
{
    const u32 carry_on = carry_len != 0;
    u64 s, l;
    if (carry_on && k == 0) { s = carry; l = carry_len; }
    else {
        const u64 at = (u64)(k - carry_on) * bs;
        s = p + at; l = n - at < bs ? n - at : bs;
    }
    *src = s; *len = (u32)l; *enc = (u64)k * stride; *cap = (u32)l - 1;
}

// The backend (IO) a run goes through.  dst/p are the caller's pointers; sizes it returns may be placeholders (the device's are
// only known on the device), errors never are.
//   bool ready()                               the device can take work (else ERROR_GENERIC)
//   bool level_ok(level)                       the encoder implements the level
//   void begin(dst, hdr, n, bs)                the header's n bytes to dst; the checksum starts over, the carried block holds bs
//   void hash_begin(p, n) / hash_end(p, n)     the checksum takes the chunk (hash_end: after the blocks; hash_abort on an error)
//   void carry(at, p, n)                       n bytes at p to the carried block at offset `at`
//   size_t compress_carry(dst, cap, n, level)  the carried block of n bytes as one record: its size or an error
//   size_t compress(dst, cap, p, n, level)     the n bytes at p as records of blocks of the block size
//   void end_mark(dst, ccksum)                 the end mark and, with ccksum, the checksum
template <class IO> size_t frame_cbegin_run(FrameCState* c, IO& io, u8* dst, size_t dstMax, const LizardF_preferences_t* prefsPtr)
{   // lib/lizard_frame.c:363-429
    if (dstMax < kMaxFH) return ferr(FE_dstMaxSize_tooSmall);
    if (c->stage != 0) return ferr(FE_GENERIC);
    if (prefsPtr) c->prefs = *prefsPtr; else memset(&c->prefs, 0, sizeof c->prefs);
    if (c->prefs.frameInfo.blockSizeID == 0) c->prefs.frameInfo.blockSizeID = LizardF_max128KB;
    // the checks and the header: frame_device.cuh (the level after Lizard_verifyCompressionLevel, then the GPU level gate)
    u8 hdr[16];
    u32 len;
    u64 bs;
    const u32 v = frame_begin(frame_prefs(c->prefs), io.level_ok(frame_level(c->prefs.compressionLevel)), hdr, &len, &bs);
    c->block_size = (size_t)bs;
    if (v != kFwOk) return ferr((int)v);
    io.begin(dst, hdr, len, c->block_size);
    c->carry = 0; c->total_in = 0;
    c->stage = 1;
    return len;
}

template <class IO> size_t frame_cflush_run(FrameCState* c, IO& io, u8* dst, size_t dstMax)
{   // lib/lizard_frame.c:601-629
    if (c->carry == 0) return 0;
    if (c->stage != 1) return ferr(FE_GENERIC);
    if (dstMax < c->carry + 8) return ferr(FE_dstMaxSize_tooSmall);
    if (c->carry == 1 && dstMax < 4 + 6) return ferr(FE_dstMaxSize_tooSmall);    // a 1-byte block's record (frame_one_byte_record)
    if (!io.ready()) return ferr(FE_GENERIC);
    const size_t r = io.compress_carry(dst, dstMax, c->carry, frame_level(c->prefs.compressionLevel));
    if (!fe_is_error(r)) c->carry = 0;
    return r;
}

template <class IO> size_t frame_cupdate_run(FrameCState* c, IO& io, u8* dst, size_t dstMax, const u8* src, size_t srcSize)
{   // lib/lizard_frame.c:501-590 (independent blocks)
    if (c->stage != 1) return ferr(FE_GENERIC);
    if (dstMax < frame_compress_bound(srcSize, frame_prefs(c->prefs))) return ferr(FE_dstMaxSize_tooSmall);
    const CUpdatePlan pl = frame_cupdate_plan(c->carry, c->block_size, c->prefs.autoFlush, srcSize);
    // an input of one byte alone in its block: its record (10 bytes) outgrows any capacity below 10
    if (!c->carry && pl.whole == 1 && dstMax < 4 + 6) return ferr(FE_dstMaxSize_tooSmall);
    if (!io.ready()) return ferr(FE_GENERIC);
    const int level = frame_level(c->prefs.compressionLevel);
    // Content checksum (lib/lizard_frame.c:585-586): XXH32 over everything fed in, in order
    const bool want_hash = c->prefs.frameInfo.contentChecksumFlag == LizardF_contentChecksumEnabled;
    if (want_hash) io.hash_begin(src, srcSize);
    size_t d = 0;
    if (pl.take) io.carry(c->carry, src, pl.take);
    if (pl.carry_block) {                                   // complete the pending partial block first
        const size_t r = io.compress_carry(dst, dstMax, c->block_size, level);
        if (fe_is_error(r)) { c->carry = c->block_size; if (want_hash) io.hash_abort(); return r; }
        c->carry = 0;
        d += r;
    } else c->carry += pl.take;
    if (pl.whole) {
        const size_t r = io.compress(dst + d, dstMax - d, src + pl.take, pl.whole, level);
        if (fe_is_error(r)) { if (want_hash) io.hash_abort(); return r; }
        d += r;
    }
    if (pl.rest) { io.carry(0, src + pl.take + pl.whole, pl.rest); c->carry = pl.rest; }
    if (want_hash) io.hash_end(src, srcSize);
    c->total_in += srcSize;
    return d;
}

template <class IO> size_t frame_cend_run(FrameCState* c, IO& io, u8* dst, size_t dstMax)
{   // lib/lizard_frame.c:641-670
    const size_t r = frame_cflush_run(c, io, dst, dstMax);
    if (fe_is_error(r)) return r;
    const bool ccksum = c->prefs.frameInfo.contentChecksumFlag == LizardF_contentChecksumEnabled;
    io.end_mark(dst + r, ccksum);
    c->stage = 0;
    if (c->prefs.frameInfo.contentSize && c->prefs.frameInfo.contentSize != c->total_in) return ferr(FE_frameSize_wrong);
    return r + 4 + (ccksum ? 4 : 0);
}

}  // namespace lzb
