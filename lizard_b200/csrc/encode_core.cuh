// encode_core.cuh -- the Lizard block encoder written once for "a warp": every lane runs the same
// control flow on the same (uniform) cursor state; byte movement, histograms and bit-packing are split
// across lanes through the policy type W.  With W = HostLanes (one lane) the very same code builds with
// g++, which is how the CPU test-suite pins it byte-for-byte against the reference (-DLIZARD_RESET_MEM).
//
// Reference functions restated here:
//   lib/lizard_compress.c:75-109         Lizard_hash5 / Lizard_hashPtr
//   lib/lizard_common.h:475-490          Lizard_count
//   lib/lizard_parser_fastsmall.h:34-189 Lizard_compress_fastSmall   (levels 10, 30)
//   lib/lizard_parser_fast.h:41-196      Lizard_compress_fast        (levels 11, 31; same loop, hashLog 18)
//   lib/lizard_parser_pricefast.h:3-249  Lizard_FindMatchFast / _Faster / Lizard_compress_priceFast (21,22,41,42)
//   lib/lizard_compress_lz4.h:3-86       Lizard_encodeSequence_LZ4 / LastLiterals
//   lib/lizard_compress_liz.h:43-179     Lizard_encodeSequence_LIZv1 / LastLiterals
//   lib/lizard_compress.c:141-250        Lizard_writeStream / Lizard_writeBlock
//   lib/lizard_compress.c:472-547        Lizard_compress_generic
#pragma once
#include "common.cuh"
#include "entropy_enc.cuh"
#include "lanes.cuh"
#if !defined(__CUDACC__)
#include <string.h>
#include <stdlib.h>
#endif

namespace lzb {

// ---- unaligned little-endian loads from the source block ----------------------------------------
LZ_HD u32 ld32(const u8* p)
{
#if defined(__CUDA_ARCH__)
    const size_t a = (size_t)p;
    const u32* q = (const u32*)(a & ~(size_t)3);
    return __funnelshift_r(q[0], q[1], (u32)(a & 3) * 8);      // two aligned words, shift 0 returns the first
#else
    u32 v; memcpy(&v, p, 4); return v;
#endif
}
LZ_HD u64 ld64(const u8* p)
{
#if defined(__CUDA_ARCH__)
    const size_t a = (size_t)p;
    const u32* q = (const u32*)(a & ~(size_t)3);
    const u32 sh = (u32)(a & 3) * 8;
    const u32 w0 = q[0], w1 = q[1], w2 = q[2];
    return (u64)__funnelshift_r(w0, w1, sh) | ((u64)__funnelshift_r(w1, w2, sh) << 32);
#else
    u64 v; memcpy(&v, p, 8); return v;
#endif
}
// the 5 bytes at p as a 40-bit little-endian value: all the hash needs, and its low word is the 4-byte match test
LZ_HD u64 ld5(const u8* p)
{
#if defined(__CUDA_ARCH__)
    const size_t a = (size_t)p;
    const u32* q = (const u32*)(a & ~(size_t)3);
    const u32 sh = (u32)(a & 3) * 8;
    const u32 w0 = q[0], w1 = q[1];
    return (u64)__funnelshift_r(w0, w1, sh) | ((u64)((w1 >> sh) & 0xFFu) << 32);
#else
    u64 v; memcpy(&v, p, 8); return v & 0xFFFFFFFFFFull;
#endif
}

LZ_HD u32 hash5(u64 v, u32 hbits) { return (u32)(((v * 889523592379ULL) << 24) >> (64 - hbits)); }

// common prefix length of a[..] and b[..], a bounded by `limit` (Lizard_count)
LZ_HD u32 count_match(const u8* a, const u8* b, const u8* limit)
{
    const u8* const a0 = a;
    while (a + 7 < limit) {
        u64 d = ld64(a) ^ ld64(b);
        if (d) {
#if defined(__CUDA_ARCH__)
            return (u32)(a - a0) + ((u32)(__ffsll((long long)d) - 1) >> 3);
#else
            return (u32)(a - a0) + ((u32)__builtin_ctzll(d) >> 3);
#endif
        }
        a += 8; b += 8;
    }
    while (a < limit && *a == *b) { a++; b++; }
    return (u32)(a - a0);
}

// ---- sequence list of one inner block ---------------------------------------------------------------------
// The parsers do not write the token streams while they run: they append one record per sequence and keep
// exact byte counts of the four streams (the codeword rules below are pure functions of lit/ml/off).  When
// the block is parsed, write_block() knows every size, takes the reference's raw / does-not-fit decisions
// without moving a byte, and emit_streams() materialises all sequences lane-parallel, straight into their
// final place in dst whenever no entropy stage follows.  This keeps the literal copies (the biggest stall
// source in the first version) off the serial search->extend->record chain.
struct SeqRec { u32 anchor, lit, ml, off; };       // off == 0: repeat last offset (LIZv1 only)

struct EncStreams {
    SeqRec* rec;  u32 nseq;
    u32 nl, nf, n16, n24;                          // exact sizes of literals / flags / off16 / off24 streams
    u32 tail_anchor, tail_len;                     // last literals
};

// length extension: b<254 | 254,LE16 | 255,LE24
LZ_HD u32 ext_bytes(u32 v) { return v >= (1u << 16) ? 4u : (v >= 254 ? 3u : 1u); }
LZ_HD void put_ext_at(u8* p, u32 v)
{
    if (v >= (1u << 16)) { p[0] = 255; wr_le24(p + 1, v); }
    else if (v >= 254)   { p[0] = 254; wr_le16(p + 1, v); }
    else                 p[0] = (u8)v;
}

// Lizard_encodeSequence_LZ4 (lib/lizard_compress_lz4.h:3-71): literals src[anchor..ip) + match(ml, off)
template <class W> LZ_HD void emit_lz4(EncStreams& s, const u8*, u32 anchor, u32 ip, u32 ml, u32 off)
{
    const u32 lit = ip - anchor, m = ml - kMinMatch;
    s.nl += (lit >= 15 ? ext_bytes(lit - 15) : 0) + lit + 2 + (m >= 15 ? ext_bytes(m - 15) : 0);
    s.nf += 1;
    if (W::lane() == 0) { SeqRec r; r.anchor = anchor; r.lit = lit; r.ml = ml; r.off = off; s.rec[s.nseq] = r; }
    s.nseq++;
}

// Lizard_encodeSequence_LIZv1 (lib/lizard_compress_liz.h:43-165).  off == 0 means "repeat last offset".
template <class W> LZ_HD void emit_lizv1(EncStreams& s, const u8*, u32 anchor, u32 ip, u32 ml, u32 off, u32& last_off)
{
    const u32 lit = ip - anchor;
    const bool far = off >= kMax16BitOffset;
    if (lit > 0 || !far) {
        s.nl += (lit >= 7 ? ext_bytes(lit - 7) : 0) + lit;
        if (far) s.nf += 1;                                   // carrier token for the literals
    }
    if (far) {
        if (ml - kMmLongOff >= kLastLongOff) s.nl += ext_bytes(ml - kMmLongOff - kLastLongOff);
        s.n24 += 3;
        last_off = off;
    } else {
        if (off != 0) { last_off = off; s.n16 += 2; }
        if (ml >= 15) s.nl += ext_bytes(ml - 15);
    }
    s.nf += 1;
    if (W::lane() == 0) { SeqRec r; r.anchor = anchor; r.lit = lit; r.ml = ml; r.off = off; s.rec[s.nseq] = r; }
    s.nseq++;
}

template <class W> LZ_HD void emit_last_literals(EncStreams& s, const u8*, u32 anchor, u32 end)
{
    s.tail_anchor = anchor; s.tail_len = end - anchor;
    s.nl += end - anchor;
}

// Materialise the recorded sequences: lane i of each batch owns sequence base+i, prefix sums give its place
// in every stream, it writes its own token / extension / offset bytes, and the warp copies the batch's
// literal runs (two runs in flight).  Byte layout per sequence: see the two emitters cited above.
template <class W> LZ_HD void emit_streams(const EncStreams& s, const u8* src, bool lizv1, u8* dl, u8* df, u8* d16, u8* d24)
{
    const u32 NL = W::lanes(), lane = W::lane();
    u32 pl = 0, pf = 0, p16 = 0, p24 = 0;
    W::sync();                                                  // records were written by lane 0
    for (u32 base = 0; base < s.nseq; base += NL) {
        const u32 nb = s.nseq - base < NL ? s.nseq - base : NL;
        const bool act = lane < nb;
        SeqRec r; r.anchor = 0; r.lit = 0; r.ml = 0; r.off = 0;
        if (act) r = s.rec[base + lane];
        u32 e1 = 0, e2 = 0, lbytes = 0, fbytes = 0, b16 = 0, b24 = 0, t0 = 0, t1 = 0;
        bool first = false, far = false;
        if (act) {
            if (!lizv1) {
                const u32 m = r.ml - kMinMatch;
                e1 = r.lit >= 15 ? ext_bytes(r.lit - 15) : 0;
                e2 = m >= 15 ? ext_bytes(m - 15) : 0;
                lbytes = e1 + r.lit + 2 + e2; fbytes = 1;
                t0 = (r.lit >= 15 ? 15u : r.lit) | ((m >= 15 ? 15u : m) << 4);
            } else {
                far = r.off >= kMax16BitOffset;
                first = r.lit > 0 || !far;
                if (first) { e1 = r.lit >= 7 ? ext_bytes(r.lit - 7) : 0; t0 = r.lit >= 7 ? 7u : r.lit; }
                if (far) {
                    const u32 m = r.ml - kMmLongOff;
                    e2 = m >= kLastLongOff ? ext_bytes(m - kLastLongOff) : 0;
                    t1 = m >= kLastLongOff ? (u32)kLastLongOff : m;
                    b24 = 3; fbytes = first ? 2 : 1;
                    if (first) t0 += 1u << 7;
                } else {
                    e2 = r.ml >= 15 ? ext_bytes(r.ml - 15) : 0;
                    t0 += (r.off == 0 ? (1u << 7) : 0u) + ((r.ml >= 15 ? 15u : r.ml) << 3);
                    b16 = r.off != 0 ? 2 : 0; fbytes = 1;
                }
                lbytes = (first ? e1 + r.lit : 0) + e2;
            }
        }
        u32 tl = 0, tf = 0, t16 = 0, t24 = 0;
        const u32 Pl = pl + W::excl_scan(lbytes, &tl);
        const u32 Pf = pf + W::excl_scan(fbytes, &tf);
        const u32 P16 = p16 + W::excl_scan(b16, &t16);
        const u32 P24 = p24 + W::excl_scan(b24, &t24);
        const u32 lit_dst = Pl + e1;
        if (act) {
            if (!lizv1) {
                df[Pf] = (u8)t0;
                if (e1) put_ext_at(dl + Pl, r.lit - 15);
                wr_le16(dl + lit_dst + r.lit, r.off);
                if (e2) put_ext_at(dl + lit_dst + r.lit + 2, r.ml - kMinMatch - 15);
            } else {
                if (first && e1) put_ext_at(dl + Pl, r.lit - 7);
                const u32 ext_at = first ? lit_dst + r.lit : Pl;
                if (far) {
                    if (first) { df[Pf] = (u8)t0; df[Pf + 1] = (u8)t1; } else df[Pf] = (u8)t1;
                    if (e2) put_ext_at(dl + ext_at, r.ml - kMmLongOff - kLastLongOff);
                    wr_le24(d24 + P24, r.off);
                } else {
                    df[Pf] = (u8)t0;
                    if (e2) put_ext_at(dl + ext_at, r.ml - 15);
                    if (b16) wr_le16(d16 + P16, r.off);
                }
            }
        }
        // literal runs of the batch
        const u32 cp_len = (act && (!lizv1 || first)) ? r.lit : 0;
        {   // short runs go several at a time (one lane group each), long ones take the whole warp
            typedef LaneGroups<W> LG;
            const bool is_long = cp_len > LG::kMaxBytes;
            const u32 shorts = W::ballot(cp_len != 0 && !is_long);
            u32 longs = W::ballot(is_long);
            const u32 sub = lane / LG::kGroup;
            const u32 short_len = is_long ? 0u : cp_len;
            for (u32 k0 = 0; k0 < nb; k0 += LG::kRuns) {
                if (((shorts >> k0) & ((1u << LG::kRuns) - 1)) == 0) continue;
                const u32 k = k0 + sub;
                const u32 len0 = W::shfl(short_len, k), a0 = W::shfl(r.anchor, k), d0 = W::shfl(lit_dst, k);
                lanes_copy_groups<W, true>(dl + d0, src + a0, len0);
            }
            for (; longs; longs &= longs - 1) {
                const u32 k = ctz32(longs);
                const u32 len0 = W::shfl(cp_len, k), a0 = W::shfl(r.anchor, k), d0 = W::shfl(lit_dst, k);
                if (len0 >= kWideMinBytes) lanes_copy_wide<W, true>(dl + d0, src + a0, len0, false);
                else lanes_copy_rows<W, true>(dl + d0, src + a0, len0);
            }
        }
        pl += tl; pf += tf; p16 += t16; p24 += t24;
    }
    lanes_copy_wide<W, true>(dl + pl, src + s.tail_anchor, s.tail_len, false);
    W::sync();
}

// ---- hash table ------------------------------------------------------------------------------------------------
// The reference keeps 32-bit absolute indices (position + 2^24, 0 = never written).  For units of at most one
// inner block (<= 128 KiB, i.e. every independent frame block) a position needs 17 bits, so the shared-memory
// form packs an entry as position+1 (0 = empty) in 16 low bits + 1 bit in a bitmap: 8.5 KiB instead of 16 KiB at
// level 10, 34 KiB instead of 64 KiB at levels 21/41 -- the table size is what bounds resident warps per SM.
// The parsers insert positions in increasing order, so the bitmap is untouched (all zero) until the parse crosses
// position 65535 and from then on bits are only ever set; `pos_hint` (a position not below anything inserted so
// far) lets the first half of a block skip the bitmap altogether.
// Larger units (several dependent inner blocks) use plain 32-bit entries in global memory.
// Candidate tags (fastSmall / fast parsers).  On datagen -P50 a 128 KiB block makes ~60 000 probes and finds ~1000
// matches: once the table has filled, nearly every probe finds an in-range candidate, reads its four bytes -- a 32-byte
// sector somewhere in the last 64 KiB of one of 4000 blocks in flight, i.e. mostly DRAM -- and throws it away.  An entry
// therefore also carries a few hash bits of the four bytes at its position (tag8; independent of the bucket hash), and a
// probe only reads the candidate when the tags agree.  A differing tag proves the bytes differ, so the parse is unchanged.
// Only the fast parsers keep tags up to date (set_t) and consult them (get_t / maybe); the others use get / set and never
// look at them.
LZ_HD u32 tag8(u32 v4) { return (v4 * 0x9E3779B1u) >> 24; }
enum : u32 { kNoTag = 0x100u };

struct HashTable {       // runtime descriptor handed to encode_unit
    u32* t32;            // plain form (global memory), or null
    u16* lo;             // packed form
    u32* hi;
    u8*  tag;            // packed form: one tag byte per entry, or null
    u32  tagged;         // plain form: every position of the unit is below 2^17, bits 25..31 of an entry hold a tag
};
struct PlainTable {
    static constexpr bool kOneBlock = false;    // any unit
    static constexpr bool kDict = false;        // positions start at the unit (DictTable: at a loaded dictionary)
    u32* t32; u32 tagged;
    LZ_HDM explicit PlainTable(const HashTable& d) : t32(d.t32), tagged(d.tagged) {}
    LZ_HDM u32 get(u32 h, u32) const { const u32 e = t32[h]; return tagged ? e & 0x1FFFFFFu : e; }
    LZ_HDM void set(u32 h, u32 abs_index) const { t32[h] = abs_index; }
    LZ_HDM u32 get_t(u32 h, u32, u32* tag) const
    {
        const u32 e = t32[h];
        if (!tagged) { *tag = kNoTag; return e; }
        *tag = e >> 25;
        return e & 0x1FFFFFFu;
    }
    LZ_HDM void set_t(u32 h, u32 abs_index, u32 tag) const { t32[h] = tagged ? abs_index | (tag >> 1) << 25 : abs_index; }
    LZ_HDM bool maybe(u32 stored, u32 mine) const { return stored == kNoTag || stored == (mine >> 1); }
    template <class W> LZ_HDM void clear(u32 hash_log) const
    {
        const u32 n = 1u << hash_log;
        for (u32 i = W::lane(); i < n; i += W::lanes()) t32[i] = 0;
        W::sync();
    }
};
struct PackedTable {
    static constexpr bool kOneBlock = true;     // units of one inner block only (positions below 2^17)
    static constexpr bool kDict = false;
    u16* lo; u32* hi; u8* tag;
    LZ_HDM explicit PackedTable(const HashTable& d) : lo(d.lo), hi(d.hi), tag(d.tag) {}
    LZ_HDM u32 get(u32 h, u32 pos_hint) const
    {
        u32 p = lo[h];
        if (pos_hint >= 0xFFFFu) p |= ((hi[h >> 5] >> (h & 31)) & 1u) << 16;
        return p ? p - 1 + kDictSize : 0u;
    }
    LZ_HDM void set(u32 h, u32 abs_index) const
    {
        const u32 p = abs_index - kDictSize + 1;
        lo[h] = (u16)p;
        const u32 bit = 1u << (h & 31);
#if defined(__CUDA_ARCH__)
        if (p >> 16) { if (!(hi[h >> 5] & bit)) atomicOr(&hi[h >> 5], bit); }
#else
        if (p >> 16) hi[h >> 5] |= bit;
        else if (hi[h >> 5] & bit) abort();        // insertion order assumption violated
#endif
    }
    LZ_HDM u32 get_t(u32 h, u32 pos_hint, u32* t) const { *t = tag ? (u32)tag[h] : (u32)kNoTag; return get(h, pos_hint); }
    LZ_HDM void set_t(u32 h, u32 abs_index, u32 t) const { set(h, abs_index); if (tag) tag[h] = (u8)t; }
    LZ_HDM bool maybe(u32 stored, u32 mine) const { return stored == kNoTag || stored == mine; }
    template <class W> LZ_HDM void clear(u32 hash_log) const
    {
        const u32 n = 1u << hash_log;
        u32* lo32 = reinterpret_cast<u32*>(lo);
        for (u32 i = W::lane(); i < n / 2; i += W::lanes()) lo32[i] = 0;
        for (u32 i = W::lane(); i < n / 32; i += W::lanes()) hi[i] = 0;
        W::sync();                                  // tags of empty entries are never looked at
    }
};
// hashChain and priceFast against a loaded dictionary (Lizard_loadDict + Lizard_compress_continue, lib/lizard_compress.c:426-450,
// 550-580).
// Positions count from the dictionary's first byte: the dictionary is [0, dend), the unit starts at dend, and an entry is
// position + kDictSize, the reference's own index.  The table after Lizard_loadDict is built once per dictionary and shared
// read-only by every unit that uses it (`sh`, with the chain entries of the positions it inserted in `dchain`); a unit writes
// only its own overlay `ov`, where 0 means "not written by this unit": every write a unit makes stores one of its own
// positions (>= own0), so an empty overlay entry is exactly a bucket the unit has not changed.  The overlay is cleared per
// unit as the plain table is.  ext: the dictionary is external (Lizard_setExternalDict ran) and its bytes are at dsrc;
// otherwise it lies directly in front of the unit and dsrc is the parse's own base.
struct DictTable {
    static constexpr bool kOneBlock = false;
    static constexpr bool kDict = true;
    u32* ov; const u32* sh; const u16* dchain; const u8* dsrc;
    u32 dend;            // dictionary size (= the unit's first position)
    u32 own0;            // hashChain's nextToUpdate: dend, or dend - 7 for a prefix dictionary (priceFast writes positions >= dend)
    u32 low;             // ctx->lowLimit as an index
    u32 ext;
    LZ_HDM u32 get(u32 h, u32) const { const u32 e = ov[h]; return e ? e : sh[h]; }
    LZ_HDM void set(u32 h, u32 abs_index) const { if (abs_index >= own0 + kDictSize) ov[h] = abs_index; }
    LZ_HDM u32 get_t(u32 h, u32 pos_hint, u32* t) const { *t = kNoTag; return get(h, pos_hint); }      // priceFast: no tags
    LZ_HDM void set_t(u32 h, u32 abs_index, u32) const { set(h, abs_index); }
    LZ_HDM bool maybe(u32, u32) const { return true; }
    template <class W> LZ_HDM void clear(u32 hash_log) const
    {
        const u32 n = 1u << hash_log;
        for (u32 i = W::lane(); i < n; i += W::lanes()) ov[i] = 0;
        W::sync();
    }
};

// Which tables carry tags: the plain table has the bits to spare (fast parsers and priceFast use them; single-block units
// only); a packed table pays a byte per entry, which the small level-10/30 tables of the fast parsers are given and the
// 34 KiB priceFast tables are not.
#if !defined(LZB_ENC_TAGS)
#define LZB_ENC_TAGS 1
#endif
LZ_HD bool enc_tagged(const LevelParams& lp) { return LZB_ENC_TAGS && (lp.parser == kParserFastSmall || lp.parser == kParserFast); }
LZ_HD bool enc_tagged_plain(const LevelParams& lp) { return LZB_ENC_TAGS && (enc_tagged(lp) || lp.parser == kParserPriceFast || lp.parser == kParserFastBig); }

// bytes of a packed table: 16-bit entries + the bit plane (+ one tag byte per entry for the fast parsers)
LZ_HD size_t hash_packed_bytes(u32 hash_log, bool tagged)
{
    return ((size_t)2 << hash_log) + ((size_t)1 << hash_log) / 8 + (tagged ? (size_t)1 << hash_log : 0);
}

// ---- parser state shared by the inner blocks of one unit -----------------------------------------------
template <class TT> struct ParseCtx {
    const u8* src;        // unit start (position 0); table entries are position + kDictSize, 0 = empty
    TT        T;
    u32       hash_log;
    u32       window_log;
};

// ---- lane-parallel building blocks ---------------------------------------------------------------------
// Position of the j-th probe of one fastSmall search relative to its first probe: the stride grows by one
// every 64 probes (step = searchMatchNb++ >> 6, lizard_parser_fastsmall.h:69-75), so the offsets are
// 0,1,2,...,65,67,69,... independent of the data.
LZ_HD u32 probe_offset(u32 j)
{
    if (j <= 65) return j;                       // the common case: the first two batches of a search
    const u32 m = 62 + j;
    if (m < 64) return 1;
    const u32 q = m >> 6;
    return 1 + 32 * q * (q - 1) + q * (m - 64 * q + 1);
}

// Lizard_count with the lanes comparing consecutive 8-byte groups
template <class W> LZ_HD u32 count_match_par(const u8* a, const u8* b, const u8* limit)
{
    u32 total = 0;
    for (;;) {
        const u32 off = total + 8 * W::lane();
        const u8* pa = a + off;
        u32 n = 0; bool full = false;
        if (pa + 8 <= limit) {
            const u64 d = ld64(pa) ^ ld64(b + off);
            if (d == 0) { n = 8; full = true; }
            else {
#if defined(__CUDA_ARCH__)
                n = (u32)(__ffsll((long long)d) - 1) >> 3;
#else
                n = (u32)__builtin_ctzll(d) >> 3;
#endif
            }
        } else {
            while (pa + n < limit && pa[n] == b[off + n]) n++;
        }
        const u32 stop = W::ballot(!full);
        if (stop) { const u32 f = ctz32(stop); return total + 8 * f + W::shfl(n, f); }
        total += 8 * W::lanes();
    }
}

// backward extension: how many bytes before (ip, mpos) are equal, not crossing anchor / position 0
template <class W> LZ_HD u32 extend_back_par(const u8* src, u32 ip, u32 mpos, u32 anchor)
{
    u32 done = 0;
    for (;;) {
        const u32 k = done + W::lane() + 1;
        const bool can = ip >= anchor + k && mpos >= k;
        const bool eq = can && src[ip - k] == src[mpos - k];
        const u32 bad = W::ballot(!eq);
        if (bad) return done + ctz32(bad);
        done += W::lanes();
    }
}

// Lizard_compress_fastSmall / Lizard_compress_fast with the no-match run probed W::lanes() positions at a
// time.  Exactness argument: inside one search the probe positions do not depend on the data, each probe
// reads its bucket after all earlier probes wrote theirs, and the search stops at the first probe that
// matches.  So lanes evaluate probes j0..j0+L-1 together; a lane's candidate is the latest earlier lane of
// the same batch with the same bucket, else the table; the lowest hitting lane wins and only buckets of
// lanes up to the winner are committed (last writer per bucket).
// kBig = Lizard_compress_fastBig (lib/lizard_parser_fastbig.h:35-175, levels 20 / 40): the same walk with LIZv1 codewords
// and one more acceptance rule -- a candidate 65536 or more bytes back is only taken when the match (backward extension
// included; the post-match probe: forward part only) is at least MM_LONGOFF + MINMATCH long (:99, :142); a refused
// candidate is an ordinary miss: its position stays in the table and the search goes on with the next probe.
template <class W, class TT, bool kBig = false> LZ_HD void parse_fast_par(const ParseCtx<TT>& c, u32 b0, u32 b1, EncStreams& s)
{
    const u8* const src = c.src;
    const TT T = c.T;
    const u32 hl = c.hash_log;
    const u32 lane = W::lane(), NL = W::lanes();
    const bool wr = lane == 0;
    const u32 max_dist = (1u << c.window_log) - 1;
    const u32 bias = kDictSize;
    const u32 low_limit = (bias + max_dist >= b0 + bias) ? bias : b0 + bias - max_dist;
    u32 anchor = b0, ip = b0;
    u32 ml = 0, mpos = 0;
    u32 last_off = 0;                                                          // LIZv1 emitter state (kBig)
    if (b1 - b0 < kMinInputForLz) goto last_literals;
    {
        const u32 mflimit = b1 - kMfLimit;
        const u8* const matchlimit = src + b1 - kLastLiterals;
        if (wr) { const u64 v0 = ld5(src + ip); T.set_t(hash5(v0, hl), ip + bias, tag8((u32)v0)); }
        W::sync();
        ip++;
        for (;;) {
            {   // ---- search: batches of NL probes ----
                const u32 ip0 = ip;
                u32 j0 = 0;
                u64 v_ahead = 0; bool have_ahead = false;                      // next batch's bytes, requested one batch early
                for (;;) {
                  u32 j_hit = 0;
                  for (;;) {
                    const u32 j = j0 + lane;
                    const u32 P = ip0 + probe_offset(j);
                    const bool valid = ip0 + probe_offset(j + 1) <= mflimit;   // else this probe ends the block
                    u64 v = 0; u32 h = 0x80000000u | lane;                     // unique key: matches nobody
                    if (valid) { v = have_ahead ? v_ahead : ld5(src + P); h = hash5(v, hl); }
                    have_ahead = false;
                    if (j0) {   // a search that missed a whole batch tends to go on: request the next batch's bytes now so
                                // that their latency overlaps this batch's bucket / candidate work
                        const u32 jn = j + NL;
                        have_ahead = ip0 + probe_offset(jn + 1) <= mflimit;
                        v_ahead = have_ahead ? ld5(src + ip0 + probe_offset(jn)) : 0;
                    }
                    const u32 peers = W::match_any(h);
                    const u32 below = peers & ((1u << lane) - 1);
                    const u32 pl = below ? highbit32(below) : lane;
                    const u32 prevP = W::shfl(P, pl);
                    const u32 cur = P + bias;
                    u32 cand = 0, ctag = kNoTag;
                    if (valid) cand = below ? prevP + bias : T.get_t(h, P, &ctag);
                    bool hit = false;
                    if (valid && cand >= low_limit && cand < cur && cand + max_dist >= cur && cur - cand >= kMinOffset &&
                        T.maybe(ctag, tag8((u32)v)))
                        hit = ld32(src + (cand - bias)) == (u32)v;
                    const u32 hits = W::ballot(hit);
                    const u32 term = W::ballot(!valid);
                    const u32 w_lane = hits ? ctz32(hits) : 32;
                    const u32 t_lane = term ? ctz32(term) : 32;
                    const bool matched = w_lane < t_lane;
                    // lanes whose table write happens in program order before the search stops
                    u32 commit;
                    if (matched) commit = (w_lane >= 31) ? 0xffffffffu : ((2u << w_lane) - 1);
                    else commit = (t_lane >= 32) ? 0xffffffffu : ((1u << t_lane) - 1);
                    W::sync();
                    if ((commit >> lane) & 1) {
                        const u32 grp = peers & commit;
                        if (highbit32(grp) == lane) T.set_t(h, cur, tag8((u32)v));
                    }
                    W::sync();
                    if (matched) { ip = W::shfl(P, w_lane); mpos = W::shfl(cand, w_lane) - bias; j_hit = j0 + w_lane; break; }
                    if (t_lane < 32) { goto last_literals; }
                    j0 += NL;
                  }
                  ml = count_match_par<W>(src + ip + kMinMatch, src + mpos + kMinMatch, matchlimit);
                  const u32 back = extend_back_par<W>(src, ip, mpos, anchor);
                  if (kBig && ml + back < kMmLongOff && ip - mpos >= kMax16BitOffset) {   // refused: the search goes on behind it
                      j0 = j_hit + 1; have_ahead = false;
                      continue;
                  }
                  ip -= back; mpos -= back; ml += back;
                  break;
                }
            }
            for (;;) {   // _next_match
                if (kBig) emit_lizv1<W>(s, src, anchor, ip, ml + kMinMatch, ip - mpos, last_off);
                else emit_lz4<W>(s, src, anchor, ip, ml + kMinMatch, ip - mpos);
                ip += ml + kMinMatch;
                anchor = ip;
                if (ip > mflimit) goto last_literals;
                if (wr) { const u64 v2 = ld5(src + ip - 2); T.set_t(hash5(v2, hl), ip - 2 + bias, tag8((u32)v2)); }
                W::sync();
                const u64 v = ld5(src + ip);
                const u32 h = hash5(v, hl);
                u32 ctag = kNoTag;
                const u32 cand = T.get_t(h, ip, &ctag);
                W::sync();
                if (wr) T.set_t(h, ip + bias, tag8((u32)v));
                W::sync();
                const u32 cur = ip + bias;
                if (cand >= low_limit && cand < cur && cand + max_dist >= cur && cur - cand >= kMinOffset &&
                    T.maybe(ctag, tag8((u32)v))) {
                    mpos = cand - bias;
                    if (ld32(src + mpos) == (u32)v) {
                        ml = count_match_par<W>(src + ip + kMinMatch, src + mpos + kMinMatch, matchlimit);
                        if (!kBig || ml >= kMmLongOff || ip - mpos < kMax16BitOffset) continue;
                    }
                }
                break;
            }
            ip++;
        }
    }
last_literals:
    emit_last_literals<W>(s, src, anchor, b1);
}

// ---- window form of the same parser (32-lane warps) ------------------------------------------------------------
// parse_fast_par spends one batch per sequence plus a serial "next match" step (insert ip-2, probe ip).  Here a
// window is 32 CONSECUTIVE positions w0..w0+31 whose bytes, hashes, table values and table-candidate comparisons are
// fetched once, in parallel; the reference's walk over those positions is then replayed with ballots and shuffles
// only, for as many sequences as end inside the window:
//   * `committed` = lanes whose position the reference has inserted into the table so far (program order = lane
//     order, because positions only grow);
//   * a walk segment starts at lane `s`: either the post-match probe of position ip (has_next; lizard_parser_
//     fastsmall.h:138-160: insert ip-2, probe ip) followed by a fresh search from ip+1, or a search in progress;
//   * lane L's bucket content at its turn is the latest lane below it that is committed or lies in [s, L) and
//     shares the bucket, else the table value read at the start of the window.  An in-window candidate is compared
//     through a shuffle (its first four bytes are that lane's own bytes), so no memory access is needed;
//   * the lowest hitting lane ends the segment; lanes [s, hit] become committed; after the match is measured and
//     recorded, ip-2 is committed and the walk resumes at ip if that is still inside the window.
// When the walk leaves the window the committed lanes write their buckets (last writer per bucket wins).
// Consecutive positions hold while a search has made at most 65 probes (probe_offset); a longer miss run falls
// back to the batch search with its growing stride.
#if !defined(LZB_ENC_SRC_PF)
#define LZB_ENC_SRC_PF 384
#endif
template <class W, class TT, bool kBig = false> LZ_HD void parse_fast_win(const ParseCtx<TT>& c, u32 b0, u32 b1, EncStreams& st)
{
    const u8* const src = c.src;
    const TT T = c.T;
    const u32 hl = c.hash_log;
    const u32 lane = W::lane(), NL = W::lanes();
    const u32 max_dist = (1u << c.window_log) - 1;
    const u32 bias = kDictSize;
    const u32 low_limit = (bias + max_dist >= b0 + bias) ? bias : b0 + bias - max_dist;
    const u32 lt_mask = (1u << lane) - 1;
    u32 anchor = b0;
    u32 last_off = 0;                                              // LIZv1 emitter state (kBig)
    if (b1 - b0 >= kMinInputForLz) {
        const u32 mflimit = b1 - kMfLimit;
        const u8* const matchlimit = src + b1 - kLastLiterals;
        // window state
        u32 w0 = b0;            // first position
        u32 committed = 1;      // position b0 is inserted before the first search (lizard_parser_fastsmall.h:51-53)
        u32 s = 1;              // the first search starts at b0+1
        bool has_next = false;
        u32 jbase = 0;          // probe number of lane s + has_next within its search
        for (;;) {
            // ---- fetch: everything memory-bound, once per window ----
            const u32 P = w0 + lane;
            const bool ld_ok = P <= mflimit;
            const bool s_valid = P + 1 <= mflimit;                 // as a search probe: else it ends the block
            u64 v = 0; u32 h = 0x80000000u | lane;                 // unique key: shares a bucket with nobody
            if (ld_ok) { v = ld5(src + P); h = hash5(v, hl); }
            if (P + LZB_ENC_SRC_PF < b1) W::prefetch(src + P + LZB_ENC_SRC_PF);   // the input is walked once, front to back
            const u32 same = W::match_any(h);
            const u32 below = same & lt_mask;
            const u32 mytag = tag8((u32)v);
            u32 ttag = kNoTag;
            const u32 tv = ld_ok ? T.get_t(h, P, &ttag) : 0u;
            bool hit_t = false;
            {
                const u32 cur = P + bias;
                if (ld_ok && tv >= low_limit && tv < cur && tv + max_dist >= cur && cur - tv >= kMinOffset && T.maybe(ttag, mytag))
                    hit_t = ld32(src + (tv - bias)) == (u32)v;
            }
            // ---- replay the reference's walk over the window ----
            u32 slow_ip0 = 0, slow_j0 = 0; bool go_slow = false, finished = false;
            u32 refused = 0;                                       // kBig: lanes whose far candidate was too short -- plain misses
            for (;;) {
                const u32 ge_s = ~((1u << s) - 1);
                const u32 m = below & (committed | ge_s);
                const u32 pl = m ? highbit32(m) : lane;
                const u32 pv = W::shfl((u32)v, pl);
                bool hit = m ? (pv == (u32)v && lane - pl >= kMinOffset) : hit_t;
                const u32 a = s + (has_next ? 1u : 0u);            // first lane acting as a search probe
                hit = hit && lane >= s && (s_valid || (has_next && lane == s));
                if (kBig) hit = hit && !((refused >> lane) & 1u);
                const u32 hits = W::ballot(hit);
                const u32 term = W::ballot(lane >= a && !s_valid);
                const u32 w_lane = hits ? ctz32(hits) : 32;
                const u32 t_lane = term ? ctz32(term) : 32;
                if (w_lane < t_lane) {
                    const u32 cpos = m ? w0 + pl : tv - bias;
                    u32 ip = w0 + w_lane;
                    u32 mpos = W::shfl(cpos, w_lane);
                    u32 ml = count_match_par<W>(src + ip + kMinMatch, src + mpos + kMinMatch, matchlimit);
                    u32 back = 0;
                    if (!(has_next && w_lane == s)) back = extend_back_par<W>(src, ip, mpos, anchor);   // the post-match probe is taken as it is
                    if (kBig && ml + back < kMmLongOff && ip - mpos >= kMax16BitOffset) { refused |= 1u << w_lane; continue; }
                    committed |= ge_s & (w_lane >= 31 ? 0xffffffffu : ((2u << w_lane) - 1));
                    ip -= back; mpos -= back; ml += back;
                    if (kBig) emit_lizv1<W>(st, src, anchor, ip, ml + kMinMatch, ip - mpos, last_off);
                    else emit_lz4<W>(st, src, anchor, ip, ml + kMinMatch, ip - mpos);
                    ip += ml + kMinMatch;
                    anchor = ip;
                    if (ip > mflimit) { finished = true; break; }
                    const u32 lp = ip - w0;
                    if (lp < NL) { committed |= 1u << (lp - 2); s = lp; has_next = true; jbase = 0; continue; }
                    break;                                          // next window starts at ip-2
                }
                if (t_lane < 32) { committed |= ge_s & ((1u << t_lane) - 1); finished = true; anchor |= 0; break; }
                // the whole rest of the window missed: the search goes on
                committed |= ge_s;
                slow_j0 = jbase + (NL - a);
                slow_ip0 = w0 + a - jbase;
                go_slow = true;
                break;
            }
            // ---- leave the window: committed lanes write their buckets, last writer per bucket ----
            W::sync();
            if ((committed >> lane) & 1) {
                const u32 grp = same & committed;
                if (highbit32(grp) == lane) T.set_t(h, P + bias, mytag);
            }
            W::sync();
            if (finished) break;
            if (!go_slow) { w0 = anchor - 2; committed = 1; s = 2; has_next = true; jbase = 0; continue; }
            if (slow_j0 + NL <= 66) { w0 += NL; committed = 0; s = 0; has_next = false; jbase = slow_j0; continue; }
            // ---- long miss run: batch search with the growing stride (as parse_fast_par) ----
            {
                const u32 ip0 = slow_ip0;
                u32 j0 = slow_j0;
                u32 ip = 0, mpos = 0, ml = 0; bool ended = false;
                for (;;) {
                  u32 j_hit = 0;
                  for (;;) {
                    const u32 j = j0 + lane;
                    const u32 Pj = ip0 + probe_offset(j);
                    const bool valid = ip0 + probe_offset(j + 1) <= mflimit;
                    u64 vj = 0; u32 hj = 0x80000000u | lane;
                    if (valid) { vj = ld5(src + Pj); hj = hash5(vj, hl); }
                    if (Pj + 512 < b1) W::prefetch(src + Pj + 512);
                    const u32 peers = W::match_any(hj);
                    const u32 blw = peers & lt_mask;
                    const u32 plj = blw ? highbit32(blw) : lane;
                    const u32 prevP = W::shfl(Pj, plj);
                    const u32 prevV = W::shfl((u32)vj, plj);         // the four bytes at prevP
                    const u32 cur = Pj + bias;
                    u32 cand = 0, ctag = kNoTag;
                    if (valid) cand = blw ? prevP + bias : T.get_t(hj, Pj, &ctag);
                    bool hit = false;
                    if (valid && cand >= low_limit && cand < cur && cand + max_dist >= cur && cur - cand >= kMinOffset) {
                        if (blw) hit = prevV == (u32)vj;
                        else if (T.maybe(ctag, tag8((u32)vj))) hit = ld32(src + (cand - bias)) == (u32)vj;
                    }
                    const u32 hits = W::ballot(hit);
                    const u32 term = W::ballot(!valid);
                    const u32 w_lane = hits ? ctz32(hits) : 32;
                    const u32 t_lane = term ? ctz32(term) : 32;
                    const bool matched = w_lane < t_lane;
                    u32 commit;
                    if (matched) commit = (w_lane >= 31) ? 0xffffffffu : ((2u << w_lane) - 1);
                    else commit = (t_lane >= 32) ? 0xffffffffu : ((1u << t_lane) - 1);
                    W::sync();
                    if ((commit >> lane) & 1) {
                        const u32 grp = peers & commit;
                        if (highbit32(grp) == lane) T.set_t(hj, cur, tag8((u32)vj));
                    }
                    W::sync();
                    if (matched) { ip = W::shfl(Pj, w_lane); mpos = W::shfl(cand, w_lane) - bias; j_hit = j0 + w_lane; break; }
                    if (t_lane < 32) { ended = true; break; }
                    j0 += NL;
                  }
                  if (ended) break;
                  ml = count_match_par<W>(src + ip + kMinMatch, src + mpos + kMinMatch, matchlimit);
                  const u32 back = extend_back_par<W>(src, ip, mpos, anchor);
                  if (kBig && ml + back < kMmLongOff && ip - mpos >= kMax16BitOffset) { j0 = j_hit + 1; continue; }   // refused
                  ip -= back; mpos -= back; ml += back;
                  break;
                }
                if (ended) break;
                if (kBig) emit_lizv1<W>(st, src, anchor, ip, ml + kMinMatch, ip - mpos, last_off);
                else emit_lz4<W>(st, src, anchor, ip, ml + kMinMatch, ip - mpos);
                ip += ml + kMinMatch;
                anchor = ip;
                if (ip > mflimit) break;
                w0 = ip - 2; committed = 1; s = 2; has_next = true; jbase = 0;
            }
        }
    }
    emit_last_literals<W>(st, src, anchor, b1);
}

// ---- hashChain parser (levels 13-17 / 34-38): lib/lizard_parser_hashchain.h ---------------------------------------
// LZ4HC-style: every position is entered into bucket + chain (the chain stores the distance to the previous position
// of the same bucket, clamped to the window), a search walks at most searchNum chain links and keeps the longest
// match, and up to three overlapping candidates are arbitrated before the first one is written.  The control flow is
// uniform over the warp; lanes share the work of inserting a range of positions (same-bucket groups are replayed in
// order, as in the priceFast search) and of measuring a candidate (forward / backward extension).
struct ChainState {
    u16* chain;          // [1 << chainLog] distance to the previous position of the bucket (<= 65535 = the window)
    u32  chain_mask;
    u32  next_insert;    // first position of the unit not yet entered (ctx->nextToUpdate)
    u32  search_num;
    u32  mls;            // 5 -> hash5, 4 -> hash4 (Lizard_hashPtr, lizard_compress.c:99-109)
};
LZ_HD u32 hc_hash(const u8* p, u32 hl, u32 mls)
{
    if (mls == 5) return hash5(ld64(p), hl);
    return (u32)(ld32(p) * 2654435761U) >> (32 - hl);
}
// Lizard_Insert (:13-41): positions [next_insert, upto)
template <class W, class TT> LZ_HD void hc_insert(const u8* src, const TT& T, u32 hl, u32 max_dist, ChainState& cs, u32 upto)
{
    const u32 lane = W::lane(), NL = W::lanes(), bias = kDictSize;
    for (u32 base = cs.next_insert; base < upto; base += NL) {
        const u32 P = base + lane;
        const bool valid = P < upto;
        const u32 idx = P + bias;
        u32 h = 0x80000000u | lane;
        if (valid) h = hc_hash(src + P, hl, cs.mls);
        const u32 peers = W::match_any(h);
        u32 below = peers & ((1u << lane) - 1);
        u32 seen = valid ? T.get(h, P) : 0;
        while (below) {                                   // earlier lanes of the same bucket, in order
            const u32 bl = ctz32(below); below &= below - 1;
            const u32 pb = base + bl + bias;
            if (seen >= pb || pb >= seen + kMinOffset) seen = pb;
        }
        if (valid) {
            const u32 dist = idx - seen;
            cs.chain[P & cs.chain_mask] = (u16)(dist > max_dist ? max_dist : dist);
        }
        const u32 newval = (seen >= idx || idx >= seen + kMinOffset) ? idx : seen;
        W::sync();
        if (valid && highbit32(peers) == lane) T.set(h, newval);
        W::sync();
    }
    cs.next_insert = upto;
}
// DictTable helpers.  Lizard_count_2segments (lizard_compress.c:118-124): a match read from the external dictionary that
// reaches its end goes on at the unit's first byte.
template <class W> LZ_HD u32 count_2seg(const u8* a, const u8* b, const u8* a_limit, const u8* b_end, const u8* a_start)
{
    const u8* v_end = (size_t)(b_end - b) < (size_t)(a_limit - a) ? a + (b_end - b) : a_limit;
    const u32 n = count_match_par<W>(a, b, v_end);
    if (b + n != b_end) return n;
    return n + count_match_par<W>(a + n, a_start, a_limit);
}
template <class W> LZ_HD u32 count_2seg_1(const u8* a, const u8* b, const u8* a_limit, const u8* b_end, const u8* a_start)
{   // the same with one lane
    const u8* v_end = (size_t)(b_end - b) < (size_t)(a_limit - a) ? a + (b_end - b) : a_limit;
    const u32 n = count_match(a, b, v_end);
    if (b + n != b_end) return n;
    return n + count_match(a + n, a_start, a_limit);
}
#if defined(LZB_DICT_ENC_STATS) && !defined(__CUDA_ARCH__)
// host shim only: matches of the priceFast dictionary parse that start in the dictionary (tests prove both kinds occur)
enum { kDictRepInDict, kDictMatchInDict, kDictEncStats };
extern unsigned long long g_dict_enc_stats[kDictEncStats];
#define LZB_DICT_COUNT(k) do { if (W::lane() == 0) g_dict_enc_stats[k]++; } while (0)
#else
#define LZB_DICT_COUNT(k) do { } while (0)
#endif
// backward extension with the two sides in different buffers: a[ip - k] against b[mpos - k], ip - k >= floor, mpos - k >= mlow
template <class W> LZ_HD u32 extend_back_2seg(const u8* a, u32 ip, const u8* b, u32 mpos, u32 floor, u32 mlow)
{
    u32 done = 0;
    for (;;) {
        const u32 k = done + W::lane() + 1;
        const bool can = ip >= floor + k && mpos >= mlow + k;
        const bool eq = can && a[ip - k] == b[mpos - k];
        const u32 bad = W::ballot(!eq);
        if (bad) return done + ctz32(bad);
        done += W::lanes();
    }
}
template <class TT> LZ_HD u32 hc_next(const TT& T, const ChainState& cs, u32 c)
{
    if constexpr (TT::kDict) { if (c < T.own0) return T.dchain[c & 0xFFFFu]; }   // inserted by Lizard_loadDict
    return cs.chain[c & cs.chain_mask];
}

// Lizard_InsertAndFindBestMatch (:45-106); returns the length (0 = none), *ref = match position
template <class W, class TT> LZ_HD u32 hc_best(const u8* src, const TT& T, u32 hl, u32 max_dist, ChainState& cs,
                                               u32 ip, const u8* limit, u32* ref)
{
    const u32 bias = kDictSize, cur = ip + bias;
    u32 low = (bias + max_dist >= cur) ? bias : cur - max_dist;
    if constexpr (TT::kDict) low = (T.low + max_dist >= cur) ? T.low : cur - max_dist;
    hc_insert<W, TT>(src, T, hl, max_dist, cs, ip);
    u32 m = T.get(hc_hash(src + ip, hl, cs.mls), ip);
    u32 tries = cs.search_num, best = 0;
    const u32 v = ld32(src + ip);
    while (m < cur && m >= low && tries) {
        const u32 c = m - bias;
        tries--;
        bool ext_dict = false;
        if constexpr (TT::kDict) ext_dict = T.ext && c < T.dend;
        if (ext_dict) {                                  // the external dictionary's branch (:85-97)
            if constexpr (TT::kDict) {
                if (ip - c >= kMinOffset && T.dend - 1 - c >= 3 && ld32(T.dsrc + c) == v) {
                    const u32 len = count_2seg<W>(src + ip + kMinMatch, T.dsrc + c + kMinMatch, limit, T.dsrc + T.dend, src + T.dend) + kMinMatch;
                    if (len > best) { best = len; *ref = c; }
                }
            }
        } else if (ip - c >= kMinOffset && src[c + best] == src[ip + best] && ld32(src + c) == v) {
            const u32 len = count_match_par<W>(src + ip + kMinMatch, src + c + kMinMatch, limit) + kMinMatch;
            if (len > best) { best = len; *ref = c; }
        }
        const u32 d = hc_next(T, cs, c);
        if (d > m) break;
        m -= d;
    }
    return best;
}
// Lizard_InsertAndGetWiderMatch (:109-185): candidates may also grow backwards, down to `floor`
template <class W, class TT> LZ_HD u32 hc_wider(const u8* src, const TT& T, u32 hl, u32 max_dist, ChainState& cs,
                                                u32 ip, u32 floor, const u8* limit, u32 longest, u32* ref, u32* start)
{
    const u32 bias = kDictSize, cur = ip + bias;
    u32 low = (bias + max_dist >= cur) ? bias : cur - max_dist;
    if constexpr (TT::kDict) low = (T.low + max_dist >= cur) ? T.low : cur - max_dist;
    const u32 lead = ip - floor;
    hc_insert<W, TT>(src, T, hl, max_dist, cs, ip);
    u32 m = T.get(hc_hash(src + ip, hl, cs.mls), ip);
    u32 tries = cs.search_num;
    const u32 v = ld32(src + ip);
    while (m < cur && m >= low && tries) {
        const u32 c = m - bias;
        tries--;
        bool ext_dict = false;
        if constexpr (TT::kDict) ext_dict = T.ext && c < T.dend;
        if (ext_dict) {                                  // the external dictionary's branch (:158-170): back down to the window
            if constexpr (TT::kDict) {
                if (ip - c >= kMinOffset && T.dend - 1 - c >= 3 && ld32(T.dsrc + c) == v) {
                    u32 len = kMinMatch + count_2seg<W>(src + ip + kMinMatch, T.dsrc + c + kMinMatch, limit, T.dsrc + T.dend, src + T.dend);
                    const u32 back = extend_back_2seg<W>(src, ip, T.dsrc, c, floor, low - bias);
                    len += back;
                    if (len > longest) { longest = len; *ref = c - back; *start = ip - back; }
                }
            }
        // c - lead + longest >= c + 3 in both call sites (lead = longest - 3), so the probe stays inside the unit
        } else if (ip - c >= kMinOffset && src[floor + longest] == src[c - lead + longest] && ld32(src + c) == v) {
            u32 len = kMinMatch + count_match_par<W>(src + ip + kMinMatch, src + c + kMinMatch, limit);
            u32 back;
            if constexpr (TT::kDict) {   // back down to lowPrefixPtr: the unit's start, or the prefix dictionary's
                const u32 p0 = T.ext ? T.dend : 0u;
                back = extend_back_par<W>(src + p0, ip - p0, c - p0, floor - p0);
            } else back = extend_back_par<W>(src, ip, c, floor);
            len += back;
            if (len > longest) { longest = len; *ref = c - back; *start = ip - back; }
        }
        const u32 d = hc_next(T, cs, c);
        if (d > m) break;
        m -= d;
    }
    return longest;
}
// Lizard_compress_hashChain (:188-369).  a = the match about to be written, b / c = the later candidates.
template <class W, class TT> LZ_HD_COLD void parse_hash_chain(const ParseCtx<TT>& c, u32 b0, u32 b1, EncStreams& st, ChainState& cs)
{
    const u8* const src = c.src;
    const TT T = c.T;
    const u32 hl = c.hash_log;
    const u32 max_dist = (1u << c.window_log) - 1;
    const int kOpt = 18;                                     // OPTIMAL_ML = (ML_MASK_LZ4 - 1) + MINMATCH
    u32 anchor = b0;
    if (b1 - b0 > kMfLimit + 1) {
        const u32 mflimit = b1 - kMfLimit;
        const u8* const matchlimit = src + b1 - kLastLiterals;
        u32 ip = b0 + 1;
        int la = 0, lb = 0, lc = 0, l0 = 0;
        u32 ra = 0, sb = 0, rb = 0, sc = 0, rc = 0, s0 = 0, r0 = 0;
        while (ip < mflimit) {
            la = (int)hc_best<W, TT>(src, T, hl, max_dist, cs, ip, matchlimit, &ra);
            if (!la) { ip++; continue; }
            s0 = ip; r0 = ra; l0 = la;
            bool again2 = true;                               // _Search2
            while (again2) {
                again2 = false;
                lb = (ip + (u32)la < mflimit) ? (int)hc_wider<W, TT>(src, T, hl, max_dist, cs, ip + (u32)la - 2, ip + 1, matchlimit, (u32)la, &rb, &sb) : la;
                if (lb == la) { emit_lz4<W>(st, src, anchor, ip, (u32)la, ip - ra); ip += (u32)la; anchor = ip; break; }
                if (s0 < ip && sb < ip + (u32)l0) { ip = s0; ra = r0; la = l0; }
                if ((int)(sb - ip) < 3) { la = lb; ip = sb; ra = rb; again2 = true; continue; }
                bool again3 = true;                           // _Search3
                while (again3) {
                    again3 = false;
                    if ((int)(sb - ip) < kOpt) {
                        int keep = la > kOpt ? kOpt : la;
                        if ((long)ip + keep > (long)sb + lb - (int)kMinMatch) {
                            keep = (int)(sb - ip) + lb - (int)kMinMatch;
                            if (keep < (int)kMinMatch) { emit_lz4<W>(st, src, anchor, ip, (u32)la, ip - ra); ip += (u32)la; anchor = ip; break; }
                        }
                        const int shift = keep - (int)(sb - ip);
                        if (shift > 0) { sb += (u32)shift; rb += (u32)shift; lb -= shift; }
                    }
                    lc = (sb + (u32)lb < mflimit) ? (int)hc_wider<W, TT>(src, T, hl, max_dist, cs, sb + (u32)lb - 3, sb, matchlimit, (u32)lb, &rc, &sc) : lb;
                    if (lc == lb) {                            // two sequences
                        if (sb < ip + (u32)la) la = (int)(sb - ip);
                        emit_lz4<W>(st, src, anchor, ip, (u32)la, ip - ra); ip += (u32)la; anchor = ip;
                        ip = sb;
                        emit_lz4<W>(st, src, anchor, ip, (u32)lb, ip - rb); ip += (u32)lb; anchor = ip;
                        break;
                    }
                    if (sc < ip + (u32)la + 3) {               // no room for b
                        if (sc >= ip + (u32)la) {              // write a; b is dropped or trimmed, c becomes a
                            if (sb < ip + (u32)la) {
                                const int shift = (int)(ip + (u32)la - sb);
                                sb += (u32)shift; rb += (u32)shift; lb -= shift;
                                if (lb < (int)kMinMatch) { sb = sc; rb = rc; lb = lc; }
                            }
                            emit_lz4<W>(st, src, anchor, ip, (u32)la, ip - ra); ip += (u32)la; anchor = ip;
                            ip = sc; ra = rc; la = lc;
                            s0 = sb; r0 = rb; l0 = lb;
                            again2 = true;
                            break;
                        }
                        sb = sc; rb = rc; lb = lc;
                        again3 = true;
                        continue;
                    }
                    if (sb < ip + (u32)la) {                   // three ascending candidates: write the first
                        if ((int)(sb - ip) < 15) {             // ML_MASK_LZ4
                            if (la > kOpt) la = kOpt;
                            if ((long)ip + la > (long)sb + lb - (int)kMinMatch) {
                                la = (int)(sb - ip) + lb - (int)kMinMatch;
                                if (la < (int)kMinMatch) {
                                    emit_lz4<W>(st, src, anchor, ip, (u32)la, ip - ra); ip += (u32)la; anchor = ip;
                                    ip = sc; ra = rc; la = lc;
                                    s0 = sb; r0 = rb; l0 = lb;
                                    again2 = true;
                                    break;
                                }
                            }
                            const int shift = la - (int)(sb - ip);
                            if (shift > 0) { sb += (u32)shift; rb += (u32)shift; lb -= shift; }
                        } else la = (int)(sb - ip);
                    }
                    emit_lz4<W>(st, src, anchor, ip, (u32)la, ip - ra); ip += (u32)la; anchor = ip;
                    ip = sb; ra = rb; la = lb;
                    sb = sc; rb = rc; lb = lc;
                    again3 = true;
                }
            }
        }
    }
    emit_last_literals<W>(st, src, anchor, b1);
}

// priceFast's backward extension against a loaded dictionary: down to lowPrefixPtr (:177, :195), the unit's start or the prefix
// dictionary's.  A candidate in an external dictionary lies below lowPrefixPtr as a virtual pointer, so it never extends.
template <class W> LZ_HD u32 dict_back(const DictTable& T, const u8* src, u32 ip, u32 ref, u32 floor)
{
    if (T.ext && ref < T.dend) return 0;
    const u32 p0 = T.ext ? T.dend : 0u;
    return extend_back_par<W>(src + p0, ip - p0, ref - p0, floor - p0);
}

// Lizard_compress_priceFast with the no-match run probed W::lanes() consecutive positions at a time.
// Per position the reference (lizard_parser_pricefast.h:158-173) tests the repeat offset first, then the
// bucket's candidate, then conditionally refreshes the bucket.  last_off is constant during a no-match run,
// positions advance by one, so L lanes evaluate L consecutive positions; the only cross-lane dependency is
// the bucket value, which each lane reconstructs by replaying the conditional updates of the earlier lanes
// that share its bucket.  The lowest hitting lane wins; buckets of lanes up to the winner are committed.
template <class W, class TT> LZ_HD void parse_price_fast_par(const ParseCtx<TT>& c, u32 b0, u32 b1, EncStreams& s, u32 min_match_long)
{
    const u8* const src = c.src;
    const TT T = c.T;
    const u32 hl = c.hash_log;
    const u32 lane = W::lane(), NL = W::lanes();
    const bool wr = lane == 0;
    const u32 bias = kDictSize;
    const u32 max_dist = (1u << c.window_log) - 1;
    u32 anchor = b0, ip = b0 + 1;
    u32 last_off = 0;
    u64 v_ahead = 0; u32 ahead_pos = 0xffffffffu;              // per lane: bytes at position ahead_pos, if loaded
    // (Prefetching the NEXT batch's buckets one batch early -- prefetch.global.L2 on the plain table, with the input requested
    // two batches ahead -- gave no speed-up and more DRAM traffic; not kept.)
    if (b1 - b0 >= kMfLimit) {
    const u32 mflimit = b1 - kMfLimit;
    const u8* const matchlimit = src + b1 - kLastLiterals;
    while (ip < mflimit) {
        u32 ml = 0, ref = 0;
        {   // ---- batch of NL positions ----
            const u32 P = ip + lane;
            const bool valid = P < mflimit;
            const u32 cur = P + bias;
            u32 low = (bias + max_dist >= cur) ? bias : cur - max_dist;
            if constexpr (TT::kDict) low = (T.low + max_dist >= cur) ? T.low : cur - max_dist;
            u64 v = 0; u32 h = 0x80000000u | lane;
            if (valid) { v = (ahead_pos == P) ? v_ahead : ld5(src + P); h = hash5(v, hl); }
            {   // request the bytes of the following NL positions one batch early (used if this batch finds nothing)
                const u32 Pn = P + NL;
                ahead_pos = Pn < mflimit ? Pn : 0xffffffffu;
                v_ahead = Pn < mflimit ? ld5(src + Pn) : 0;
            }
            const u32 peers = W::match_any(h);
            u32 below = peers & ((1u << lane) - 1);
            const u32 mytag = tag8((u32)v);
            u32 ttag = kNoTag;
            u32 seen = valid ? T.get_t(h, P, &ttag) : 0;
            u32 seen_lane = NL;                               // whose position `seen` is: an earlier lane's, or the table's (NL)
            while (below) {                                   // replay earlier same-bucket lanes, in order
                const u32 bl = ctz32(below); below &= below - 1;
                const u32 pb = ip + bl + bias;
                if (seen >= pb || pb >= seen + kMinOffset) { seen = pb; seen_lane = bl; }
            }
            // the four bytes at an earlier lane's position are that lane's own bytes: no memory access for those
            const u32 seen_v = W::shfl((u32)v, seen_lane < NL ? seen_lane : lane);
            bool rep_hit = false, hash_hit = false;
            if (valid) {
                if (last_off >= kMinOffset && last_off <= P && cur - last_off >= low) {
                    bool ext_dict = false;
                    if constexpr (TT::kDict) ext_dict = T.ext && P - last_off < T.dend;
                    if (ext_dict) {                            // the external dictionary's branch (lizard_parser_pricefast.h:32-42)
                        if constexpr (TT::kDict)
                            rep_hit = T.dend - 1 - (P - last_off) >= 3 && ld32(T.dsrc + (P - last_off)) == (u32)v;
                    } else rep_hit = ld32(src + (P - last_off)) == (u32)v;
                }
                if (!rep_hit && seen < cur && seen >= low) {
                    const u32 m = seen - bias;
                    bool eq4 = false, ext_dict = false;
                    if constexpr (TT::kDict) ext_dict = T.ext && m < T.dend;
                    if (P - m >= kMinOffset) {
                        if (seen_lane < NL) eq4 = seen_v == (u32)v;
                        else if (ext_dict) {                   // :76-85
                            if constexpr (TT::kDict) eq4 = T.dend - 1 - m >= 3 && ld32(T.dsrc + m) == (u32)v;
                        } else if (T.maybe(ttag, mytag)) eq4 = ld32(src + m) == (u32)v;
                    }
                    if (eq4) {
                        if (P - m < kMax16BitOffset) hash_hit = true;
                        else if (ext_dict) {
                            if constexpr (TT::kDict)
                                hash_hit = count_2seg_1<W>(src + P + kMinMatch, T.dsrc + m + kMinMatch, matchlimit, T.dsrc + T.dend,
                                                           src + T.dend) + kMinMatch >= min_match_long;
                        } else hash_hit = count_match(src + P + kMinMatch, src + m + kMinMatch, matchlimit) + kMinMatch >= min_match_long;
                    }
                }
            }
            const bool take = seen >= cur || cur >= seen + kMinOffset;
            const u32 newval = take ? cur : seen;
            const u32 new_lane = take ? lane : seen_lane;      // NL: the bucket keeps the table's entry, nothing to write
            const u32 new_tag = W::shfl(mytag, new_lane < NL ? new_lane : lane);
            const u32 hits = W::ballot(rep_hit || hash_hit);
            const u32 vmask = W::ballot(valid);
            const u32 w_lane = hits ? ctz32(hits) : 32;
            const u32 commit = (w_lane < 32) ? ((w_lane >= 31) ? 0xffffffffu : ((2u << w_lane) - 1)) : vmask;
            W::sync();
            if ((commit >> lane) & 1) {
                const u32 grp = peers & commit;
                if (highbit32(grp) == lane && new_lane < NL) T.set_t(h, newval, new_tag);
            }
            W::sync();
            if (w_lane == 32) { ip += NL; continue; }
            ip = W::shfl(P, w_lane);
            const u32 is_rep = W::shfl(rep_hit ? 1u : 0u, w_lane);
            ref = is_rep ? ip - last_off : W::shfl(seen, w_lane) - bias;
            if constexpr (TT::kDict) {
                if (ref < T.dend) LZB_DICT_COUNT(is_rep ? kDictRepInDict : kDictMatchInDict);
                if (T.ext && ref < T.dend)
                    ml = count_2seg<W>(src + ip + kMinMatch, T.dsrc + ref + kMinMatch, matchlimit, T.dsrc + T.dend, src + T.dend) + kMinMatch;
                else ml = count_match_par<W>(src + ip + kMinMatch, src + ref + kMinMatch, matchlimit) + kMinMatch;
            } else ml = count_match_par<W>(src + ip + kMinMatch, src + ref + kMinMatch, matchlimit) + kMinMatch;
        }

        u32 ml2 = 0, start2 = 0, ref2 = 0;
        bool encode_now = false;
        if (ip - ref == last_off) { ref = ip; encode_now = true; }
        else {
            u32 back;
            if constexpr (TT::kDict) back = dict_back<W>(T, src, ip, ref, anchor);
            else back = extend_back_par<W>(src, ip, ref, anchor);
            ip -= back; ref -= back; ml += back;
        }

        for (;;) {
            if (!encode_now) {
                while (true) {
                    if (ip + ml >= mflimit) break;
                    start2 = ip + ml - 2;
                    {   // Lizard_FindMatchFaster (uniform: one position)
                        const u32 cur2 = start2 + bias;
                        u32 low2 = (bias + max_dist >= cur2) ? bias : cur2 - max_dist;
                        if constexpr (TT::kDict) low2 = (T.low + max_dist >= cur2) ? T.low : cur2 - max_dist;
                        const u64 v2 = ld5(src + start2);
                        const u32 h2 = hash5(v2, hl);
                        u32 tag2 = kNoTag;
                        const u32 cand2 = T.get_t(h2, start2, &tag2);
                        ml2 = 0;
                        bool ok = false, ext_dict = false; u32 m = 0;
                        if (cand2 < cur2 && cand2 >= low2) {
                            m = cand2 - bias;
                            if constexpr (TT::kDict) ext_dict = T.ext && m < T.dend;
                            if (ext_dict) {                    // :118-126
                                if constexpr (TT::kDict) ok = start2 - m >= kMinOffset && T.dend - 1 - m >= 3 && ld32(T.dsrc + m) == (u32)v2;
                            } else ok = start2 - m >= kMinOffset && T.maybe(tag2, tag8((u32)v2)) && ld32(src + m) == (u32)v2;
                        }
                        W::sync();
                        if (wr && (cand2 >= cur2 || cur2 >= cand2 + kMinOffset)) T.set_t(h2, cur2, tag8((u32)v2));   // lizard_parser_pricefast.h:190
                        W::sync();
                        if (ok) {
                            u32 mlt;
                            if constexpr (TT::kDict) {
                                if (ext_dict) mlt = count_2seg<W>(src + start2 + kMinMatch, T.dsrc + m + kMinMatch, matchlimit, T.dsrc + T.dend, src + T.dend) + kMinMatch;
                                else mlt = count_match_par<W>(src + start2 + kMinMatch, src + m + kMinMatch, matchlimit) + kMinMatch;
                            } else mlt = count_match_par<W>(src + start2 + kMinMatch, src + m + kMinMatch, matchlimit) + kMinMatch;
                            if (mlt >= min_match_long || start2 - m < kMax16BitOffset) { ml2 = mlt; ref2 = m; }
                        }
                    }
                    if (!ml2) break;
                    {
                        u32 back;
                        if constexpr (TT::kDict) back = dict_back<W>(T, src, start2, ref2, ip);
                        else back = extend_back_par<W>(src, start2, ref2, ip);
                        start2 -= back; ref2 -= back; ml2 += back;
                    }
                    if (ml2 <= ml) { ml2 = 0; break; }
                    if (start2 <= ip) { ip = start2; ref = ref2; ml = ml2; ml2 = 0; break; }
                    if (start2 - ip < 3) { ip = start2; ref = ref2; ml = ml2; ml2 = 0; continue; }
                    if (start2 < ip + ml) {
                        const u32 corr = ml - (start2 - ip);
                        start2 += corr; ref2 += corr; ml2 -= corr;
                        if (ml2 < 3) ml2 = 0;
                        if (ml2 < min_match_long && start2 - ref2 >= kMax16BitOffset) ml2 = 0;
                    }
                    break;
                }
            }
            emit_lizv1<W>(s, src, anchor, ip, ml, ip - ref, last_off);
            ip += ml;
            anchor = ip;
            if (!ml2) break;
            ip = start2; ref = ref2; ml = ml2; ml2 = 0;
            encode_now = false;
        }
    }
    }
    emit_last_literals<W>(s, src, anchor, b1);
}

// ---- Huffman stage of one stream --------------------------------------------------------------------------
struct EncHufWork {               // per-warp scratch for the entropy stage
    HufEncScratch ws;
    u32 (*seg_count)[256];        // [4][256] per-segment byte histograms (shared memory on the device)
    u32 count[256];
    HufPlan plan;
    u32 pack[(kBlockSizePad + 512) / 4 + 64];   // aligned staging of packed segments
};

template <class W> LZ_HD void histogram4(const u8* p, u32 n, u32 seg, u32 (*seg_count)[256], u32* count)
{
    for (u32 i = W::lane(); i < 1024; i += W::lanes()) (&seg_count[0][0])[i] = 0;
    W::sync();
    for (u32 i = W::lane(); i < n; i += W::lanes()) {
        u32 k = i / seg;
#if defined(__CUDA_ARCH__)
        atomicAdd(&seg_count[k][p[i]], 1u);
#else
        seg_count[k][p[i]]++;
#endif
    }
    W::sync();
    for (u32 i = W::lane(); i < 256; i += W::lanes()) count[i] = seg_count[0][i] + seg_count[1][i] + seg_count[2][i] + seg_count[3][i];
    W::sync();
}

// Pack symbols p[0..m) last-to-first, LSB-first, then a 1 bit (HUF_compress1X_usingCTable).  `out` is a
// 4-byte aligned staging area; returns nothing, size is already known from the plan.
template <class W> LZ_HD void huf_pack_segment(u32* out, const u8* p, u32 m, const HufCode* codes)
{
    const u32 L = W::lanes(), lane = W::lane();
    const u32 chunk = (m + L - 1) / L;
    // lane l owns symbol indices [hi - chunk, hi) with hi = m - l*chunk, walked downward
    const long hi = (long)m - (long)lane * chunk;
    long lo = hi - (long)chunk; if (lo < 0) lo = 0;
    u32 mybits = 0;
    for (long i = hi - 1; i >= lo; --i) mybits += codes[p[i]].nbits;
    const bool owns_end = (lo == 0 && hi > 0) || (m == 0 && lane == 0);
    if (owns_end) mybits += 1;
    u32 total = 0;
    const u32 start = W::excl_scan(mybits, &total);
    if (mybits) { out[start >> 5] = 0; out[(start + mybits - 1) >> 5] = 0; }
    W::sync();
    if (mybits) {
        u64 acc = 0; u32 nacc = 0;          // bits waiting to be stored, aligned so that bit 0 is stream bit `pos`
        u32 pos = start;
        const u32 last_word = (start + mybits - 1) >> 5;
        // bring the accumulator to a word boundary view: keep (pos & 31) zero bits in front
        nacc = pos & 31; pos &= ~31u;
        for (long i = hi - 1; i >= lo; --i) {
            const HufCode c = codes[p[i]];
            acc |= (u64)c.val << nacc; nacc += c.nbits;
            if (nacc >= 32) {
                const u32 w = pos >> 5;
                const u32 v = (u32)acc;
                if (w == (start >> 5) || w == last_word) {
#if defined(__CUDA_ARCH__)
                    atomicOr(&out[w], v);
#else
                    out[w] |= v;
#endif
                } else out[w] = v;
                acc >>= 32; nacc -= 32; pos += 32;
            }
        }
        if (owns_end) { acc |= 1ull << nacc; nacc += 1; }
        while (nacc > 0) {
            const u32 w = pos >> 5;
            const u32 v = (u32)acc;
            if (w == (start >> 5) || w == last_word) {
#if defined(__CUDA_ARCH__)
                atomicOr(&out[w], v);
#else
                out[w] |= v;
#endif
            } else out[w] = v;
            acc >>= 32; nacc = nacc > 32 ? nacc - 32 : 0; pos += 32;
        }
    }
    W::sync();
}

// Lizard_writeStream: returns 1 (Huffman'd), 0 (raw) or -1 (does not fit)
template <class W> LZ_HD int write_stream(bool use_huff, const u8* p, u32 n, u8* dst, long& op, long oend, EncHufWork* hw)
{
    const bool wr = W::lane() == 0;
    if (use_huff && n > 1024) {
        if (op + 6 > oend) return -1;
        const u32 seg = (n + 3) / 4;
        histogram4<W>(p, n, seg, hw->seg_count, hw->count);
        if (wr) huf_plan(hw->plan, hw->count, hw->seg_count, n, p[0], &hw->ws);
        W::sync();
        const int status = W::bcast(hw->plan.status);
        const u32 c = (u32)W::bcast((int)hw->plan.total);
        if (status != kHufPlanRaw && c > 0 && c + c / 8 + 512 < n) {
            if (oend - (op + 6) < (long)c) return -1;
            if (wr) { wr_le24(dst + op, n); wr_le24(dst + op + 3, c); }
            long o = op + 6;
            if (status == kHufPlanRle) { if (wr) dst[o] = hw->plan.rle_byte; }
            else {
                const u32 hs = (u32)W::bcast((int)hw->plan.header_size);
                lanes_copy<W>(dst + o, hw->ws.header, hs);
                o += hs;
                if (wr) { wr_le16(dst + o, hw->plan.seg_bytes[0]); wr_le16(dst + o + 2, hw->plan.seg_bytes[1]); wr_le16(dst + o + 4, hw->plan.seg_bytes[2]); }
                o += 6;
                for (u32 k = 0; k < 4; ++k) {
                    const u32 m = k < 3 ? seg : n - 3 * seg;
                    huf_pack_segment<W>(hw->pack, p + k * seg, m, hw->ws.codes);
                    const u32 sb = (u32)W::bcast((int)hw->plan.seg_bytes[k]);
                    lanes_copy_rows<W>(dst + o, (const u8*)hw->pack, sb);
                    W::sync();
                    o += sb;
                }
            }
            op += (long)c + 6;
            return 1;
        }
    }
    if (op + 3 + (long)n > oend) return -1;
    if (wr) wr_le24(dst + op, n);
    lanes_copy_rows<W>(dst + op + 3, p, n);
    op += 3 + (long)n;
    return 0;
}

// Lizard_writeBlock (lib/lizard_compress.c:186-250): 0 ok, 1 output error.  `in` is the inner block's first byte.
// All sizes are known from the sequence list, so the reference's decisions (raw block, stream does not fit,
// gain too small) are taken in its order before bytes move; only entropy-coded levels build flags/literals in
// scratch first.
template <class W> LZ_HD int write_block(const EncStreams& s, const u8* src, const u8* in, u32 in_size, u8* dst, long& op, long oend,
                                        bool huffman, bool lizv1, u8* scratch_lits, u8* scratch_flags, EncHufWork* hw)
{
    const bool wr = W::lane() == 0;
    const long start = op;
    const u32 sum = s.nf + s.nl + s.n16 + s.n24;
    bool raw = (s.nl < kWildCopy) || (sum + 5 * 3 + 1 > in_size);
    if (!raw) {
        long o = start + 1;
        if (o + 3 > oend) return 1;                                   // (empty) lengths stream
        const long o_len = o; o += 3;
        if (o + 3 + (long)s.n16 > oend) return 1;
        const long o16 = o; o += 3 + (long)s.n16;
        if (o + 3 + (long)s.n24 > oend) return 1;
        const long o24 = o; o += 3 + (long)s.n24;
        const bool entropy = huffman && (s.nf > 1024 || s.nl > 1024);
        if (!entropy) {
            if (o + 3 + (long)s.nf > oend) return 1;
            const long of = o; o += 3 + (long)s.nf;
            if (o + 3 + (long)s.nl > oend) return 1;
            const long ol = o; o += 3 + (long)s.nl;
            const u32 out = (u32)(o - start);
            if (out + out / 32 + 512 > in_size) raw = true;
            else {
                if (wr) {
                    dst[start] = 0;
                    wr_le24(dst + o_len, 0); wr_le24(dst + o16, s.n16); wr_le24(dst + o24, s.n24);
                    wr_le24(dst + of, s.nf); wr_le24(dst + ol, s.nl);
                }
                emit_streams<W>(s, src, lizv1, dst + ol + 3, dst + of + 3, dst + o16 + 3, dst + o24 + 3);
                op = o;
                return 0;
            }
        } else {
            if (wr) { wr_le24(dst + o_len, 0); wr_le24(dst + o16, s.n16); wr_le24(dst + o24, s.n24); }
            emit_streams<W>(s, src, lizv1, scratch_lits, scratch_flags, dst + o16 + 3, dst + o24 + 3);
            op = o;
            u32 hdr = 0;
            int r = write_stream<W>(huffman, scratch_flags, s.nf, dst, op, oend, hw); if (r < 0) return 1;  hdr += (u32)r * kFlagFlags;
            r = write_stream<W>(huffman, scratch_lits, s.nl, dst, op, oend, hw);       if (r < 0) return 1;  hdr += (u32)r * kFlagLiterals;
            if (wr) dst[start] = (u8)hdr;
            const u32 out = (u32)(op - start);
            if (out + out / 32 + 512 > in_size) raw = true;
            else return 0;
        }
    }
    if ((u32)(oend - start) < in_size + 4 || oend - start < 0) return 1;
    W::sync();      // abandoned stream bytes (written by other lanes) must not land after the raw copy
    if (wr) { dst[start] = (u8)kFlagRaw; wr_le24(dst + start + 1, in_size); }
    lanes_copy_rows<W>(dst + start + 4, in, in_size);
    op = start + 4 + (long)in_size;
    return 0;
}

struct EncWork {                 // per-warp global scratch
    SeqRec seq[kBlockSize / kMinMatch + 8];   // a sequence consumes >= 4 input bytes
    u16 chain[1u << 16];         // hashChain levels: chain table (contentLog 16)
    u8 lits[kBlockSizePad];      // flags / literals streams, only when an entropy stage follows
    u8 flags[kBlockSizePad];
    EncHufWork huf;
};

// ---- parser families -----------------------------------------------------------------------------------------
// The encoder is compiled once per family so that a level only carries the code (and the register allocation) of the
// parsers it can reach.  Fast: fastSmall / fast without an entropy stage (levels 10, 11); FastBig: fastBig without one
// (level 20); Generic: every level, parser and Huffman stage picked at run time (hashChain, priceFast, 30/31/40).
// The device launches the family's kernel instance; encode_unit() (host build, emulated warps) picks the same family
// at run time, so both run the same per-family code.
enum EncFamily : int { kEncFamFast = 0, kEncFamFastBig = 1, kEncFamGeneric = 2, kEncFamilies = 3 };
LZ_HD int enc_family(const LevelParams& lp)
{
    if (lp.huffman) return kEncFamGeneric;
    if (lp.parser == kParserFastSmall || lp.parser == kParserFast) return kEncFamFast;
    if (lp.parser == kParserFastBig) return kEncFamFastBig;
    return kEncFamGeneric;
}

// the fastSmall / fast / fastBig walk: window form on real and emulated warps, batch form on narrow lane policies
template <class W, class TT, bool kBig> LZ_HD void parse_fast_any(const ParseCtx<TT>& pc, u32 b0, u32 b1, EncStreams& s)
{
    if (W::kLanes >= 4) parse_fast_win<W, TT, kBig>(pc, b0, b1, s);
    else parse_fast_par<W, TT, kBig>(pc, b0, b1, s);
}

// Lizard_compress_extState with a clean table: returns compressed size or 0.  kFam fixes the parser (Fast, FastBig) and
// compiles the entropy stage out of the families that never run it.
template <class W, class TT, int kFam> LZ_HD int encode_unit_t(const u8* src, u32 src_size, u8* dst, u32 cap, int level,
                                                              const TT T, EncWork* work)
{
    const LevelParams lp = level_params(level);
    if (lp.parser == kParserUnsupported) return 0;
    if (src_size > kMaxInputSize) return 0;
    if (TT::kOneBlock && src_size > kBlockSize) return 0;
    T.template clear<W>(lp.hashLog);
    const bool wr = W::lane() == 0;
    long op = 0;
    const long oend = (long)cap;
    if (cap < 1) return 0;                          // the reference would write the level byte regardless
    if (wr) dst[0] = (u8)level;
    op = 1;
    ParseCtx<TT> pc = { src, T, lp.hashLog, lp.windowLog };
    ChainState cs = { work->chain, (1u << (lp.chainLog ? lp.chainLog : 16)) - 1, 0, lp.searchNum, lp.searchLength };
    const bool huffman = kFam == kEncFamGeneric && lp.huffman != 0;
    const bool lizv1 = kFam == kEncFamFastBig || (kFam == kEncFamGeneric && lp.lizv1 != 0);
    u32 pos = 0;
    while (pos < src_size) {
        const u32 part = src_size - pos < kBlockSize ? src_size - pos : kBlockSize;
        EncStreams s;
        s.rec = work->seq; s.nseq = 0;
        s.nl = s.nf = s.n16 = s.n24 = 0; s.tail_anchor = pos; s.tail_len = 0;
        if (kFam == kEncFamFast) parse_fast_any<W, TT, false>(pc, pos, pos + part, s);
        else if (kFam == kEncFamFastBig) parse_fast_any<W, TT, true>(pc, pos, pos + part, s);
        else if (lp.parser == kParserHashChain) parse_hash_chain<W, TT>(pc, pos, pos + part, s, cs);
        else if (lp.parser == kParserPriceFast) parse_price_fast_par<W, TT>(pc, pos, pos + part, s, lp.minMatchLongOff);
        else if (lp.parser == kParserFastBig) parse_fast_any<W, TT, true>(pc, pos, pos + part, s);
        else parse_fast_any<W, TT, false>(pc, pos, pos + part, s);
        W::sync();
        if (write_block<W>(s, src, src + pos, part, dst, op, oend, huffman, lizv1,
                           work->lits, work->flags, &work->huf)) return 0;
        W::sync();
        if (TT::kOneBlock) break;   // a packed table serves one inner block: the loop state is dead while it is written
        pos += part;
    }
    return (int)op;
}
// one family; the packed form only holds positions of a single inner block
template <class W, int kFam> LZ_HD int encode_unit_fam(const u8* src, u32 src_size, u8* dst, u32 cap, int level,
                                                      const HashTable& T, EncWork* work)
{
    if (T.t32) return encode_unit_t<W, PlainTable, kFam>(src, src_size, dst, cap, level, PlainTable(T), work);
    return encode_unit_t<W, PackedTable, kFam>(src, src_size, dst, cap, level, PackedTable(T), work);
}
// the level's family picked at run time
template <class W> LZ_HD int encode_unit(const u8* src, u32 src_size, u8* dst, u32 cap, int level,
                                        const HashTable& T, EncWork* work)
{
    switch (enc_family(level_params(level))) {
    case kEncFamFast:    return encode_unit_fam<W, kEncFamFast>(src, src_size, dst, cap, level, T, work);
    case kEncFamFastBig: return encode_unit_fam<W, kEncFamFastBig>(src, src_size, dst, cap, level, T, work);
    default:             return encode_unit_fam<W, kEncFamGeneric>(src, src_size, dst, cap, level, T, work);
    }
}

// ---- compression against a loaded dictionary (hashChain and priceFast levels) ------------------------------------------------------
// Lizard_loadDict's table (lizard_compress.c:426-437): Lizard_Insert over dictionary positions [0, upto) into a zero table and
// the dictionary's chain (indexed by position & 0xFFFF; entries of positions the replay did not reach are never read: the
// table and every chain delta only lead to inserted positions, or out of the window).
template <class W> LZ_HD void dict_load(const u8* dict, u32 upto, const LevelParams& lp, u32* table, u16* chain)
{
    HashTable d; d.t32 = table; d.lo = nullptr; d.hi = nullptr; d.tag = nullptr; d.tagged = 0;
    const PlainTable T(d);
    T.template clear<W>(lp.hashLog);
    ChainState cs = { chain, 0xFFFFu, 0, 0, lp.searchLength };
    hc_insert<W, PlainTable>(dict, T, lp.hashLog, (1u << lp.windowLog) - 1, cs, upto);
    W::sync();
}
// The parsers that search a loaded dictionary through the table Lizard_Insert fills (Lizard_hashPtr with the level's
// searchLength): hashChain (13-17, 34-38) and priceFast (21, 22, 41, 42).
LZ_HD bool dict_parser(const LevelParams& lp) { return lp.parser == kParserHashChain || lp.parser == kParserPriceFast; }
// Lizard_compress_continue on a stream that Lizard_loadDict prepared (lizard_compress.c:550-580) at a dict_parser() level: returns
// the compressed size or 0.  src is the parse's base (position 0 = the dictionary's first byte; the unit is at src + T.dend),
// so for an external dictionary it is virtual and only positions >= T.dend are read through it.  One window runs across the
// dictionary and every inner block of the unit.
template <class W> LZ_HD int encode_unit_dict(const u8* src, u32 src_size, u8* dst, u32 cap, int level, const DictTable T,
                                             EncWork* work)
{
    const LevelParams lp = level_params(level);
    if (!dict_parser(lp)) return 0;
    if (src_size > kMaxInputSize) return 0;
    T.template clear<W>(lp.hashLog);
    const bool wr = W::lane() == 0;
    if (cap < 1) return 0;
    if (wr) dst[0] = (u8)level;
    long op = 1;
    const long oend = (long)cap;
    ParseCtx<DictTable> pc = { src, T, lp.hashLog, lp.windowLog };
    ChainState cs = { work->chain, (1u << lp.chainLog) - 1, T.own0, lp.searchNum, lp.searchLength };
    for (u32 pos = 0; pos < src_size;) {
        const u32 part = src_size - pos < kBlockSize ? src_size - pos : kBlockSize;
        const u32 b0 = T.dend + pos;
        EncStreams s;
        s.rec = work->seq; s.nseq = 0;
        s.nl = s.nf = s.n16 = s.n24 = 0; s.tail_anchor = b0; s.tail_len = 0;
        if (lp.parser == kParserHashChain) parse_hash_chain<W, DictTable>(pc, b0, b0 + part, s, cs);
        else parse_price_fast_par<W, DictTable>(pc, b0, b0 + part, s, lp.minMatchLongOff);
        W::sync();
        if (write_block<W>(s, src, src + b0, part, dst, op, oend, lp.huffman != 0, lp.lizv1 != 0,
                           work->lits, work->flags, &work->huf)) return 0;
        W::sync();
        pos += part;
    }
    return (int)op;
}
// The parse's view of one unit and its dictionary (dict_size already trimmed to the last kDictSize bytes): the layout, the
// first position the unit inserts, and ctx->lowLimit after the overlap check of Lizard_compress_continue (:568-577).
LZ_HD DictTable dict_view(const u8* unit, u32 unit_size, const u8* dict, u32 dict_size)
{
    DictTable T;
    T.ov = nullptr; T.sh = nullptr; T.dchain = nullptr;
    T.dsrc = dict; T.dend = dict_size;
    T.ext = dict + dict_size != unit;
    T.own0 = T.ext ? dict_size : (dict_size >= 8 ? dict_size - 7 : 0u);
    u32 low = 0;
    if (T.ext && unit + unit_size > dict && unit < dict + dict_size) {
        const u8* e = unit + unit_size < dict + dict_size ? unit + unit_size : dict + dict_size;
        low = (u32)(e - dict);
        if (dict_size - low < 4) low = dict_size;
    }
    T.low = low + kDictSize;
    return T;
}

}  // namespace lzb
