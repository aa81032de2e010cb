// encode_lp.cuh -- the lowestPrice parser (levels 23-25, Huffman twins 43-45), written once for "a warp" like the parsers
// of encode_core.cuh: uniform control flow, lane-parallel inserts, match measurement and price scan.  With W = HostLanes the
// same code builds with g++ and is pinned byte-for-byte against the reference (-DLIZARD_RESET_MEM) by the CPU suite.
//
// Reference functions restated here:
//   lib/lizard_parser_lowestprice.h:4-26     Lizard_more_profitable / Lizard_better_price
//   lib/lizard_parser_lowestprice.h:29-122   Lizard_FindMatchLowestPrice
//   lib/lizard_parser_lowestprice.h:125-251  Lizard_GetWiderMatch
//   lib/lizard_parser_lowestprice.h:256-375  Lizard_compress_lowestPrice
//   lib/lizard_compress_liz.h:186-301        Lizard_get_price_LIZv1 (the lowestPrice branches: no frequency statistics)
//   lib/lizard_parser_hashchain.h:13-41      Lizard_Insert
//   lib/lizard_common.h:251-253, 274-276     the level rows
#pragma once
#include "encode_core.cuh"

namespace lzb {

// ---- levels --------------------------------------------------------------------------------------------------------
// windowLog 22, contentLog 22, minMatchLongOff 16 and sufficientLength 64 at all six levels; hashLog 18 at 23/43 and 23 at
// the others; searchNum 1 / 2 / 8; searchLength 5 / 5 / 4.
struct LpParams { u32 hashLog, searchNum, searchLength; bool huffman; };
enum : u32 { kLpWindowLog = 22, kLpContentLog = 22, kLpSufficient = 64, kLpMaxHashLog = 23, kLpMaxPrice = 1u << 28 };
LZ_HD bool lp_level(int level) { return (level >= 23 && level <= 25) || (level >= 43 && level <= 45); }
LZ_HD LpParams lp_params(int level)
{
    const int b = level >= 40 ? level - 20 : level;
    LpParams p;
    p.hashLog = b == 23 ? 18u : 23u;
    p.searchNum = b == 23 ? 1u : (b == 24 ? 2u : 8u);
    p.searchLength = b == 25 ? 4u : 5u;
    p.huffman = level >= 40;
    return p;
}

// ---- Lizard_get_price_LIZv1 for parserType == lowestPrice --------------------------------------------------------------
// The literal length arrives as the reference's size_t: Lizard_more_profitable passes differences that wrap, so every sum
// here is 64-bit unsigned with the same wrap.  Lizard_highbit32(0) (a repeat offset) is 31 - clz(0): the reference's
// compiler emits a bit scan for it, which gives no offset surcharge either way; the surcharge starts at bit 16 / 20.
LZ_HD u64 lp_len_price(u64 len) { return len >= (1u << 16) ? 32u : (len >= 254 ? 24u : 8u); }
LZ_HD u64 lp_price(u64 lit, u32 off, u64 ml, bool huf)
{
    u64 price = 8 * lit;
    if (lit > 0 || off < kMax16BitOffset) {
        if (lit >= 7) price += lp_len_price(lit - 7);
        if (off >= kMax16BitOffset) price += 8;
    }
    if (off >= kMax16BitOffset) {
        if (ml < kMmLongOff) return kLpMaxPrice;
        if (ml - kMmLongOff >= kLastLongOff) price += lp_len_price(ml - kMmLongOff - kLastLongOff);
        price += 24;
    } else {
        if (off != 0) {
            if (off < kMinOffset || ml < kMinMatch) return kLpMaxPrice;
            price += 16;
        }
        if (ml >= 15) price += lp_len_price(ml - 15);
    }
    if (off > 0 || ml > 0) {
        const u32 load = off ? highbit32(off) : 0u;
        if (huf) price += (load >= 20 ? (u64)(load - 19) * 4 : 0) + 4 + (ml == 1);
        else     price += (load >= 16 ? (u64)(load - 15) * 4 : 0) + 6 + (ml == 1);
        price += 8;
    }
    return price;
}
// Lizard_better_price (:20-26): offsets equal to last_off (compared as int) price as repeat codes
LZ_HD bool lp_better_price(u32 best_off, u64 best_common, u32 off, u64 common, u32 last_off, bool huf)
{
    if (off == last_off) off = 0;
    if (best_off == last_off) best_off = 0;
    return lp_price(0, off, common, huf) < lp_price(common - best_common, best_off, best_common, huf);
}
// Lizard_more_profitable (:4-17); `literals` is ref0 - ref as a size_t, often "negative"
LZ_HD bool lp_more_profitable(u32 best_off, u64 best_common, u32 off, u64 common, u64 literals, u32 last_off, bool huf)
{
    u64 sum;
    if (literals > 0) sum = common + literals > best_common ? common + literals : best_common;
    else sum = common > best_common - literals ? common : best_common - literals;
    if (off == last_off) off = 0;
    if (best_off == last_off) best_off = 0;
    return lp_price(sum - common, off, common, huf) <= lp_price(sum - best_common, best_off, best_common, huf);
}

// ---- tables --------------------------------------------------------------------------------------------------------
// The reference starts every call with a zero hash table of 2^hashLog u32 entries (absolute index = position + 2^24) and a
// chain of 2^22 u32 deltas.  Two exact forms stand in for it:
//  * LpMap, units of one inner block: an open-addressed map of (bucket, position) pairs in 2^18 u64 slots.  A unit inserts
//    at most 2^17 positions, so the load stays at or below 1/2, and linear probing without deletions is exact.  A slot
//    carries the unit's epoch in its top 23 bits: a slot of another epoch is empty, so a new unit starts on an empty map
//    without clearing it (the owner clears the map once, before its first unit, and when the epoch wraps).
//    Layout: epoch (63..41) | bucket (40..18) | position + 1 (17..0).  The home slot is the bucket's top 18 bits (the
//    bucket is itself a hash): at hashLog 18 that is the bucket, and no probe sequence is longer than one slot.
//  * LpPlain, units of several inner blocks: the reference's table in full.  It must be zero when the unit starts; the
//    unit leaves it zero by re-walking the positions it inserted (lp_plain_unclear), so clearing costs what inserting did.
// The chain needs no clearing in either form: a walk starts at a bucket entry, i.e. a position inserted in this unit, and
// follows deltas written when that position was inserted; a delta never points below the window (empty buckets give a
// delta clamped to maxDistance, which ends the walk at the lowLimit test).  Positions are chain[pos & mask]: the bias 2^24
// is a multiple of 2^22, so `index & contentMask` is the position modulo 2^22, and a unit of one inner block needs 2^17.
enum : u32 { kLpMapLog = 18, kLpEpochMax = (1u << 23) - 1 };
#if defined(LZB_LP_STATS) && !defined(__CUDA_ARCH__)
// host shim only: every slot a lookup or insert visits past its home slot (tests prove that hostile input builds long
// probe runs and runs that wrap past the last slot)
enum { kLpProbeLongest, kLpProbes, kLpProbeWraps, kLpProbeStats };
extern unsigned long long g_lp_probe[kLpProbeStats];
inline void lp_probe_count(u32 home, u32 i)
{
    if (i == home) return;
    const unsigned long long run = (i - home) & ((1u << kLpMapLog) - 1);
    g_lp_probe[kLpProbes]++;
    if (run > g_lp_probe[kLpProbeLongest]) g_lp_probe[kLpProbeLongest] = run;
    if (i == 0) g_lp_probe[kLpProbeWraps]++;
}
#define LZB_LP_PROBE(home, i) lp_probe_count(home, i)
#else
#define LZB_LP_PROBE(home, i) do { } while (0)
#endif
struct LpMap {
    u64* slot; u64 tag; u32 shift;
    LZ_HDM LpMap(u64* s, u32 epoch, u32 hash_log) : slot(s), tag((u64)epoch << 41), shift(hash_log - kLpMapLog) {}
    LZ_HDM u32 get(u32 h) const
    {
        for (u32 i = h >> shift;; i = (i + 1) & ((1u << kLpMapLog) - 1)) {
            LZB_LP_PROBE(h >> shift, i);
            const u64 e = slot[i];
            if ((e & ~((1ull << 41) - 1)) != tag) return 0;
            if ((u32)(e >> 18 & 0x7FFFFFu) == h) return (u32)(e & 0x3FFFFu) - 1 + kDictSize;
        }
    }
    LZ_HDM void set(u32 h, u32 abs_index) const
    {
        const u64 v = tag | (u64)h << 18 | (u64)(abs_index - kDictSize + 1);
        for (u32 i = h >> shift;; i = (i + 1) & ((1u << kLpMapLog) - 1)) {
            LZB_LP_PROBE(h >> shift, i);
            const u64 e = slot[i];
            if ((e & ~((1ull << 41) - 1)) != tag) {            // empty: claim it (lanes of other buckets may race for it)
#if defined(__CUDA_ARCH__)
                const u64 was = atomicCAS((unsigned long long*)&slot[i], (unsigned long long)e, (unsigned long long)v);
                if (was == e) return;
                if ((u32)(was >> 18 & 0x7FFFFFu) == h && (was & ~((1ull << 41) - 1)) == tag) { slot[i] = v; return; }
                continue;                                       // taken by another bucket: go on probing
#else
                slot[i] = v; return;
#endif
            }
            if ((u32)(e >> 18 & 0x7FFFFFu) == h) { slot[i] = v; return; }
        }
    }
};
struct LpPlain {
    u32* t32;
    LZ_HDM u32 get(u32 h) const { return t32[h]; }
    LZ_HDM void set(u32 h, u32 abs_index) const { t32[h] = abs_index; }
};

struct LpChain {
    u32* chain;
    u32  mask;           // 2^17 - 1 (LpMap units) or 2^22 - 1
    u32  next_insert;    // ctx->nextToUpdate
};

// Lizard_Insert: positions [next_insert, upto), 32 per step; same-bucket lanes replayed in order under the reference's
// "replace unless within 8" rule.  Like the reference it sets next_insert = upto even when upto is lower (after a backward
// extension), so those positions are inserted again later.
template <class W, class TT> LZ_HD void lp_insert(const u8* src, const TT& T, u32 hl, u32 mls, LpChain& cs, u32 upto)
{
    const u32 lane = W::lane(), NL = W::lanes(), bias = kDictSize, max_dist = (1u << kLpWindowLog) - 1;
    for (u32 base = cs.next_insert; base < upto; base += NL) {
        const u32 P = base + lane;
        const bool valid = P < upto;
        const u32 idx = P + bias;
        u32 h = 0x80000000u | lane;
        if (valid) h = hc_hash(src + P, hl, mls);
        const u32 peers = W::match_any(h);
        u32 below = peers & ((1u << lane) - 1);
        u32 seen = valid ? T.get(h) : 0;
        while (below) {
            const u32 bl = ctz32(below); below &= below - 1;
            const u32 pb = base + bl + bias;
            if (seen >= pb || pb >= seen + kMinOffset) seen = pb;
        }
        if (valid) {
            const u32 dist = idx - seen;
            cs.chain[P & cs.mask] = dist > max_dist ? max_dist : dist;
        }
        const u32 newval = (seen >= idx || idx >= seen + kMinOffset) ? idx : seen;
        W::sync();
        if (valid && highbit32(peers) == lane) T.set(h, newval);
        W::sync();
    }
    cs.next_insert = upto;
}
// leave an LpPlain table zero again: every bucket the unit wrote is the bucket of a position below `upto`
template <class W> LZ_HD void lp_plain_unclear(const u8* src, const LpPlain& T, u32 hl, u32 mls, u32 upto)
{
    W::sync();
    for (u32 p = W::lane(); p < upto; p += W::lanes()) T.t32[hc_hash(src + p, hl, mls)] = 0;
    W::sync();
}

#if defined(LZB_LP_STATS)
// host shim only: how often the rare paths run (tests prove they are reached)
enum { kLpShortRep, kLpFarOffset, kLpMoreProfitableYes, kLpMoreProfitableNo, kLpScanElse, kLpSequences, kLpStats };
extern unsigned long long g_lp_stats[kLpStats];
#define LZB_LP_COUNT(k) do { if (W::lane() == 0) g_lp_stats[k]++; } while (0)
#else
#define LZB_LP_COUNT(k) do { } while (0)
#endif

// ---- the parser -------------------------------------------------------------------------------------------------------
template <class TT> struct LpCtx {
    const u8* src; TT T; LpChain* cs; u32 hl, mls, search_num; bool huf;
};

// Lizard_FindMatchLowestPrice (:29-122): the repeat offset first (counted from ip itself, taken at 2 bytes or more), then at
// most searchNum chain links.  Returns the length, 0 = none.
template <class W, class TT> LZ_HD u32 lp_find(const LpCtx<TT>& c, u32 ip, const u8* iLimit, u32 last_off, u32* ref)
{
    const u8* const src = c.src;
    const u32 bias = kDictSize, max_dist = (1u << kLpWindowLog) - 1, cur = ip + bias;
    const u32 low = (bias + max_dist >= cur) ? bias : cur - max_dist;
    u32 m = c.T.get(hc_hash(src + ip, c.hl, c.mls));
    if (last_off >= kMinOffset && cur - last_off >= low) {
        const u32 mlt = count_match_par<W>(src + ip, src + ip - last_off, iLimit);
        if (mlt > 1) { *ref = ip - last_off; return mlt; }
    }
    u32 ml = 0, tries = c.search_num;
    const u32 v = ld32(src + ip);
    while (m < cur && m >= low && tries) {
        tries--;
        const u32 p = m - bias;
        if (ip - p >= kMinOffset && src[p + ml] == src[ip + ml] && ld32(src + p) == v) {
            const u32 mlt = count_match_par<W>(src + ip + kMinMatch, src + p + kMinMatch, iLimit) + kMinMatch;
            if ((mlt >= kMmLongOff || ip - p < kMax16BitOffset) &&
                (!ml || (mlt > ml && lp_better_price(ip - *ref, ml, ip - p, mlt, last_off, c.huf)))) { ml = mlt; *ref = p; }
        }
        m -= c.cs->chain[p & c.cs->mask];
    }
    return ml;
}

// Lizard_GetWiderMatch (:125-251) with longest = 0: candidates grow backwards down to `floor` (the anchor).  The table is
// the one the caller's insert left, filled only up to the match being improved, not up to ip.
template <class W, class TT> LZ_HD u32 lp_wider(const LpCtx<TT>& c, u32 ip, u32 floor, const u8* iLimit, u32 last_off,
                                                u32* ref, u32* start)
{
    const u8* const src = c.src;
    const u32 bias = kDictSize, max_dist = (1u << kLpWindowLog) - 1, cur = ip + bias;
    const u32 low = (bias + max_dist >= cur) ? bias : cur - max_dist;
    u32 m = c.T.get(hc_hash(src + ip, c.hl, c.mls));
    const u32 v = ld32(src + ip);
    u32 longest = 0;
    if (last_off >= kMinOffset && cur - last_off >= low) {
        const u32 p = ip - last_off;
        if (ld32(src + p) == v) {
            u32 mlt = count_match_par<W>(src + ip + kMinMatch, src + p + kMinMatch, iLimit) + kMinMatch;
            const u32 back = extend_back_par<W>(src, ip, p, floor);
            mlt += back;
            if (mlt > longest && (mlt >= kMmLongOff || last_off < kMax16BitOffset)) { *ref = p - back; *start = ip - back; longest = mlt; }
        }
    }
    u32 tries = c.search_num;
    while (m < cur && m >= low && tries) {
        tries--;
        const u32 p = m - bias;
        if (ip - p >= kMinOffset && ld32(src + p) == v) {
            u32 mlt = count_match_par<W>(src + ip + kMinMatch, src + p + kMinMatch, iLimit) + kMinMatch;
            const u32 back = extend_back_par<W>(src, ip, p, floor);
            mlt += back;
            if ((mlt >= kMmLongOff || ip - p < kMax16BitOffset) &&
                (!longest || (mlt > longest && lp_better_price(*start - *ref, longest, ip - p, mlt, last_off, c.huf)))) {
                longest = mlt; *start = ip - back; *ref = p - back;
            }
        }
        m -= c.cs->chain[p & c.cs->mask];
    }
    return longest;
}

// The price scan of :305-341: for pos = ip+ml down to start2, the cost of writing [ip, pos) as the first match and the rest
// of the second match from pos.  Lane k prices pos = ip + ml - k; the reference's loop runs downward with a strict <, so of
// equal prices the highest pos (lowest k) wins.  Its last step (common0 < MINMATCH) prices the second match whole and, if
// that is cheaper, moves best_pos there without updating best_price, then stops.  Returns the new ml = best_pos - ip.
template <class W> LZ_HD u32 lp_scan(u32 ip, u32 ml, u32 ref, u32 start2, u32 ml2, u32 ref2, u32 anchor, u32 last_off, bool huf)
{
    const u32 NL = W::lanes(), lane = W::lane();
    const int off0 = (int)(ip - ref), off1 = (int)(start2 - ref2);
    // positions with common0 >= MINMATCH and pos >= start2: k = 0 .. kn-1
    const u32 lo = start2 > ip + kMinMatch ? start2 : ip + kMinMatch;
    const u32 kn = ip + ml >= lo ? ip + ml - lo + 1 : 0;
    u32 best_price = kLpMaxPrice, best_k = 0xFFFFFFFFu;
    for (u32 k0 = 0; k0 < kn; k0 += NL) {
        const u32 k = k0 + lane;
        u32 price = 0xFFFFFFFFu;
        if (k < kn) {
            const u32 pos = ip + ml - k;
            const u32 common0 = pos - ip;
            u64 p = (u64)(long long)(int)lp_price(ip - anchor, off0 == (int)last_off ? 0u : (u32)off0, common0, huf);
            const int common1 = (int)(start2 + ml2 - pos);
            if (common1 >= (int)kMinMatch) p += lp_price(0, off1 == off0 ? 0u : (u32)off1, (u64)common1, huf);
            else p += lp_price((u64)(long long)common1, 0, 0, huf);
            price = (u32)p;                                     // < 2^30: literal runs of one inner block, two terms <= 2^28
        }
        u32 mn = price;                                         // minimum over the lanes
        for (u32 o = NL >> 1; o; o >>= 1) { const u32 t = W::shfl(mn, lane ^ o); mn = t < mn ? t : mn; }
        if (mn < best_price) { best_price = mn; best_k = k0 + ctz32(W::ballot(price == mn)); }
    }
    u32 best_pos = best_k == 0xFFFFFFFFu ? ip : ip + ml - best_k;
    const u32 pos_end = ip + (ml < kMinMatch - 1 ? ml : kMinMatch - 1);   // the first pos with common0 < MINMATCH
    if (pos_end >= start2) {
        const u64 p = lp_price(start2 - anchor, off1 == (int)last_off ? 0u : (u32)off1, ml2, huf);
        if (p < best_price) best_pos = pos_end;
        LZB_LP_COUNT(kLpScanElse);
    }
    return best_pos - ip;
}

// Lizard_compress_lowestPrice (:256-375) over the inner block [b0, b1)
template <class W, class TT> LZ_HD_COLD void parse_lowest_price(const LpCtx<TT>& c, u32 b0, u32 b1, EncStreams& st)
{
    const u8* const src = c.src;
    u32 anchor = b0, last_off = 0;
    if (b1 - b0 > kMfLimit) {
        const u32 mflimit = b1 - kMfLimit;
        const u8* const matchlimit = src + b1 - kLastLiterals;
        u32 ip = b0;
        while (ip < mflimit) {
            lp_insert<W, TT>(src, c.T, c.hl, c.mls, *c.cs, ip);
            u32 ref = 0;
            u32 ml = lp_find<W, TT>(c, ip, matchlimit, last_off, &ref);
            if (!ml) { ip++; continue; }
            {   const u32 back = extend_back_par<W>(src, ip, ref, anchor); ml += back; ip -= back; ref -= back; }
            const u32 start0 = ip, ref0 = ref, ml0 = ml;
            for (;;) {                                                          // _Search
                if (ip + ml >= mflimit || ml >= kLpSufficient) break;
                lp_insert<W, TT>(src, c.T, c.hl, c.mls, *c.cs, ip);
                u32 ref2 = 0, start2 = 0;
                const u32 ml2 = lp_wider<W, TT>(c, ip + ml - 2, anchor, matchlimit, last_off, &ref2, &start2);
                if (!ml2) break;
                ml = lp_scan<W>(ip, ml, ref, start2, ml2, ref2, anchor, last_off, c.huf);
                if (ml < kMinMatch || (ml < kMmLongOff && ip - ref >= kMax16BitOffset)) { ip = start2; ref = ref2; ml = ml2; continue; }
                break;
            }
            if (start0 < ip) {                                                  // _Encode
                const bool back = lp_more_profitable(ip - ref, ml, start0 - ref0, ml0, (u64)(long long)((long long)ref0 - (long long)ref),
                                                     last_off, c.huf);
                if (back) { ip = start0; ref = ref0; ml = ml0; LZB_LP_COUNT(kLpMoreProfitableYes); }
                else LZB_LP_COUNT(kLpMoreProfitableNo);
            }
            const u32 off = ip - ref == last_off ? 0u : ip - ref;
            if (off == 0 && ml < kMinMatch) LZB_LP_COUNT(kLpShortRep);
            if (off >= kMax16BitOffset) LZB_LP_COUNT(kLpFarOffset);
            LZB_LP_COUNT(kLpSequences);
            emit_lizv1<W>(st, src, anchor, ip, ml, off, last_off);
            ip += ml;
            anchor = ip;
        }
    }
    emit_last_literals<W>(st, src, anchor, b1);
}

// ---- one unit ------------------------------------------------------------------------------------------------------
struct LpWork {                  // per-warp scratch of the lowestPrice encoder
    SeqRec seq[kBlockSize / 2 + 8];     // a sequence consumes >= 2 input bytes (repeat matches of 2-3 bytes)
    u32 chain[kBlockSize];              // LpMap units: positions below 2^17
    u8 lits[kBlockSizePad];
    u8 flags[kBlockSizePad];
    EncHufWork huf;
    u64 map[1u << kLpMapLog];
};
// one big slot: the reference's full tables for units of several inner blocks
constexpr size_t kLpBigTableBytes = (size_t)4 << kLpMaxHashLog, kLpBigChainBytes = (size_t)4 << kLpContentLog;
constexpr size_t kLpBigSlotBytes = kLpBigTableBytes + kLpBigChainBytes;

// Lizard_compress_extState at levels 23-25 / 43-45 with a clean state: returns the compressed size or 0.  Units of one
// inner block run on work->map under `epoch` (1 .. kLpEpochMax); larger ones need `big` (a zero big slot, left zero).
template <class W, class TT> LZ_HD int encode_unit_lp_t(const u8* src, u32 src_size, u8* dst, u32 cap, int level, const TT& T,
                                                        LpChain cs, LpWork* work)
{
    const LpParams lp = lp_params(level);
    const bool wr = W::lane() == 0;
    if (cap < 1) return 0;
    if (wr) dst[0] = (u8)level;
    long op = 1;
    const LpCtx<TT> c = { src, T, &cs, lp.hashLog, lp.searchLength, lp.searchNum, lp.huffman };
    int r = (int)op;
    for (u32 pos = 0; pos < src_size;) {
        const u32 part = src_size - pos < kBlockSize ? src_size - pos : kBlockSize;
        EncStreams s;
        s.rec = work->seq; s.nseq = 0;
        s.nl = s.nf = s.n16 = s.n24 = 0; s.tail_anchor = pos; s.tail_len = 0;
        parse_lowest_price<W, TT>(c, pos, pos + part, s);
        W::sync();
        if (write_block<W>(s, src, src + pos, part, dst, op, (long)cap, lp.huffman, true, work->lits, work->flags, &work->huf)) { r = 0; break; }
        W::sync();
        pos += part;
        r = (int)op;
    }
    return r;
}
template <class W> LZ_HD int encode_unit_lp(const u8* src, u32 src_size, u8* dst, u32 cap, int level, LpWork* work, u32 epoch, u8* big)
{
    if (!lp_level(level) || src_size > kMaxInputSize) return 0;
    const LpParams lp = lp_params(level);
    if (src_size <= kBlockSize) {
        const LpChain cs = { work->chain, kBlockSize - 1, 0 };
        return encode_unit_lp_t<W, LpMap>(src, src_size, dst, cap, level, LpMap(work->map, epoch, lp.hashLog), cs, work);
    }
    const LpPlain T = { reinterpret_cast<u32*>(big) };
    const LpChain cs = { reinterpret_cast<u32*>(big + kLpBigTableBytes), (1u << kLpContentLog) - 1, 0 };
    const int r = encode_unit_lp_t<W, LpPlain>(src, src_size, dst, cap, level, T, cs, work);
    // every inserted position lies below the last block's mflimit, src_size - 20
    lp_plain_unclear<W>(src, T, lp.hashLog, lp.searchLength, src_size > kMfLimit ? src_size - kMfLimit : 0);
    return r;
}

}  // namespace lzb
