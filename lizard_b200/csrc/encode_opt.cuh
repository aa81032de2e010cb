// encode_opt.cuh -- the optimal parser with the binary-tree match finder and LZ4 codewords (levels 18, 19, Huffman twin 39),
// written once for "a warp" like encode_lp.cuh: the reference's serial dependencies stay serial (the tree walk, the DP over
// positions), the lanes share the match count at each tree node, the price fill of each match (32 lengths per step), the
// rescale of the token statistics and the emission of the streams.  With W = HostLanes the same code builds with g++ and is
// pinned byte-for-byte against the reference (-DLIZARD_RESET_MEM) by the CPU suite.
//
// Reference functions restated here:
//   lib/lizard_parser_optimal.h:181-320   Lizard_BinTree_GetAllMatches (Lizard_BinTree_Insert does nothing at MINMATCH 4)
//   lib/lizard_parser_optimal.h:323-678   SET_PRICE / Lizard_compress_optimalPrice, LZ4 codewords
//   lib/lizard_compress_lz4.h:3-71        Lizard_encodeSequence_LZ4 (the token statistics of huffType)
//   lib/lizard_compress_lz4.h:89-162      Lizard_get_price_LZ4
//   lib/lizard_compress_liz.h:1-40        Lizard_setLog2Prices / Lizard_rescaleFreqs
//   lib/lizard_common.h:245-246, 269      the level rows
#pragma once
#include "encode_lp.cuh"

namespace lzb {

// ---- levels --------------------------------------------------------------------------------------------------------
// windowLog 16, contentLog 17, searchLength 4 (hash4), minMatchLongOff 0, sufficientLength 1024, fullSearch 1 at all three;
// hashLog 18 / searchNum 16 at 18, hashLog 23 / searchNum 256 at 19 and 39.  At LZ4 codewords the reference's repeat-offset
// branches are dead (lizardOptimalMinOffset = 1 << 30, last_off never reaches it) and every price is Lizard_get_price_LZ4.
struct OptParams { u32 hashLog, searchNum; bool huffman; };
enum : u32 {
    kOptWindowLog = 16, kOptContentLog = 17, kOptSufficient = 1024, kOptNum = 1u << 12,   // LIZARD_OPT_NUM
    kOptMinOffset = 8,                                                                    // LIZARD_OPTIMAL_MIN_OFFSET
    kOptMaxSearch = 256, kOptMaxPrice = 1u << 28, kOptNoLink = 0xFFFFFFFFu
};
LZ_HD bool opt_level(int level) { return level == 18 || level == 19 || level == 39; }
LZ_HD OptParams opt_params(int level)
{
    OptParams p;
    p.hashLog = level == 18 ? 18u : 23u;
    p.searchNum = level == 18 ? 16u : 256u;
    p.huffman = level >= 30;
    return p;
}

// ---- token statistics (huffType) -------------------------------------------------------------------------------------
// Only the flag (token) frequencies move at LZ4 codewords: the literal statistics of Lizard_encodeSequence_LZ4 are compiled
// out in the reference, so litSum only tells the first inner block of a call (every frequency 2, sums 512) from the later
// ones (1 + (f >> 5)).  One warp's copy lives in shared memory on the device.
struct OptStats { u32 freq[256]; u32 sum, log2sum; };
template <class W> LZ_HD void opt_stats_rescale(OptStats* s, bool first)
{
    W::sync();
    u32 part = 0;
    for (u32 i = W::lane(); i < 256; i += W::lanes()) {
        const u32 f = first ? 2u : 1u + (s->freq[i] >> 5);
        s->freq[i] = f;
        part += f;
    }
    const u32 sum = W::sum(part);
    if (W::lane() == 0) { s->sum = sum; s->log2sum = highbit32(sum + 1); }
    W::sync();
}

// ---- Lizard_get_price_LZ4 ----------------------------------------------------------------------------------------------
LZ_HD u32 opt_len_price(u32 len) { return len >= (1u << 16) ? 32u : (len >= 254 ? 24u : 8u); }
LZ_HD u32 opt_price(const OptStats* s, bool huf, u32 lit, u32 off, u32 ml)
{
    u32 price = 8 * lit, token;
    if (lit >= 15) { token = 15; price += opt_len_price(lit - 15); }
    else token = lit;
    if (off) {
        price += 16;
        if (off < kOptMinOffset || ml < kMinMatch) return kOptMaxPrice;
        const u32 m = ml - kMinMatch;
        if (m >= 15) { token += 15u << 4; price += opt_len_price(m - 15); }
        else token += m << 4;
    }
    if (huf) price += (off > 0 || ml > 0 ? 2u : 0u) + s->log2sum - highbit32(s->freq[token] + 1);
    else price += 8;
    return price;
}

// ---- tables --------------------------------------------------------------------------------------------------------
// The hash table is encode_lp.cuh's: LpMap (2^18 epoch-tagged slots) for a unit of one inner block, LpPlain in a big slot
// for a larger one.  Lizard_BinTree_GetAllMatches stores HashTable[h] = current unconditionally.
// The binary tree is 2^17 u32 per warp (contentLog 17; node `idx` = position + 2^24 at tree[idx*2 & mask] (the "smaller"
// side) and tree[idx*2+1 & mask]) and is never cleared.  A walk starts at a hash entry, i.e. a position inserted in this unit,
// and follows links written when inserted positions were searched; it stops below the 64 KiB window.  An insert writes both
// nodes of its position before anything can read them, so every node a walk reads was written in this unit, and after its
// position: the 2^16 positions of a window own distinct node pairs, and a window position's pair is only overwritten by the
// insert 2^16 positions later.  DESIGN.md 3.1b.
#if defined(LZB_OPT_STATS) && !defined(__CUDA_ARCH__)
// host shim only: how often each reference behaviour runs (tests prove that each one is reached)
enum {
    kOptSearched,        // positions searched (and inserted into the tree)
    kOptNearEnd,         // positions within MINMATCH of iHighLimit: no search, no insert
    kOptSkipped,         // DP positions left unsearched by a sufficient match (goto encode)
    kOptLongMatch,       // goto encode on a match longer than sufficientLength
    kOptRescue,          // a node closer than 8 bytes: the smallest multiple of its distance >= 8 counted afresh
    kOptRescueTaken,     // ... and entered into the match list
    kOptWalkLong,        // walk stopped by a match longer than LIZARD_OPT_NUM
    kOptWalkEnd,         // walk stopped by a match reaching iHighLimit
    kOptWalkLeaf,        // walk stopped at a (U32)-1 link
    kOptWalkTries,       // walk stopped after searchNum nodes
    kOptGapFill,         // SET_PRICE filled positions between last_pos and the target with LIZARD_MAX_PRICE
    kOptCapped,          // match lengths capped at LIZARD_OPT_NUM - cur
    kOptLitTie,          // the literal step replaced an entry of equal price
    kOptMatchTie,        // a match left an entry of equal price in place
    kOptRescale,         // token statistics rescaled at a later inner block (huffType)
    kOptSequences,       // sequences emitted
    kOptStats
};
extern unsigned long long g_opt_stats[kOptStats];
#define LZB_OPT_COUNT(k, n) do { if (W::lane() == 0) g_opt_stats[k] += (unsigned long long)(n); } while (0)
#else
#define LZB_OPT_COUNT(k, n) do { } while (0)
#endif

struct OptNode  { u32 price; int off; u32 mlen, litlen; };     // off -1: a literal
struct OptMatch { u32 off, len; };

template <class TT> struct OptCtx {
    const u8* src; TT T; u32* tree; OptNode* opt; OptMatch* match; OptStats* stats; u32 hl, search_num; bool huf;
};

// Lizard_BinTree_GetAllMatches (:181-320) at position ip: inserts ip into the tree and lists the matches of strictly
// increasing length above max(best_mlen, MINMATCH - 1).  Returns their number (at most searchNum).
template <class W, class TT> LZ_HD u32 opt_matches(const OptCtx<TT>& c, u32 ip, u32 high, u32 best_mlen)
{
    const u8* const src = c.src;
    const bool wr = W::lane() == 0;
    if (ip + kMinMatch > high) { LZB_OPT_COUNT(kOptNearEnd, 1); return 0; }
    LZB_OPT_COUNT(kOptSearched, 1);
    const u32 bias = kDictSize, max_dist = (1u << kOptWindowLog) - 1, mask = (1u << kOptContentLog) - 1;
    const u32 cur = ip + bias;
    const u32 low = (bias + max_dist >= cur) ? bias : cur - max_dist;
    const u32 h = hc_hash(src + ip, c.hl, kMinMatch);
    u32 mi = c.T.get(h);
    W::sync();
    if (wr) c.T.set(h, cur);
    u32 p0 = (cur * 2 + 1) & mask, p1 = (cur * 2) & mask;
    u32 d0 = cur - mi, d1 = d0;
    if (best_mlen < kMinMatch - 1) best_mlen = kMinMatch - 1;
    u32 tries = c.search_num, n = 0;
    const u8* const limit = src + high;
    bool leaf = false, stop = false;
    while (mi < cur && mi >= low && tries) {
        tries--;
        const u32 mp = mi - bias;
        const u32 mlt = count_match_par<W>(src + ip, src + mp, limit);
        if (cur - mi >= kOptMinOffset) {
            if (mlt > best_mlen) {
                best_mlen = mlt;
                if (wr) { c.match[n].off = cur - mi; c.match[n].len = mlt; }
                n++;
                if (mlt > kOptNum) { LZB_OPT_COUNT(kOptWalkLong, 1); stop = true; break; }
                if (ip + mlt >= high) { LZB_OPT_COUNT(kOptWalkEnd, 1); stop = true; break; }
            }
        } else {                                          // :274-296, with the node's own mlt for the walk below
            u32 newoff = 0;
            do newoff += cur - mi; while (newoff < kOptMinOffset);
            const u32 newml = ip >= newoff ? count_match_par<W>(src + ip, src + ip - newoff, limit) : 0u;
            LZB_OPT_COUNT(kOptRescue, 1);
            if (newml > best_mlen) {
                LZB_OPT_COUNT(kOptRescueTaken, 1);
                best_mlen = newml;
                if (wr) { c.match[n].off = newoff; c.match[n].len = newml; }
                n++;
                if (newml > kOptNum) { LZB_OPT_COUNT(kOptWalkLong, 1); stop = true; break; }
                if (ip + newml >= high) { LZB_OPT_COUNT(kOptWalkEnd, 1); stop = true; break; }
            }
        }
        if (src[ip + mlt] < src[mp + mlt]) {
            if (wr) c.tree[p0] = d0;
            p0 = (mi * 2) & mask;
            const u32 d = c.tree[p0];
            if (d == kOptNoLink) { leaf = true; break; }
            d0 = d; d1 += d; mi -= d;
        } else {
            if (wr) c.tree[p1] = d1;
            p1 = (mi * 2 + 1) & mask;
            const u32 d = c.tree[p1];
            if (d == kOptNoLink) { leaf = true; break; }
            d1 = d; d0 += d; mi -= d;
        }
    }
    if (leaf) LZB_OPT_COUNT(kOptWalkLeaf, 1);
    else if (!stop && !tries) LZB_OPT_COUNT(kOptWalkTries, 1);
    if (wr) { c.tree[p0] = kOptNoLink; c.tree[p1] = kOptNoLink; }
    W::sync();
    return n;
}

// The prices of one match (offset `off`) at lengths [m0, m1] from position cur2: target t = cur2 + mlen, price = base +
// Lizard_get_price_LZ4(lit, off, mlen).  The targets are distinct, so lane k prices length m0 + k and replaces its entry when
// the target lies beyond last_pos or the price is strictly lower; SET_PRICE's serial gap fill becomes one store of
// LIZARD_MAX_PRICE per position between the old last_pos and the first target.  Returns the new last_pos.
template <class W> LZ_HD u32 opt_fill(const OptStats* st, bool huf, OptNode* opt, u32 last_pos, u32 cur2, u32 m0, u32 m1,
                                      u32 base, u32 lit, u32 off, u32 litlen)
{
    if (m0 > m1) return last_pos;
    const u32 lane = W::lane(), NL = W::lanes();
    for (u32 k0 = m0; k0 <= m1; k0 += NL) {
        const u32 mlen = k0 + lane;
        bool tie = false;
        if (mlen <= m1) {
            const u32 t = cur2 + mlen;
            const u32 price = base + opt_price(st, huf, lit, off, mlen);
            if (t > last_pos || price < opt[t].price) {
                OptNode e; e.price = price; e.off = (int)off; e.mlen = mlen; e.litlen = litlen;
                opt[t] = e;
            } else tie = price == opt[t].price;
        }
#if defined(LZB_OPT_STATS) && !defined(__CUDA_ARCH__)
        const u32 ties = W::ballot(tie);                    // every lane takes part in the vote
        LZB_OPT_COUNT(kOptMatchTie, __builtin_popcount(ties));
#endif
        (void)tie;
    }
    const u32 first = cur2 + m0;
    if (first > last_pos + 1) LZB_OPT_COUNT(kOptGapFill, 1);
    for (u32 t = last_pos + 1 + lane; t < first; t += NL) opt[t].price = kOptMaxPrice;
    W::sync();
    return cur2 + m1 > last_pos ? cur2 + m1 : last_pos;
}

// Lizard_compress_optimalPrice (:334-678) over the inner block [b0, b1), LZ4 codewords, fullSearch 1.  Only opt[0] is reset per
// window; every other entry the window reads was written in it (DESIGN.md 3.1b).
template <class W, class TT> LZ_HD_COLD void parse_optimal(const OptCtx<TT>& c, u32 b0, u32 b1, EncStreams& st)
{
    const u8* const src = c.src;
    const bool wr = W::lane() == 0;
    OptNode* const opt = c.opt;
    const OptMatch* const match = c.match;
    const OptStats* const stats = c.stats;
    const bool huf = c.huf;
    u32 anchor = b0;
    if (b1 - b0 > kMfLimit) {
        const u32 mflimit = b1 - kMfLimit;
        const u32 high = b1 - kLastLiterals;                    // matchlimit
        u32 ip = b0;
        while (ip < mflimit) {
            W::sync();                                          // the previous window's readers of opt[] are done
            if (wr) { OptNode z; z.price = 0; z.off = 0; z.mlen = 0; z.litlen = 0; opt[0] = z; }
            W::sync();
            u32 last_pos = 0, cur = 0, best_mlen = 0, best_off = 0;
            const u32 llen = ip - anchor;
            u32 n = opt_matches<W, TT>(c, ip, high, 0);
            if (!n) { ip++; continue; }
            if (match[n - 1].len > kOptSufficient) {
                LZB_OPT_COUNT(kOptLongMatch, 1);
                best_mlen = match[n - 1].len; best_off = match[n - 1].off; cur = 0; last_pos = 1;
                goto encode;
            }
            for (u32 i = 0; i < n; ++i) {
                const u32 m0 = i > 0 ? match[i - 1].len + 1 : kMinMatch;
                const u32 m1 = match[i].len < kOptNum ? match[i].len : kOptNum;
                if (match[i].len > kOptNum) LZB_OPT_COUNT(kOptCapped, 1);
                last_pos = opt_fill<W>(stats, huf, opt, last_pos, 0, m0, m1, 0, llen, match[i].off, 0);
            }
            if (last_pos < kMinMatch) { ip++; continue; }
            if (wr) { opt[0].mlen = 1; opt[0].off = -1; }
            W::sync();
            for (cur = 1; cur <= last_pos; cur++) {
                const u32 inr = ip + cur;
                u32 litlen, price;
                {
                    const OptNode prev = opt[cur - 1];
                    if (prev.off == -1) {
                        litlen = prev.litlen + 1;
                        if (cur != litlen) price = opt[cur - litlen].price + opt_price(stats, huf, litlen, 0, 0);
                        else price = opt_price(stats, huf, llen + litlen, 0, 0);
                    } else {
                        litlen = 1;
                        price = prev.price + opt_price(stats, huf, 1, 0, 0);
                    }
                }
                {
                    const u32 have = opt[cur].price;
                    if (price <= have) {
                        if (price == have) LZB_OPT_COUNT(kOptLitTie, 1);
                        W::sync();
                        if (wr) { OptNode e; e.price = price; e.off = -1; e.mlen = 1; e.litlen = litlen; opt[cur] = e; }
                        W::sync();
                    }
                }
                if (cur == last_pos) break;
                n = opt_matches<W, TT>(c, inr, high, 0);
                if (n > 0 && match[n - 1].len > kOptSufficient) {
                    LZB_OPT_COUNT(kOptLongMatch, 1);
                    LZB_OPT_COUNT(kOptSkipped, last_pos - cur - 1);
                    best_mlen = match[n - 1].len; best_off = match[n - 1].off; last_pos = cur + 1;
                    goto encode;
                }
                if (n) {
                    const OptNode here = opt[cur];
                    u32 base = here.price, lit = 0, litlen2 = 0;
                    if (here.off == -1) {
                        litlen2 = here.litlen;
                        if (cur != litlen2) { base = opt[cur - litlen2].price; lit = litlen2; }
                        else { base = 0; lit = llen + litlen2; }
                    }
                    for (u32 i = 0; i < n; ++i) {
                        const u32 m0 = i > 0 ? match[i - 1].len + 1 : kMinMatch;
                        const u32 m1 = cur + match[i].len < kOptNum ? match[i].len : kOptNum - cur;
                        if (cur + match[i].len >= kOptNum && m0 <= m1) LZB_OPT_COUNT(kOptCapped, 1);
                        last_pos = opt_fill<W>(stats, huf, opt, last_pos, cur, m0, m1, base, lit, match[i].off, litlen2);
                    }
                }
            }
            best_mlen = opt[last_pos].mlen;
            best_off = (u32)opt[last_pos].off;
            cur = last_pos - best_mlen;
        encode:
            // the path, reversed in place (:634-645): each node on it gets the step that leaves it
            W::sync();
            if (wr) {
                opt[0].mlen = 1;
                for (;;) {
                    const u32 mlen = opt[cur].mlen, offset = (u32)opt[cur].off;
                    opt[cur].mlen = best_mlen; opt[cur].off = (int)best_off;
                    best_mlen = mlen; best_off = offset;
                    if (mlen > cur) break;
                    cur -= mlen;
                }
            }
            W::sync();
            // emission (:652-667): literals only advance ip
            cur = 0;
            while (cur < last_pos) {
                const OptNode e = opt[cur];
                if (e.off == -1) { ip++; cur++; continue; }
                cur += e.mlen;
                emit_lz4<W>(st, src, anchor, ip, e.mlen, (u32)e.off);
                LZB_OPT_COUNT(kOptSequences, 1);
                if (huf) {                                          // Lizard_encodeSequence_LZ4 :58-64
                    const u32 lit = ip - anchor, m = e.mlen - kMinMatch;
                    const u32 token = (lit >= 15 ? 15u : lit) + ((m >= 15 ? 15u : m) << 4);
                    W::sync();
                    if (wr) { c.stats->freq[token]++; c.stats->sum++; c.stats->log2sum = highbit32(c.stats->sum + 1); }
                    W::sync();
                }
                ip += e.mlen;
                anchor = ip;
            }
        }
    }
    emit_last_literals<W>(st, src, anchor, b1);
}

// ---- one unit ------------------------------------------------------------------------------------------------------
struct OptWork {                 // per-warp scratch of the optimal encoder
    LpWork lp;                   // sequence list, streams, Huffman scratch and map of the lowestPrice encoder; lp.chain is the tree
    OptNode opt[kOptNum + 4];
    OptMatch match[kOptMaxSearch];
};
static_assert(sizeof(((LpWork*)0)->chain) >= (sizeof(u32) << kOptContentLog), "the tree is 2^17 u32");
static_assert(sizeof(((LpWork*)0)->seq) / sizeof(SeqRec) >= kBlockSize / kMinMatch + 8, "an LZ4 sequence covers >= 4 bytes");

template <class W, class TT> LZ_HD int encode_unit_opt_t(const u8* src, u32 src_size, u8* dst, u32 cap, int level, const TT& T,
                                                         OptWork* work, OptStats* stats)
{
    const OptParams op_ = opt_params(level);
    if (cap < 1) return 0;
    if (W::lane() == 0) dst[0] = (u8)level;
    long op = 1;
    const OptCtx<TT> c = { src, T, work->lp.chain, work->opt, work->match, stats, op_.hashLog, op_.searchNum, op_.huffman };
    int r = (int)op;
    for (u32 pos = 0; pos < src_size;) {
        const u32 part = src_size - pos < kBlockSize ? src_size - pos : kBlockSize;
        if (op_.huffman) {
            if (pos) LZB_OPT_COUNT(kOptRescale, 1);
            opt_stats_rescale<W>(stats, pos == 0);
        }
        EncStreams s;
        s.rec = work->lp.seq; s.nseq = 0;
        s.nl = s.nf = s.n16 = s.n24 = 0; s.tail_anchor = pos; s.tail_len = 0;
        parse_optimal<W, TT>(c, pos, pos + part, s);
        W::sync();
        if (write_block<W>(s, src, src + pos, part, dst, op, (long)cap, op_.huffman, false, work->lp.lits, work->lp.flags,
                           &work->lp.huf)) { r = 0; break; }
        W::sync();
        pos += part;
        r = (int)op;
    }
    return r;
}
// Lizard_compress_extState at levels 18 / 19 / 39 with a clean state: returns the compressed size or 0.  Units of one inner
// block run on work->lp.map under `epoch` (1 .. kLpEpochMax); larger ones need `big` (a zero big slot of the lowestPrice pool,
// left zero).  `stats`: the warp's token statistics (level 39; set up at the first inner block).
template <class W> LZ_HD int encode_unit_opt(const u8* src, u32 src_size, u8* dst, u32 cap, int level, OptWork* work, u32 epoch,
                                             u8* big, OptStats* stats)
{
    if (!opt_level(level) || src_size > kMaxInputSize) return 0;
    const OptParams p = opt_params(level);
    if (src_size <= kBlockSize)
        return encode_unit_opt_t<W, LpMap>(src, src_size, dst, cap, level, LpMap(work->lp.map, epoch, p.hashLog), work, stats);
    const LpPlain T = { reinterpret_cast<u32*>(big) };
    const int r = encode_unit_opt_t<W, LpPlain>(src, src_size, dst, cap, level, T, work, stats);
    // every inserted position p has p + MINMATCH <= its block's matchlimit <= src_size - LASTLITERALS
    lp_plain_unclear<W>(src, T, p.hashLog, kMinMatch, src_size > kLastLiterals + kMinMatch ? src_size - kLastLiterals - kMinMatch + 1 : 0);
    return r;
}

}  // namespace lzb
