// decode.cuh -- Lizard block decoder written against the lane policy W (lanes.cuh): one warp per
// independent compressed unit on the device, one lane (or 32 emulated lanes) in the CPU test build.
//
// A "unit" is exactly what one Lizard_decompress_safe() call receives: [level byte] followed by
// inner blocks of <= 128 KiB (reference: lib/lizard_decompress.c:115-264 Lizard_decompress_generic).
// Frame blocks of 128 KiB hold one inner block, so the frame layer hands us thousands of independent
// units per launch; one warp walks one unit, the grid is a persistent set of warps pulling unit
// indices from an atomic counter.
//
// Per inner block the warp
//   1. parses the 5 stream headers (all lanes redundantly; they are ~20 bytes),
//   2. expands Huffman'd streams into its private scratch (lane-parallel over the 4 bitstreams),
//   3. runs the token loop in BATCHES of W::lanes() tokens: lane i owns token i.  Everything a token needs
//      except its position in the literals stream is a function of the token byte; the position depends on
//      the earlier literal-length extension bytes, so those (about half of the tokens on datagen data) are
//      resolved in a short serial chain of broadcast loads, everything else (cursor positions, output
//      positions, bounds checks) is prefix sums and ballots.  Then the warp copies the batch's literal runs
//      and resolves its matches in order.  Any token that fails a check, or uses a multi-byte length
//      extension, sends the batch down the serial path, which follows the reference statement by statement
//      so that accept/reject and the returned error codes are identical
//      (lib/lizard_decompress_lz4.h:7-163, lib/lizard_decompress_liz.h:14-220).
#pragma once
#include "common.cuh"
#include "lanes.cuh"
#include "entropy_dec.cuh"
#include "huf_expand.cuh"

namespace lzb {

#define LZB_FULL 0xffffffffu

// Optional streaming hand-shake for the host-pipelined entry points: units become available as their input
// chunk lands (`ready` = number of leading units whose bytes are in HBM, published by a 4-byte copy queued
// behind each H2D chunk), and the last unit of every chunk raises a flag in mapped pinned memory so the host
// can start that chunk's D2H while later units are still being processed.  All null = everything is resident.
struct Progress {
    const volatile u32* ready;      // device: units [0, *ready) may be read
    u32*                done_count; // device: [n_chunks] finished units per chunk
    volatile u32*       host_done;  // mapped pinned: [n_chunks] set to 1 when a chunk is complete
    u32                 chunk_units;
    u32                 n_units;
    u32                 ramp_unit;  // 0, or the size of chunk 0 of a doubling ramp: chunks of ramp_unit << i units (i < ramp_chunks,
    u32                 ramp_chunks;//    ramp_unit << ramp_chunks == chunk_units) in front of the chunk_units-sized ones
};
// chunk of a unit, the chunk's first unit and its size (the same arithmetic as FrameChunks on the host, frame.inl)
LZ_HD u32 progress_chunk(const Progress& pg, u32 unit, u32* first, u32* cnt)
{
    u32 c, f, size;
    const u32 ramp_total = pg.ramp_unit ? pg.chunk_units - pg.ramp_unit : 0u;       // ramp_unit * (2^ramp_chunks - 1)
    if (unit < ramp_total) {
        c = highbit32(unit / pg.ramp_unit + 1u);
        f = pg.ramp_unit * ((1u << c) - 1u); size = pg.ramp_unit << c;
    } else {
        const u32 k = (unit - ramp_total) / pg.chunk_units;
        c = (pg.ramp_unit ? pg.ramp_chunks : 0u) + k; f = ramp_total + k * pg.chunk_units; size = pg.chunk_units;
    }
    *first = f; *cnt = pg.n_units - f < size ? pg.n_units - f : size;
    return c;
}

#if defined(__CUDACC__)
__device__ __forceinline__ void progress_wait(const Progress& pg, u32 unit, u32 lane)
{
    if (pg.ready) {
        if (lane == 0) { while (*pg.ready <= unit) __nanosleep(400); }
        __syncwarp();
        __threadfence();
    }
}
__device__ __forceinline__ void progress_done(const Progress& pg, u32 unit, u32 lane)
{
    if (pg.done_count && lane == 0) {
        __threadfence_system();                        // the unit's result may live in pinned host memory
        u32 first, cnt;
        const u32 c = progress_chunk(pg, unit, &first, &cnt);
        if (atomicAdd(&pg.done_count[c], 1u) == cnt - 1) { __threadfence_system(); pg.host_done[c] = 1u; }
    }
}
#endif

struct DecodeBatch {
    const u8*  src_base;    // compressed bytes of all units
    const u64* src_off;     // [n] byte offset of unit i in src_base
    const u32* src_len;     // [n] compressed size of unit i
    u8*        dst_base;    // output arena
    const u64* dst_off;     // [n] where unit i decodes to
    const u32* dst_cap;     // [n] capacity available to unit i (maxDecompressedSize)
    int*       result;      // [n] Lizard_decompress_safe return value
    u32        n_units;
    u8*        scratch;     // n_warps * kDecScratchPerWarp bytes (Huffman-expanded streams)
    u32*       counter;     // work queue head
    Progress   progress;
    const UnitPre* pre;     // [n] streams expanded by the Huffman pre-pass (huf_expand.cuh), or null
    const u8*  arena;       // the pre-pass's expansion arena
    const UnitSeq* seq;     // [n] blocks parsed by the token pre-pass, or null
    const PoolRun* recs;    // its sequence records
    const int* target;      // [n] targetOutputSize of a partial decode (lizard_decode_partial_units_kernel), null for a full one
    // decoding against dictionaries (lizard_decode_dict_units_kernel): unit i's dictionary is the dict_len[i] bytes at
    // dict_base + dict_off[i] (dict_len[i] == 0: none).  dict_reach null: the reach follows from dict_len and the prefix test
    // (dictionary end == the unit's output), as in Lizard_decompress_safe_usingDict; otherwise dict_reach[i] is the reach of
    // a dictionary that was staged shorter than the caller's (see DictWin)
    const u8*  dict_base;
    const u64* dict_off;
    const u32* dict_len;
    const u32* dict_reach;
};

// ---- decoding against a dictionary (Lizard_decompress_safe_usingDict / _continue, lib/lizard_decompress.c:322-360) ----
// A unit sees the `avail` bytes in front of `end` as the bytes in front of its own start: `end` is the dictionary's end
// (the unit's own output in the reference's prefix mode, where the dictionary lies in place in front of it).  A match may
// start up to `reach` bytes below the unit start before the reference's offset check (lowLimit = lowPrefix - dictSize)
// rejects it; kDictUnchecked = the reference's checkOffset is off.  No match starts more than 65535 (fastLZ4 codewords) or
// 2^24 - 1 (LIZv1) bytes below the unit start, so `avail` may be shorter than the caller's dictionary; `reach` may not.
struct DictWin { const u8* end; u32 avail; u32 reach; };
enum : u32 { kDictUnchecked = 0xffffffffu, kDictPrefixMax = (1u << 24) - 1 };
// the reach of a dictionary of `size` bytes, `prefix` = it ends where the output starts (lib/lizard_decompress.c:349-360 picks
// noDict with lowPrefix = dest - size, or withPrefix64k with lowPrefix = dest - 2^24 from size 2^24 - 1 on; usingExtDict
// checks offsets only below size 2^24)
LZ_HD u32 dict_reach(u32 size, bool prefix)
{
    if (prefix) return size >= kDictPrefixMax ? (1u << 24) : size;
    return size >= (1u << 24) ? kDictUnchecked : size;
}
// farthest any match of a unit at this level starts below the unit start
LZ_HD u32 dict_window(int level) { return level_is_lizv1(level) ? kDictPrefixMax : 65535u; }

#if defined(LZB_DICT_STATS) && !defined(__CUDA_ARCH__)
static unsigned long long g_dict_only = 0, g_dict_straddle = 0;      // matches read from the dictionary alone / across its end
#define LZB_COUNT_DICT(only, straddle) (g_dict_only += (only), g_dict_straddle += (straddle))
#else
#define LZB_COUNT_DICT(only, straddle)
#endif

enum : u32 { kDecStreamScratch = kBlockSize + 64, kDecBigTableBytes = 2u << kHufTableLogMax,
             kDecScratchPerWarp = 4 * kDecStreamScratch + kDecBigTableBytes };

typedef PoolRun SeqDesc;                          // 16-byte sequence descriptor (see run_batch_copies)

struct alignas(16) ChainRec { u32 ent, epre, vl, vm; };   // list entry, bytes of extension data before it, value | size << 24 of its two fields

struct DecWarpCore {               // per-warp shared memory every decoder generation needs
    u16* big_table;                // single-symbol table of the in-kernel Huffman expansion: 2^12 entries in the warp's
                                   // global scratch (the pre-pass expands the streams of real batches; keeping 4 KiB per
                                   // warp in shared memory for the rest would cost the token loops their L1)
    union {
        HufStatsScratch stats;                       // while a Huffman header is being read
        struct { u32 ent[32]; u32 epre[32]; } chain; // during the token loops: length-extension chain of a batch
        ChainRec chainw[32];                         // the same for the windowed chain (ext_chain_win)
    };
    u8  weights[256];
    u32 rank[kHufTableLogMax + 1];
    u32 pad[3];
};
struct DecWarpShared : DecWarpCore {   // first generation (decode_tokens_*): plus the batch's copy descriptors
    SeqDesc desc[64];              // literal-run and match descriptors of the current token batch
};

// ---- lane-cooperative byte movers --------------------------------------------------------------
template <class W> LZ_HD void lanes_fill(u8* dst, u8 v, u32 n)
{
    for (u32 i = W::lane(); i < n; i += W::lanes()) dst[i] = v;
}
// LZ77 match: dst[op+i] = dst[op-off+i] with byte-serial semantics.  An overlapping match is a
// periodic extension of the `off` bytes before op, so every source byte already exists.
template <class W> LZ_HD void lanes_match(u8* dst, long op, u32 off, u32 len)
{
    const u8* s = dst + op - off;
    u8* d = dst + op;
    if (off >= len) { for (u32 i = W::lane(); i < len; i += W::lanes()) d[i] = s[i]; }
    else if (off != 0) { for (u32 i = W::lane(); i < len; i += W::lanes()) d[i] = s[i % off]; }
    else { for (u32 i = W::lane(); i < len; i += W::lanes()) d[i] = 0; }     // offset 0 (no encoder emits it; the reference copies
                                                                              // whatever dst held): defined output, nothing stale leaks
}
// The same match of a unit decoded against a dictionary: a source below the unit start reads the dictionary, and a match
// that runs past the dictionary's end continues from the unit start with LZ77 overlap (lizard_decompress_lz4.h:99-121), the
// bytes [dict][unit] read as one window.
template <class W> LZ_HD void dict_match(u8* dst, long op, u32 off, u32 len, const DictWin& dw)
{
    if ((long)off <= op) { lanes_match<W>(dst, op, off, len); return; }
    const u32 below = (u32)((long)off - op);
    const u32 head = len < below ? len : below;
    for (u32 i = W::lane(); i < head; i += W::lanes()) dst[op + i] = dw.end[(long)i - (long)below];
    LZB_COUNT_DICT(W::lane() == 0 && len <= below ? 1 : 0, W::lane() == 0 && len > below ? 1 : 0);
    if (len > below) { W::sync(); lanes_match<W>(dst, (long)off, off, len - below); }
}

// ---- Huffman stream expansion -----------------------------------------------------------------
// single-symbol decode of one of the 4 segments by one lane; true when the bitstream ended exactly
LZ_HD u64 ld64_any(const u8* p)          // unaligned 8-byte little-endian load through aligned 8-byte words
{
#if defined(__CUDA_ARCH__)
    const size_t a = (size_t)p;
    const u64* q = reinterpret_cast<const u64*>(a & ~(size_t)7);
    const u32 sh = (u32)(a & 7) * 8;
    const u64 lo = q[0];
    if (sh == 0) return lo;
    return (lo >> sh) | (q[1] << (64 - sh));            // q[1] holds p[8 - (a&7)] .. p[7]: bytes of the same load
#else
    return rd_le64(p);
#endif
}
template <class T> LZ_HD u32 huf_step(BitReader& b, const T& tab)          // single-symbol step (HUF_decodeSymbolX2)
{
    const u32 e = tab.look((u32)((b.win << (b.used & 63)) >> 32));
    b.used += e >> 8;
    return e & 255;
}

// literals-stream prefetch of the token loops: every batch requests LINES 128-byte lines from DIST bytes behind the batch's
// first literal byte.  A batch consumes ~2.7 KB of the stream at level 10 and an SM's L1 is ~5 KB per resident warp, so the
// lines have to be requested just in time: distance 0 (the batch's own bytes, all 32 lines in flight at once before the
// extension chain starts walking them) beat 512 / 1024 / 2048 / 4096 and no prefetch at all, in that order.
// LZB_DEC_LIT_PF_NEXT: request the NEXT batch's lines before this batch's copy sweeps instead (A/B builds).
#if !defined(LZB_DEC_LIT_PF_DIST)
#define LZB_DEC_LIT_PF_DIST 0
#endif
#if !defined(LZB_DEC_LIT_PF_LINES)
#define LZB_DEC_LIT_PF_LINES 32
#endif
#if !defined(LZB_DEC_LIT_PF_NEXT)
#define LZB_DEC_LIT_PF_NEXT 0
#endif
#if !defined(LZB_DEC_LIT_PF_LOAD)
#define LZB_DEC_LIT_PF_LOAD 0
#endif
// expand kernel (A/B builds): level of the optional bitstream prefetch
#if !defined(LZB_HUF_PREFETCH_L2)
#define LZB_HUF_PREFETCH_ASM(p) asm volatile("prefetch.global.L1 [%0];" :: "l"(p))
#else
#define LZB_HUF_PREFETCH_ASM(p) asm volatile("prefetch.global.L2 [%0];" :: "l"(p))
#endif

// ---- pieces of the sixteen-symbol rounds (huf_lane_segment_t<true>) ----
#if !defined(LZB_SHIM_CHECK)
#define LZB_SHIM_CHECK(cond) ((void)0)          /* the CPU test build turns this into an abort */
#endif
#if defined(__CUDA_ARCH__)
enum : u32 { kHufRingStride = 32 };             // shared memory, word j of lane l at [j][l]: every access is conflict-free
#else
enum : u32 { kHufRingStride = 1 };
#endif
enum : u32 { kHufRingWords = 16 };              // 64 bytes per lane
struct HufVec { u32 x, y, z, w; };
LZ_HD HufVec huf_vec_zero() { HufVec v; v.x = v.y = v.z = v.w = 0; return v; }
// the aligned 16 bytes at `a`; bytes outside [lo, hi) read as zero, a vector wholly outside is not touched
LZ_HD HufVec huf_vec_load(const u8* a, const u8* lo, const u8* hi)
{
    HufVec v = huf_vec_zero();
    if (a + 16 <= lo || a >= hi) return v;
#if defined(__CUDA_ARCH__)
    const uint4 q = *reinterpret_cast<const uint4*>(a);      // an aligned vector with one valid byte lies inside the allocation
    v.x = q.x; v.y = q.y; v.z = q.z; v.w = q.w;
#else
    u32 wv[4] = {0, 0, 0, 0};
    for (u32 i = 0; i < 16; ++i) if (a + i >= lo && a + i < hi) wv[i >> 2] |= (u32)a[i] << (8 * (i & 3));
    v.x = wv[0]; v.y = wv[1]; v.z = wv[2]; v.w = wv[3];
#endif
    return v;
}
LZ_HD void huf_ring_put(u32* ring, u32 a, const HufVec& v)      // a = low address bits of the (16-byte aligned) vector
{
    const u32 j = (a >> 2) & (kHufRingWords - 4);
    ring[(j + 0) * kHufRingStride] = v.x; ring[(j + 1) * kHufRingStride] = v.y;
    ring[(j + 2) * kHufRingStride] = v.z; ring[(j + 3) * kHufRingStride] = v.w;
}
LZ_HD void huf_store16(u8* p, u32 a, u32 b, u32 c, u32 d)    // p is 16-byte aligned
{
#if defined(__CUDA_ARCH__)
    *reinterpret_cast<uint4*>(p) = make_uint4(a, b, c, d);
#else
    u32* q = reinterpret_cast<u32*>(p); q[0] = a; q[1] = b; q[2] = c; q[3] = d;
#endif
}
LZ_HD u32 fsh_r(u32 lo, u32 hi, u32 s)          // low word of (hi:lo) >> s, s < 32
{
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, s);
#else
    return s ? (lo >> s) | (hi << (32 - s)) : lo;
#endif
}
LZ_HD u32 fsh_l(u32 lo, u32 hi, u32 s)          // high word of (hi:lo) << s, s < 32
{
#if defined(__CUDA_ARCH__)
    return __funnelshift_l(lo, hi, s);
#else
    return s ? (hi << s) | (lo >> (32 - s)) : hi;
#endif
}

// one segment, one lane; true when the bitstream ended exactly
// kWide + ring: the sixteen-symbol rounds with the bitstream window in a per-lane ring (the pre-pass kernel; inside the
// token kernel's 64-register budget they spill and lose more than they gain)
template <bool kWide, class T> LZ_HD bool huf_lane_segment_t(u8* out, long count, const u8* src, u32 len, const T& tab, int* init_err,
                                                           u32* ring = nullptr)
{
    BitReader b;
    int e = bits_init(b, src, len);
    *init_err = e;
    if (e < 0) return false;
    long p = 0;
    // Bulk: same walk as the loop below (reload, then four symbols: HUF_decodeStreamX2, huf_decompress.c:155-176) with
    // the window fetched by aligned loads and the four bytes stored as one word.  It stops 16 bytes before the start
    // of the bitstream, where the reload rules change, and leaves a state the exact loop continues from.
    if (len >= 24) {
        while (p < count && ((size_t)(out + p) & 3) != 0 && b.ptr >= b.start + 16) {
            if (bits_reload(b) != kBitsUnfinished) break;
            out[p++] = (u8)huf_step(b, tab);
        }
        for (int phase = 0; phase < 2; ++phase) {        // 0: four-byte rounds up to a 16-byte boundary of the output, then the
                                                         //    sixteen-byte rounds; 1: four-byte rounds for what is left
        while (p + 4 <= count && b.ptr >= b.start + 16 && b.used <= 64 && ((size_t)(out + p) & 3) == 0 &&
               (phase == 1 || ((size_t)(out + p) & 15) != 0)) {
            b.ptr -= b.used >> 3;                          // bits_reload, "ptr >= start + 8" case
            b.used &= 7;
            b.win = ld64_any(b.ptr);
#if defined(__CUDA_ARCH__)
#if !defined(LZB_HUF_PREFETCH)
#define LZB_HUF_PREFETCH 0           /* with the ring's loads issued a round ahead an L1 / L2 prefetch changes nothing (0 / 128 / 384 / 1024) */
#endif
            if (LZB_HUF_PREFETCH && b.ptr >= b.start + LZB_HUF_PREFETCH && ((size_t)b.ptr & 127) < 6)
                asm volatile("prefetch.global.L1 [%0];" :: "l"(b.ptr - LZB_HUF_PREFETCH));
            // four table steps on a 2 x 32-bit copy of the window kept left-aligned (<= 7 + 4*12 bits leave it)
            u32 hi = (u32)(b.win >> 32), lo = (u32)b.win;
            hi = __funnelshift_l(lo, hi, b.used); lo <<= b.used;
            u32 e = tab.look(hi), n = e >> 8, word = e & 255, used = b.used + n;
            hi = __funnelshift_l(lo, hi, n); lo <<= n;
            e = tab.look(hi); n = e >> 8; word |= (e & 255) << 8; used += n;
            hi = __funnelshift_l(lo, hi, n); lo <<= n;
            e = tab.look(hi); n = e >> 8; word |= (e & 255) << 16; used += n;
            hi = __funnelshift_l(lo, hi, n);
            e = tab.look(hi); word |= e << 24; used += e >> 8;
            b.used = used;
            *reinterpret_cast<u32*>(out + p) = word;
#else
            const u32 s0 = huf_step(b, tab), s1 = huf_step(b, tab);
            const u32 s2 = huf_step(b, tab), s3 = huf_step(b, tab);
            *reinterpret_cast<u32*>(out + p) = s0 | (s1 << 8) | (s2 << 16) | (s3 << 24);
#endif
            p += 4;
        }
        if (kWide && phase == 0 && ring != nullptr) {
        // sixteen symbols per round, stored as ONE 16-byte vector: the 32 lanes of a warp write 32 different streams, so every
        // store instruction costs the memory pipe 32 line accesses whatever its width -- a quarter of the stores of the
        // four-byte form.  Same walk: four times (reload, four symbols).
        //
        // The bitstream is read backwards, ~3 bytes per reload.  Its bytes around the read position live in a 64-byte ring of
        // this lane (address-mapped: the word at address a is ring word (a >> 2) & 15), refilled at ONE place, at the top of a
        // round, for all lanes together: the aligned 16-byte vector below the ring is requested a whole round before it is
        // stored into the ring (`nx`), and a reload reads its 8 bytes from the ring.  A round moves the read position down by
        // at most 32 bytes (four reloads of <= 64 bits), so with the ring's lowest vector at floor16(ptr - 32) every reload of
        // the round finds its bytes.
        // Why not in registers: a lane needs a new vector every ~5 reloads, each lane at its own time.  With the window in
        // registers the refill is a lane-divergent branch, and the scoreboard that guards the loaded registers is the WARP's:
        // whichever lanes refill next wait for the load the previous lanes issued one reload ago -- a memory latency per
        // reload, about a third of the kernel's stall samples.  Here a loaded register is first
        // read a round (~1000 cycles) after its load was issued, by construction.
        {
        // loop state in 32 bits: positions relative to the start of the bitstream (`rel`, `wa`: may run below zero by less
        // than 48), addresses by their low 32 bits (`a0` + position: all the ring mapping and the alignment need)
        const u8* const s_end = b.start + len;
        const u32 a0 = (u32)(size_t)b.start;
        int rel = (int)(b.ptr - b.start);
        u32 used = b.used;
        int wa = 0; bool primed = false;                          // position of the ring's lowest vector
        HufVec nx = huf_vec_zero();                               // the vector at wa - 16, in flight
        u32 po = (u32)p; const u32 cnt = (u32)count, o0 = (u32)(size_t)out;
        while (po + 16 <= cnt && ((o0 + po) & 15u) == 0) {
            if (rel >= 16 && used <= 64) {
                const int tgt = (int)(((a0 + (u32)rel - 32u) & ~15u) - a0);
                if (!primed) {
                    primed = true; wa = tgt;
                    for (int k = 0; k < 4; ++k) huf_ring_put(ring, a0 + (u32)(wa + 16 * k), huf_vec_load(b.start + (wa + 16 * k), b.start, s_end));
                    nx = huf_vec_load(b.start + (wa - 16), b.start, s_end);
                } else {
                    while (wa > tgt) {                            // once; twice after a round of codes longer than 8 bits
                        wa -= 16;
                        huf_ring_put(ring, a0 + (u32)wa, nx);
                        nx = huf_vec_load(b.start + (wa - 16), b.start, s_end);
#if defined(__CUDA_ARCH__)
                        if (LZB_HUF_PREFETCH && wa >= LZB_HUF_PREFETCH && ((a0 + (u32)wa) & 127u) == 0)
                            LZB_HUF_PREFETCH_ASM(b.start + (wa - LZB_HUF_PREFETCH));
#endif
                    }
                }
            }
            u32 w4[4] = {0, 0, 0, 0};
            int r = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
            for (int q = 0; q < 4; ++q) {
                if (r == q && rel >= 16 && used <= 64) {
                    rel -= (int)(used >> 3);
                    used &= 7;
                    LZB_SHIM_CHECK(rel >= wa && rel + 8 <= wa + 64);
                    const u32 a = a0 + (u32)rel, t = a >> 2, bs = (a & 3) * 8;
                    const u32 y0 = ring[(t & 15u) * kHufRingStride], y1 = ring[((t + 1) & 15u) * kHufRingStride];
                    const u32 y2 = ring[((t + 2) & 15u) * kHufRingStride];
                    u32 lo = fsh_r(y0, y1, bs), hi = fsh_r(y1, y2, bs);                  // the 8 bytes at the read position
                    hi = fsh_l(lo, hi, used); lo <<= used;
                    u32 s0, s1, s2, s3, n0, n1, n2, n3;
                    tab.look2(hi, &s0, &n0); hi = fsh_l(lo, hi, n0); lo <<= n0;
                    tab.look2(hi, &s1, &n1); hi = fsh_l(lo, hi, n1); lo <<= n1;
                    tab.look2(hi, &s2, &n2); hi = fsh_l(lo, hi, n2);
                    tab.look2(hi, &s3, &n3);
                    used += n0 + n1 + n2 + n3;
                    w4[q] = s0 | (s1 << 8) | (s2 << 16) | (s3 << 24);
                    r = q + 1;
                }
            }
            if (r == 4) { huf_store16(out + po, w4[0], w4[1], w4[2], w4[3]); po += 16; continue; }
            // the walk reached the last 16 bytes of the bitstream inside this round: hand over what was decoded
            if (r > 0) *reinterpret_cast<u32*>(out + po) = w4[0];
            if (r > 1) *reinterpret_cast<u32*>(out + po + 4) = w4[1];
            if (r > 2) *reinterpret_cast<u32*>(out + po + 8) = w4[2];
            po += 4 * (u32)r;
            break;
        }
        b.ptr = b.start + rel; b.used = used; p = (long)po;
        }
        }
        }
    }
    for (;;) {
        if (bits_reload(b) != kBitsUnfinished) break;
        long k = count - p; if (k > 4) k = 4;
        if (k <= 0) break;
        for (long j = 0; j < k; ++j) out[p++] = (u8)huf_step(b, tab);
    }
    while (p < count) out[p++] = (u8)huf_step(b, tab);
    return bits_done(b);
}
// own function on the device: its loop must not share a register allocation with the token loops
LZ_HD_COLD bool huf_lane_segment(u8* out, long count, const u8* src, u32 len, const u16* table, u32 tl, int* init_err)
{
    HufFull tab; tab.t = table; tab.down = 32 - tl;
    return huf_lane_segment_t<false>(out, count, src, len, tab, init_err);
}

// segment k (0..3) of a stream prepared by huf_job_prepare: the pre-pass's unit of work (huf_expand.cuh).  `pay` = the
// stream behind its weight header, `pc` its size.  Same split and same walk as huf_decompress_lanes below.
// `ring`: this lane's kHufRingWords words (stride kHufRingStride) for the bitstream window
LZ_HD bool huf_job_segment(u8* dst, u32 n, const u8* pay, u32 pc, u32 k, const HufCompact& table, u32* ring)
{
    const u32 l1 = rd_le16(pay), l2 = rd_le16(pay + 2), l3 = rd_le16(pay + 4);
    const u32 l4 = pc - (l1 + l2 + l3 + 6);
    const long seg = (long)((n + 3) / 4);
    const u8* s = pay + 6 + (k > 0 ? l1 : 0) + (k > 1 ? l2 : 0) + (k > 2 ? l3 : 0);
    const u32 len = k == 0 ? l1 : k == 1 ? l2 : k == 2 ? l3 : l4;
    long cnt = k < 3 ? seg : (long)n - 3 * seg;
    if (cnt < 0) cnt = 0;
    int ierr = 0;
    const bool good = huf_lane_segment_t<true>(dst + (long)k * seg, cnt, s, len, huf_view(&table), &ierr, ring);
    return good && ierr >= 0;
}

// HUF_decompress for one stream; all lanes return the same value (n or negative)
template <class W> LZ_HD int huf_decompress_lanes(u8* dst, u32 n, const u8* src, u32 c, DecWarpCore* sh)
{
    const u32 lane = W::lane();
    if (n == 0) return kErrDstSmall;
    if (c > n) return kErrCorrupt;
    if (c == n) { lanes_copy<W>(dst, src, n); W::sync(); return (int)n; }
    if (c == 1) { lanes_fill<W>(dst, src[0], n); W::sync(); return (int)n; }
    const u32 algo = huf_select_decoder(n, c);
    int h = 0; u32 tl = 0;
    if (lane == 0) {
        u32 nsym = 0;
        h = huf_read_stats(sh->weights, sh->rank, &nsym, &tl, src, c, &sh->stats);
        if (h >= 0) huf_fill_dtable(sh->big_table, sh->weights, sh->rank, nsym, tl);
    }
    h = W::bcast(h);
    tl = (u32)W::bcast((int)tl);
    const u16* const table = sh->big_table;
    if (h < 0) return h;
    if ((u32)h >= c) return kErrSrcSize;
    W::sync();
    const u8* pay = src + h;
    const u32 pc = c - (u32)h;
    if (pc < 10) return kErrCorrupt;
    const u32 l1 = rd_le16(pay), l2 = rd_le16(pay + 2), l3 = rd_le16(pay + 4);
    if (l1 + l2 + l3 + 6 > pc) return kErrCorrupt;
    const u32 l4 = pc - (l1 + l2 + l3 + 6);
    const long seg = (long)((n + 3) / 4);
    bool ok = true;
    int ierr[4] = {0, 0, 0, 0};
    for (u32 k = lane; k < 4; k += W::lanes()) {
        const u8* s = pay + 6 + (k > 0 ? l1 : 0) + (k > 1 ? l2 : 0) + (k > 2 ? l3 : 0);
        const u32 len = k == 0 ? l1 : k == 1 ? l2 : k == 2 ? l3 : l4;
        long cnt = k < 3 ? seg : (long)n - 3 * seg;
        if (cnt < 0) cnt = 0;
        const bool good = huf_lane_segment(dst + (long)k * seg, cnt, s, len, table, tl, &ierr[k]);
        ok = ok && good;
    }
    // the reference initialises the four readers before decoding anything and returns the first failure
    for (u32 k = 0; k < 4; ++k) {
        const u32 owner = k % W::lanes();
        const int e = (int)W::shfl((u32)ierr[k], owner);
        if (e < 0) return e;
    }
    const bool all_ok = W::ballot(!ok) == 0;
    W::sync();
    if (all_ok) return (int)n;
    if (!algo) return kErrCorrupt;
    // the reference would have run its double-symbol decoder, which tolerates a few malformed tails
    int r = 0;
    if (lane == 0) r = huf_decode4_serial(dst, n, pay, pc, table, tl, 1);
    r = W::bcast(r);
    W::sync();
    return r;
}

// ---- one inner block's streams ------------------------------------------------------------------
struct Streams {
    const u8* flags;  u32 nflags;
    const u8* lits;   u32 nlits;
    const u8* off16;  u32 noff16;
    const u8* off24;  u32 noff24;
    const u8* src_begin;              // the whole compressed unit (bound for stray reads)
    const u8* src_end;
};

// byte of a stream that the reference reads without an exact bound: real memory past a raw stream is
// the rest of the compressed unit; anything further reads as zero here
LZ_HD u32 stray_byte(const u8* p, const Streams& s)
{
    return (p >= s.src_begin && p < s.src_end) ? *p : 0u;
}

// length extension byte(s): b<254 -> b ; 254 -> LE16 ; 255 -> LE24  (lizard_decompress_lz4.h:50-61)
LZ_HD u32 read_ext(const u8* lits, u32 nlits, long& lp)
{
    u32 v = lits[lp];
    if (v >= 254) {
        const u32 b1 = lp + 1 < (long)nlits ? lits[lp + 1] : 0, b2 = lp + 2 < (long)nlits ? lits[lp + 2] : 0;
        if (v == 254) { v = b1 | (b2 << 8); lp += 2; }
        else { const u32 b3 = lp + 3 < (long)nlits ? lits[lp + 3] : 0; v = b1 | (b2 << 8) | (b3 << 16); lp += 3; }
    }
    lp++;
    return v;
}

// length-extension field at lits[p]: value v (b<254 | 254,LE16 | 255,LE24) and its size in bytes; false when the
// stream does not hold the whole field (the serial path then reproduces the reference's behaviour)
LZ_HD bool ext_field(const u8* lits, long nl, long p, u32* v, u32* size)
{
    if (p >= nl) return false;
    const u32 b = lits[p];
    if (b < 254) { *v = b; *size = 1; return true; }
    const u32 sz = b == 254 ? 3u : 4u;
    if (p + (long)sz > nl) return false;
    *v = b == 254 ? rd_le16(lits + p + 1) : rd_le24(lits + p + 1);
    *size = sz;
    return true;
}

#if defined(LZB_STATS) && !defined(__CUDA_ARCH__)
static unsigned long long g_tok_fast = 0, g_tok_slow = 0;
#define LZB_COUNT_FAST(n) (g_tok_fast += (n))
#define LZB_COUNT_SLOW(n) (g_tok_slow += (n))
#else
#define LZB_COUNT_FAST(n)
#define LZB_COUNT_SLOW(n)
#endif

// cursor state of one token loop
struct TokCursor { u32 fp; long lp; long op; u32 p16, p24; u32 last_off; };

// ---- serial path: the reference's loop, one token at a time (all lanes in lock step) ------------------
// Returns 0 to continue, or the (negative) error code.  Runs at most `count` tokens.
// kPartial (Lizard_decompress_safe_partial): returns 1 when the reference's loop stops at `oexit`, with c.op where it stopped.
// kDict: matches may reach into the dictionary `dw` (c.op is the position in the unit, so offsets up to c.op + dw.reach pass).
template <class W, bool kPartial = false, bool kDict = false>
LZ_HD int lz4_serial(const Streams& s, u8* dst, long oend, TokCursor& c, u32 count, long oexit = 0, DictWin dw = DictWin())
{
    const long nl = (long)s.nlits;
    const long reach = kDict ? (long)dw.reach : 0;
    for (u32 t = 0; t < count && c.fp < s.nflags; ++t) {
        const u32 tok = s.flags[c.fp++];
        u32 len = tok & 15;
        if (len == 15) {
            if (c.lp > nl - 5) return -(int)c.fp - 1;
            len = read_ext(s.lits, s.nlits, c.lp) + 15;
        }
        if (c.op + len > oend - 16 || c.lp + len > nl - 18) return -(int)c.fp - 1;
        lanes_copy<W>(dst + c.op, s.lits + c.lp, len);
        c.op += len; c.lp += len;
        if (kPartial && c.op >= oexit) { W::sync(); return 1; }    // lizard_decompress_lz4.h:82, before the offset is read
        const u32 off = rd_le16(s.lits + c.lp); c.lp += 2;
        if ((long)off > c.op + reach) return -(int)c.fp - 1;       // match < lowLimit
        u32 ml = tok >> 4;
        if (ml == 15) {
            if (c.lp > nl - 5) return -(int)c.fp - 1;
            ml = read_ext(s.lits, s.nlits, c.lp) + 15;
        }
        ml += kMinMatch;
        if (c.op + ml > oend - 16) return -(int)c.fp - 1;
        W::sync();
        if (kDict) dict_match<W>(dst, c.op, off, ml, dw);
        else lanes_match<W>(dst, c.op, off, ml);
        W::sync();
        c.op += ml;
        if (kPartial && c.op >= oexit) return 1;                    // :144, the block's last literals are not copied
    }
    return 0;
}

template <class W, bool kPartial = false, bool kDict = false>
LZ_HD int lizv1_serial(const Streams& s, u8* dst, long oend, TokCursor& c, u32 count, long oexit = 0, DictWin dw = DictWin())
{
    const long nl = (long)s.nlits;
    const long reach = kDict ? (long)dw.reach : 0;
    for (u32 t = 0; t < count && c.fp < s.nflags; ++t) {
        if (kPartial && c.op >= oexit) return 1;                    // lizard_decompress_liz.h:55, before the flags byte is read
        const u32 tok = s.flags[c.fp++];
        u32 ml;
        if (tok >= 32) {
            u32 len = tok & 7;
            if (len == 7) {
                if (c.lp > nl - 1) return -(int)c.fp - 1;
                len = read_ext(s.lits, s.nlits, c.lp) + 7;
            }
            if (c.op + len > oend - 16 || c.lp > nl - 16) return -(int)c.fp - 1;
            {   // the reference copies first and notices an over-long run later; never read past the stream
                const u32 avail = c.lp < nl ? (u32)(nl - c.lp) : 0;
                lanes_copy<W>(dst + c.op, s.lits + c.lp, len < avail ? len : avail);
            }
            c.op += len; c.lp += len;
            if (c.p16 > s.noff16) return -(int)c.fp - 1;
            if ((tok >> 7) == 0) {                                // new 16-bit offset; bit 7 set = repeat last offset
                if (c.p16 + 2 <= s.noff16) c.last_off = rd_le16(s.off16 + c.p16);
                else c.last_off = stray_byte(s.off16 + c.p16, s) | (stray_byte(s.off16 + c.p16 + 1, s) << 8);
                c.p16 += 2;
            }
            ml = (tok >> 3) & 15;
            if (ml == 15) {
                if (c.lp > nl - 1) return -(int)c.fp - 1;
                ml = read_ext(s.lits, s.nlits, c.lp) + 15;
            }
        } else if (tok < kLastLongOff) {
            if ((long)c.p24 > (long)s.noff24 - 3) return -(int)c.fp - 1;
            ml = tok + kMmLongOff;
            c.last_off = rd_le24(s.off24 + c.p24); c.p24 += 3;
        } else {
            if (c.lp > nl - 1) return -(int)c.fp - 1;
            ml = read_ext(s.lits, s.nlits, c.lp) + kLastLongOff + kMmLongOff;
            if ((long)c.p24 > (long)s.noff24 - 3) return -(int)c.fp - 1;
            c.last_off = rd_le24(s.off24 + c.p24); c.p24 += 3;
        }
        if ((long)c.last_off > c.op + reach) return -(int)c.fp - 1; // match < lowLimit
        if (c.op + ml > oend - 16) return -(int)c.fp - 1;
        W::sync();
        if (kDict) dict_match<W>(dst, c.op, c.last_off, ml, dw);
        else lanes_match<W>(dst, c.op, c.last_off, ml);
        W::sync();
        c.op += ml;
    }
    return 0;
}

// ---- token pre-pass: one lane parses one block (huf_expand.cuh, "token pre-pass") --------------------------------------
// The reference's loops again, without the copies: every check of lz4_serial / lizv1_serial (plus the bounds the batch
// path adds so that nothing outside a stream is ever read) must hold, otherwise the function returns false and the unit
// is decoded by the in-kernel path, which reproduces the reference's verdict and error code.  Record = {a: literal run's
// place in the literals stream, b: its length, c: match offset, d: match length}.
LZ_HD void parse_prefetch(const u8* p)      // the walk is a chain of dependent loads: keep the lines ahead of it on their way
{
#if defined(__CUDA_ARCH__)
    asm volatile("prefetch.global.L1 [%0];" :: "l"(p));
#else
    (void)p;
#endif
}
LZ_HD bool parse_block_lz4(const Streams& s, u32 op0, u32 oend_u, PoolRun* out, u32* final_lp, u32* final_op)
{
    const long nl = (long)s.nlits, oend = (long)oend_u;
    if (oend_u - op0 == 0) return false;
    long lp = 0, op = op0;
    for (u32 fp = 0; fp < s.nflags; ++fp) {
        const u32 tok = s.flags[fp];
        if (lp + 1024 < nl) parse_prefetch(s.lits + lp + 1024);
        if ((fp & 63) == 0 && fp + 256 < s.nflags) parse_prefetch(s.flags + fp + 256);
        u32 len = tok & 15;
        if (len == 15) {
            u32 v, sz;
            if (lp > nl - 5 || !ext_field(s.lits, nl, lp, &v, &sz)) return false;
            len = 15 + v; lp += sz;
        }
        if (op + len > oend - 16 || lp + len > nl - 18) return false;
        PoolRun r; r.a = (u32)lp; r.b = len;
        op += len; lp += len;
        r.c = rd_le16(s.lits + lp); lp += 2;
        if ((long)r.c > op) return false;
        u32 ml = tok >> 4;
        if (ml == 15) {
            u32 v, sz;
            if (lp > nl - 5 || !ext_field(s.lits, nl, lp, &v, &sz)) return false;
            ml = 15 + v; lp += sz;
        }
        ml += kMinMatch;
        if (op + ml > oend - 16) return false;
        r.d = ml;
        out[fp] = r;
        op += ml;
    }
    const long rest = nl - lp;
    if (rest < 0 || op + rest > oend) return false;
    *final_lp = (u32)lp; *final_op = (u32)op;
    return true;
}

LZ_HD bool parse_block_lizv1(const Streams& s, u32 op0, u32 oend_u, PoolRun* out, u32* final_lp, u32* final_op)
{
    const long nl = (long)s.nlits, oend = (long)oend_u;
    if (oend_u - op0 == 0) return false;
    long lp = 0, op = op0;
    u32 p16 = 0, p24 = 0, last_off = 0;
    for (u32 fp = 0; fp < s.nflags; ++fp) {
        const u32 tok = s.flags[fp];
        if (lp + 1024 < nl) parse_prefetch(s.lits + lp + 1024);
        if ((fp & 63) == 0) {
            if (fp + 256 < s.nflags) parse_prefetch(s.flags + fp + 256);
            if (p16 + 512 < s.noff16) parse_prefetch(s.off16 + p16 + 512);
        }
        PoolRun r; r.a = (u32)lp; r.b = 0;
        u32 ml;
        if (tok >= 32) {
            u32 len = tok & 7;
            if (len == 7) {
                u32 v, sz;
                if (lp > nl - 1 || !ext_field(s.lits, nl, lp, &v, &sz)) return false;
                len = 7 + v; lp += sz;
            }
            if (op + len > oend - 16 || lp > nl - 16 || lp + (long)len > nl) return false;
            r.a = (u32)lp; r.b = len;
            op += len; lp += len;
            if ((tok >> 7) == 0) {
                if (p16 + 2 > s.noff16) return false;
                last_off = rd_le16(s.off16 + p16); p16 += 2;
            } else if (p16 > s.noff16) return false;
            ml = (tok >> 3) & 15;
            if (ml == 15) {
                u32 v, sz;
                if (lp > nl - 1 || !ext_field(s.lits, nl, lp, &v, &sz)) return false;
                ml = 15 + v; lp += sz;
            }
        } else {
            if (tok < kLastLongOff) ml = tok + kMmLongOff;
            else {
                u32 v, sz;
                if (lp > nl - 1 || !ext_field(s.lits, nl, lp, &v, &sz)) return false;
                ml = v + kLastLongOff + kMmLongOff; lp += sz;
            }
            if ((long)p24 > (long)s.noff24 - 3) return false;
            last_off = rd_le24(s.off24 + p24); p24 += 3;
        }
        if ((long)last_off > op) return false;
        if (op + ml > oend - 16) return false;
        r.c = last_off; r.d = ml;
        out[fp] = r;
        op += ml;
    }
    const long rest = nl - lp;
    if (rest < 0 || op + rest > oend) return false;
    *final_lp = (u32)lp; *final_op = (u32)op;
    return true;
}

// Streams of the first inner block of a unit for the token pre-pass: raw streams in place, Huffman-coded ones from the
// Huffman pre-pass's arena.  False when the block is not of the plain kind (stored block, damaged header, a coded stream
// the pre-pass did not expand): decode_unit then does everything itself.  Mirrors decode_unit / read_stream.
LZ_HD bool locate_first_block(const u8* src, u32 csize_u, const UnitPre* up, const u8* arena, Streams* st, int* lizv1)
{
    const long csize = (long)csize_u;
    if (csize < 2) return false;
    const int level = src[0];
    if (level < (int)kMinLevel || level > (int)kMaxLevel) return false;
    *lizv1 = level_is_lizv1(level);
    long ip = 1;
    const u32 hdr = src[ip++];
    if (hdr == kFlagRaw || (hdr & kFlagLen)) return false;
    if (ip > csize - 15) return false;
    {
        const long len_end = ip + 3 + (long)rd_le24(src + ip);
        if (len_end > csize - 3) return false;
        ip = len_end;
    }
    st->src_begin = src; st->src_end = src + csize;
    const u32 bit[4] = { kFlagOff16, kFlagOff24, kFlagFlags, kFlagLiterals };
    const u8* ptr[4]; u32 len[4];
    for (int k = 0; k < 4; ++k) {
        if (hdr & bit[k]) {
            if (k < 2 || up == nullptr) return false;
            if (ip > csize - 6) return false;
            const u32 n = rd_le24(src + ip), c = rd_le24(src + ip + 3);
            if (n > kBlockSize || ip + (long)c > csize - 6) return false;
            const u32 slot = k == 3 ? kSlotLiterals : kSlotFlags;
            if (up->state[slot] != kPreDone) return false;
            ptr[k] = arena + up->off[slot]; len[k] = n;
            ip += (long)c + 6;
        } else {
            if (ip > csize - 3) return false;
            len[k] = rd_le24(src + ip);
            ptr[k] = src + ip + 3;
            ip += 3 + (long)len[k];
        }
    }
    if (ip > csize) return false;
    st->off16 = ptr[0]; st->noff16 = len[0]; st->off24 = ptr[1]; st->noff24 = len[1];
    st->flags = ptr[2]; st->nflags = len[2]; st->lits = ptr[3]; st->nlits = len[3];
    return true;
}

// ---- batch execution shared by both flavours: copy the literal runs, then resolve the matches in order ----
// Every lane publishes its sequence as two 16-byte descriptors in the warp's shared memory; the copy loops then
// read them with uniform (broadcast) loads instead of three shuffles per sequence.
template <class W> LZ_HD void run_batch_copies(u8* dst, const u8* lits, u32 nb, u32 lit_src, u32 lit_len,
                                               u32 opos, u32 off, u32 ml, SeqDesc* desc)
{
    const u32 lane = W::lane(), L = W::lanes();
    if (lane < nb) {
        SeqDesc dl; dl.a = lit_src; dl.b = opos; dl.c = lit_len; dl.d = 0;
        SeqDesc dm; dm.a = opos + lit_len; dm.b = off; dm.c = ml; dm.d = 0;
        desc[lane] = dl; desc[32 + lane] = dm;
    }
    // warm the cache for this lane's match source while the literal runs are being moved
    if (lane < nb && off != 0 && off <= opos + lit_len) W::prefetch(dst + (opos + lit_len - off));
    W::sync();
    typedef LaneGroups<W> LG;
    const u32 sub = lane / LG::kGroup;
    const bool act = lane < nb;
    // ---- literal runs are independent of everything in this batch: short ones go one lane group each
    //      (LG::kRuns at a time), long ones take the whole warp, two at a time
    {
        const bool l_long = act && lit_len > LG::kMaxBytes;
        const u32 shorts = W::ballot(act && lit_len != 0 && !l_long);
        u32 longs = W::ballot(l_long);
        for (u32 k0 = 0; k0 < nb; k0 += LG::kRuns) {
            if (((shorts >> k0) & ((1u << LG::kRuns) - 1)) == 0) continue;
            const u32 k = k0 + sub;
            const SeqDesc d0 = desc[k];
            const u32 n = (k < nb && d0.c <= LG::kMaxBytes) ? d0.c : 0u;
            lanes_copy_groups<W>(dst + d0.b, lits + d0.a, n);
        }
        for (; longs; longs &= longs - 1) {
            const SeqDesc d0 = desc[ctz32(longs)];
            if (d0.c >= kWideMinBytes) lanes_copy_wide<W>(dst + d0.b, lits + d0.a, d0.c, false);
            else lanes_copy_rows<W>(dst + d0.b, lits + d0.a, d0.c);
        }
    }
    W::sync();
    // ---- matches, LG::kRuns sequences per step.  A match is "free" when it is short, does not overlap itself and
    //      does not read what an earlier match of the same step writes: the free ones go together, one lane group
    //      each; the others follow one by one in order.  (A match never reads the destination of a later one: its
    //      source ends before its own destination does.)
    const u32 mdst = opos + lit_len, msrc = mdst - off;
    bool clash = false;
    for (u32 j = 1; j < LG::kRuns; ++j) {
        const u32 pd = W::shfl(mdst, (lane - j) & (L - 1)), pm = W::shfl(ml, (lane - j) & (L - 1));
        if ((lane & (LG::kRuns - 1)) >= j && msrc < pd + pm && pd < msrc + ml) clash = true;
    }
    const u32 held = W::ballot(act && ml != 0 && !(ml <= LG::kMaxBytes && off >= ml && !clash));
    for (u32 k0 = 0; k0 < nb; k0 += LG::kRuns) {
        const u32 step_mask = ((1u << LG::kRuns) - 1) << k0;
        if ((~held & step_mask) != 0) {
            const u32 k = k0 + sub;
            const SeqDesc d = desc[32 + k];
            const u32 n = (k < nb && !((held >> k) & 1)) ? d.c : 0u;
            lanes_copy_groups<W>(dst + d.a, dst + d.a - d.b, n);
            W::sync();
        }
        for (u32 rest = held & step_mask; rest; rest &= rest - 1) {
            const SeqDesc d = desc[32 + ctz32(rest)];
            const u32 m = d.c, o = d.b;
            u8* const to = dst + d.a;
            if (m >= kWideMinBytes && o >= wide_min_offset<W>()) lanes_copy_wide<W>(to, to - o, m, true);
            else if (o >= m || o >= 4 * L) {
                // source entirely before the destination of each pass: plain passes, ordered by a barrier
                for (u32 base = 0; base < m; base += 4 * L) {
                    const u32 part = m - base < 4 * L ? m - base : 4 * L;
                    lanes_copy_rows<W>(to + base, to + base - o, part);
                    if (base + 4 * L < m) W::sync();
                }
            } else lanes_match<W>(dst, (long)d.a, o, m);
            W::sync();
        }
    }
}

// ---- batch execution, pooled form (decode variant 1) ---------------------------------------------------------------
// Same contract as run_batch_copies, different schedule: instead of walking the batch run by run, the runs are sorted
// into four pools -- short / long literal runs, short / long matches that read nothing a match of this batch writes --
// and every pool is moved by one sweep that keeps all lanes busy (pool_copy_short / pool_copy_long, lanes.cuh).  Only
// the matches that do read the output of an earlier match of the same batch (or themselves) follow one by one, in order.
// kDict: a match may start below the unit start (off > its destination): one that lies wholly in the dictionary `dw` reads
// nothing this batch writes and goes in a sweep of its own, one that runs past the dictionary's end goes in order.
template <class W, bool kDict = false> LZ_HD void run_batch_copies_pool(u8* dst, const u8* lits, u32 nb, u32 lit_src, u32 lit_len,
                                                                       u32 opos, u32 off, u32 ml, PoolRun* pool,
                                                                       DictWin dw = DictWin())
{
    typedef LaneGroups<W> LG;
    const u32 lane = W::lane(), L = W::lanes();
    const bool act = lane < nb;
    const u32 mdst = opos + lit_len;
    if (W::kLanes == 1) {                                   // one-lane host build: the reference's order
        if (act) {
            for (u32 i = 0; i < lit_len; ++i) dst[opos + i] = lits[lit_src + i];
            if (kDict) dict_match<W>(dst, (long)mdst, off, ml, dw);
            else lanes_match<W>(dst, (long)mdst, off, ml);
        }
        return;
    }
    if (act && off != 0 && off <= mdst) W::prefetch(dst + (mdst - off));
#if defined(LZB_DEC_MATCH_PF2)
    if (act && off != 0 && off <= mdst && ml > 1) {           // A/B: the source's last line as well, when it is another one
        const u8* const e = dst + (mdst - off) + (ml < off ? ml : off) - 1;
        if ((((size_t)e) ^ ((size_t)(dst + (mdst - off)))) >> 7) W::prefetch(e);
    }
#endif
#if !defined(LZB_DEC_STREAM_LITS)
#define LZB_DEC_STREAM_LITS 0      /* evict-first literal loads: measured no gain (profiles/r02_SUMMARY.md) */
#endif
    pool_copy_short<W, LZB_DEC_STREAM_LITS != 0>(dst, lits, W::ballot(act && lit_len != 0 && lit_len <= LG::kMaxBytes), opos, lit_src, lit_len, pool);
    pool_copy_long<W, LZB_DEC_STREAM_LITS != 0>(dst, lits, W::ballot(act && lit_len > LG::kMaxBytes), opos, lit_src, lit_len, pool + 32);
    W::sync();
    // A match is "free" when its source lies before the first match destination of this batch (older output, or the
    // first literal run), or inside ONE literal run of this batch: those bytes are final now.
    const u32 msrc = mdst - off;                            // off <= mdst was checked by the caller, unless kDict
    const bool below = kDict && act && ml != 0 && off > mdst;
    const bool dict_only = below && off - mdst >= ml;
    const bool real = act && ml != 0 && off != 0 && !below;
    if (kDict) {
        const u32 sel_s = W::ballot(dict_only && ml <= LG::kMaxBytes), sel_l = W::ballot(dict_only && ml > LG::kMaxBytes);
        if ((sel_s | sel_l) != 0) {
            // positions relative to the lowest readable dictionary byte, so that they stay unsigned
            const u8* const lo = dw.end - dw.avail;
            const u32 from = dw.avail - (off - mdst);
            pool_copy_short<W>(dst, lo, sel_s, mdst, from, ml, pool);
            pool_copy_long<W>(dst, lo, sel_l, mdst, from, ml, pool + 32);
            W::sync();                                      // the sweeps below reuse the pool
        }
        LZB_COUNT_DICT(lane == 0 ? popc32(sel_s | sel_l) : 0, 0);      // the others are counted by dict_match
    }
    const u32 first = W::shfl(mdst, 0);
    bool free_m = real && msrc + ml <= first;
    {
        u32 pos = 0;                                        // last sequence whose output starts at or before msrc
        for (u32 st = W::kLanes >> 1; st; st >>= 1) { const u32 v = W::shfl(opos, pos + st); if (v <= msrc) pos += st; }
        const u32 lit_beg = W::shfl(opos, pos), lit_end = W::shfl(mdst, pos);
        if (real && msrc >= lit_beg && msrc + ml <= lit_end) free_m = true;
    }
    pool_copy_short<W>(dst, dst, W::ballot(free_m && ml <= LG::kMaxBytes), mdst, msrc, ml, pool);
    pool_copy_long<W>(dst, dst, W::ballot(free_m && ml > LG::kMaxBytes), mdst, msrc, ml, pool + 32);
    u32 rest = W::ballot(act && ml != 0 && !free_m && !dict_only);
    if (rest == 0) return;
    W::sync();
    for (; rest; rest &= rest - 1) {
        const u32 k = ctz32(rest);
        const u32 m = W::shfl(ml, k), o = W::shfl(off, k);
        u8* const to = dst + W::shfl(mdst, k);
        if (kDict && (long)o > (long)(to - dst)) dict_match<W>(dst, (long)(to - dst), o, m, dw);
        else if (m >= kWideMinBytes && o >= wide_min_offset<W>()) lanes_copy_wide<W>(to, to - o, m, true);
        else if (o >= m || o >= 4 * L) {
            for (u32 base = 0; base < m; base += 4 * L) {
                const u32 part = m - base < 4 * L ? m - base : 4 * L;
                lanes_copy_rows<W>(to + base, to + base - o, part);
                if (base + 4 * L < m) W::sync();
            }
        } else lanes_match<W>(dst, (long)(to - dst), o, m);
        W::sync();
    }
}

// Length-extension chain of one batch, compact form.  Lanes whose token carries an extension field put
// (A | litn << 16 | has-literal-ext << 24 | has-match-ext << 25) into `ent` in token order; the warp then walks that list
// with uniform loads: only the VALUE of a literal-length field and the SIZE of any field move later tokens.  epre[j] = bytes
// of extension data before list entry j (beyond the one byte per field already counted in A).  Returns false when a field
// is cut off by the end of the stream (the serial path then reproduces the reference's verdict).  `lbias` = 15 (LZ4
// codewords, fields read only while base <= nl-5) or 7 (LIZv1, base <= nl-1); `gap` = bytes between the literal run and
// the match-length field (the inline 16-bit offset of the LZ4 flavour).
template <class W> LZ_HD bool ext_chain(const u8* lits, long nl, long lp, u32 npend, const u32* ent, u32* epre,
                                        u32 lbias, long room, u32 gap, u32* total)
{
    u32 E = 0;
    for (u32 j = 0; j < npend; ++j) {
        const u32 e = ent[j];
        const long base = lp + (long)(e & 0xffffu) + (long)E;
        if (W::lane() == 0) epre[j] = E;
        long pm;
        if (e & (1u << 24)) {
            u32 v, sz;
            if (base > nl - room || !ext_field(lits, nl, base, &v, &sz)) return false;
            E += lbias + v + (sz - 1);
            pm = base + (long)sz + (long)(lbias + v) + (long)gap;
        } else pm = base + (long)((e >> 16) & 255u) + (long)gap;
        if (e & (1u << 25)) {
            u32 v, sz;
            if (pm > nl - room || !ext_field(lits, nl, pm, &v, &sz)) return false;
            E += sz - 1;
        }
    }
    *total = E;
    return true;
}

// ---- the same chain through a shared-memory window of the literals stream ------------------------------------------
// The chain is a pointer chase: ~28 dependent one-byte loads per batch, each an L2 round trip (the
// lines are not in an L1 that 32 resident warps share).  Here the warp copies 1 KiB of the stream -- from the 16-byte
// aligned address at or below the position the chain has reached -- into shared memory with two coalesced vector loads per
// lane and walks on from there; a batch needs ~3 windows.  The window lives in the batch's copy descriptors, which are only
// written after the chain.  An entry's results go back through its record (one 16-byte store by lane 0, one 16-byte load
// by the entry's lane), so that no lane returns to the stream for its fields.  Everything is 32-bit: stream positions,
// and addresses by their low bits (`a0` + position), which is all the window mapping needs.
#if !defined(LZB_DEC_CHAIN_WIN)
#define LZB_DEC_CHAIN_WIN 1
#endif
enum : u32 { kChainWinBytes = 1024 };
struct ChainMem {                 // the chain's shared memory: 32-bit shared-space addresses on the device (kept opaque: the
#if defined(__CUDA_ARCH__)        // compiler otherwise re-derives "block base + warp * size" in front of every access)
    u32 rec_at, win_at;
#else
    ChainRec* rec; u8* win;
#endif
};
LZ_HD ChainMem chain_mem(ChainRec* rec, void* win)
{
    ChainMem m;
#if defined(__CUDA_ARCH__)
    m.rec_at = (u32)__cvta_generic_to_shared(rec); m.win_at = (u32)__cvta_generic_to_shared(win);
    asm volatile("" : "+r"(m.rec_at), "+r"(m.win_at));
#else
    m.rec = rec; m.win = (u8*)win;
#endif
    return m;
}
LZ_HD void chain_set_ent(const ChainMem& m, u32 j, u32 ent)
{
#if defined(__CUDA_ARCH__)
    asm volatile("st.shared.u32 [%0], %1;" :: "r"(m.rec_at + 16 * j), "r"(ent) : "memory");
#else
    m.rec[j].ent = ent;
#endif
}
LZ_HD u32 chain_ent(const ChainMem& m, u32 j)
{
#if defined(__CUDA_ARCH__)
    u32 e; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(e) : "r"(m.rec_at + 16 * j) : "memory"); return e;
#else
    return m.rec[j].ent;
#endif
}
LZ_HD void chain_put(const ChainMem& m, u32 j, u32 ent, u32 epre, u32 vl, u32 vm)
{
#if defined(__CUDA_ARCH__)
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" :: "r"(m.rec_at + 16 * j), "r"(ent), "r"(epre), "r"(vl), "r"(vm) : "memory");
#else
    m.rec[j].ent = ent; m.rec[j].epre = epre; m.rec[j].vl = vl; m.rec[j].vm = vm;
#endif
}
LZ_HD ChainRec chain_get(const ChainMem& m, u32 j)
{
    ChainRec r;
#if defined(__CUDA_ARCH__)
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.ent), "=r"(r.epre), "=r"(r.vl), "=r"(r.vm) : "r"(m.rec_at + 16 * j) : "memory");
#else
    r = m.rec[j];
#endif
    return r;
}
LZ_HD u32 chain_win_byte(const ChainMem& m, u32 off)
{
#if defined(__CUDA_ARCH__)
    u32 b; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(b) : "r"(m.win_at + off) : "memory"); return b;
#else
    return m.win[off];
#endif
}
// copy 1 KiB of the stream, from the 16-byte aligned address at or below position p, into the window; returns that address
// (low bits).  Two halves: `issue` starts the copy (cp.async: no registers, the data goes from L1/L2 straight to shared
// memory) and `wait` makes it visible to the warp, so that the first window of a batch travels while the batch's scans run.
template <class W> LZ_HD u32 chain_win_issue(const ChainMem& m, const u8* lits, u32 nl, u32 a0, u32 p)
{
    const u32 d = (a0 + p) & 15u;
    const int cp0 = (int)p - (int)d;                            // stream position of the window's first byte (>= -15)
    W::sync();                                                  // whoever read this memory before is done
    for (u32 c = W::lane(); c < kChainWinBytes / 16; c += W::lanes()) {
        const int cp = cp0 + 16 * (int)c;
        if (cp >= (int)nl) continue;                            // chunks wholly behind the stream are never read
#if defined(__CUDA_ARCH__)
        // an aligned chunk that holds a byte of the stream lies inside the stream's allocation
        asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" :: "r"(m.win_at + 16 * c), "l"(lits + cp) : "memory");
#else
        for (int i = 0; i < 16; ++i) m.win[16 * c + i] = (cp + i >= 0 && cp + i < (int)nl) ? lits[cp + i] : 0;
#endif
    }
    return a0 + p - d;
}
template <class W> LZ_HD void chain_win_wait()
{
#if defined(__CUDA_ARCH__)
    asm volatile("cp.async.wait_all;" ::: "memory");
#endif
    W::sync();
}
// ext_field through the window (p is the same in every lane, p < nl); `wa` = the window's first address (low bits)
template <class W> LZ_HD bool chain_win_field(const ChainMem& m, const u8* lits, u32 nl, u32 a0, u32& wa, u32 p, u32* v, u32* size)
{
    u32 off = a0 + p - wa;
    if (off > kChainWinBytes - 4) { wa = chain_win_issue<W>(m, lits, nl, a0, p); chain_win_wait<W>(); off = a0 + p - wa; }
    const u32 b = chain_win_byte(m, off);
    if (b < 254) { *v = b; *size = 1; return true; }
    const u32 sz = b == 254 ? 3u : 4u;
    if (p + sz > nl) return false;
    u32 x = chain_win_byte(m, off + 1) | (chain_win_byte(m, off + 2) << 8);
    if (b == 255) x |= chain_win_byte(m, off + 3) << 16;
    *v = x; *size = sz;
    return true;
}
// `wa`: first address (low bits) of the window the caller has issued for this batch (chain_win_issue at position lp)
template <class W> LZ_HD bool ext_chain_win(const u8* lits, u32 nl, u32 lp, u32 npend, const ChainMem& m, u32 wa,
                                            u32 lbias, u32 room, u32 gap, u32* total)
{
    *total = 0;
    chain_win_wait<W>();                                        // also orders the lanes' entries before the walk
    if (npend == 0) return true;
    if (nl < room) return false;                                // no field fits
    const u32 limit = nl - room;                                // last position a field may start at
    const u32 a0 = (u32)(size_t)lits;
    u32 E = 0;
    for (u32 j = 0; j < npend; ++j) {
        const u32 e = chain_ent(m, j);
        const u32 base = lp + (e & 0xffffu) + E;
        const u32 E0 = E;
        u32 xl = 0, xm = 0, pm;
        if (e & (1u << 24)) {
            u32 v, sz;
            if (base > limit || !chain_win_field<W>(m, lits, nl, a0, wa, base, &v, &sz)) return false;
            E += lbias + v + (sz - 1);
            pm = base + sz + lbias + v + gap;
            xl = v | (sz << 24);
        } else pm = base + ((e >> 16) & 255u) + gap;
        if (e & (1u << 25)) {
            u32 v, sz;
            if (pm > limit || !chain_win_field<W>(m, lits, nl, a0, wa, pm, &v, &sz)) return false;
            E += sz - 1;
            xm = v | (sz << 24);
        }
        if (W::lane() == 0) chain_put(m, j, e, E0, xl, xm);
    }
    *total = E;
    return true;
}

// fastLZ4 codewords (lib/lizard_decompress_lz4.h:7-163).  `op0` is the offset inside the unit's output,
// `oend` the unit's capacity; matches may reach back to offset 0 of the unit.
// kPartial: the loop of Lizard_decompress_safe_partial, which returns as soon as the output reaches `oexit` (= op0 + the
// target: the reference measures the target from the start of the inner block), after a token's literals or after its match.
// kDict: matches may reach into the dictionary `dw` (the default schedule only: the pooled sweeps read it).
template <class W, int V, bool kPartial, bool kDict = false>
LZ_HD int decode_tokens_lz4(const Streams& s, u8* dst, u32 op0, u32 oend_u, DecWarpShared* sh, long oexit, DictWin dw = DictWin())
{
    static_assert(!kDict || (V & 1) != 0, "dictionary matches need the pooled copy sweeps");
    const long nl = (long)s.nlits, oend = (long)oend_u;
    const long reach = kDict ? (long)dw.reach : 0;
    const u32 NL = W::lanes(), lane = W::lane();
    if (oend_u - op0 == 0) return (s.nflags == 1 && s.flags[0] == 0) ? 0 : -1;
    TokCursor c; c.fp = 0; c.lp = 0; c.op = op0; c.p16 = c.p24 = 0; c.last_off = 0;
    while (c.fp < s.nflags) {
        const u32 nb = s.nflags - c.fp < NL ? s.nflags - c.fp : NL;
        const bool act = lane < nb;
#if LZB_DEC_LIT_PF_LOAD && defined(__CUDA_ARCH__)
        u32 warm = 0;                                               // A/B: a real load per line instead of the prefetch hint
        if (lane < LZB_DEC_LIT_PF_LINES && c.lp + 128 * (long)lane < nl) {
#if LZB_DEC_LIT_PF_LOAD == 2
            asm volatile("ld.global.L1::evict_last.u8 %0, [%1];" : "=r"(warm) : "l"(s.lits + c.lp + 128 * (long)lane));
#else
            asm volatile("ld.global.u8 %0, [%1];" : "=r"(warm) : "l"(s.lits + c.lp + 128 * (long)lane));
#endif
        }
#else
        if ((!LZB_DEC_LIT_PF_NEXT || c.fp == 0) && lane < LZB_DEC_LIT_PF_LINES && c.lp + LZB_DEC_LIT_PF_DIST + 128 * (long)lane < nl)
            W::prefetch(s.lits + c.lp + LZB_DEC_LIT_PF_DIST + 128 * (long)lane);
#endif
#if defined(LZB_DEC_LIT_PF_FAR_L2) && defined(__CUDA_ARCH__)
        if (c.lp + LZB_DEC_LIT_PF_FAR_L2 + 128 * (long)lane < nl)      // A/B: the lines of the batches after this one, into L2 only
            asm volatile("prefetch.global.L2 [%0];" :: "l"(s.lits + c.lp + LZB_DEC_LIT_PF_FAR_L2 + 128 * (long)lane));
#endif
        const ChainMem cm = chain_mem(sh->chainw, sh->desc);
        u32 cwa = 0;
        if (LZB_DEC_CHAIN_WIN && (V & 2) != 0) cwa = chain_win_issue<W>(cm, s.lits, (u32)nl, (u32)(size_t)s.lits, (u32)c.lp);
        const u32 tok = act ? s.flags[c.fp + lane] : 0;
        const u32 litn = tok & 15, mln = tok >> 4;
        const bool need = act && litn == 15;
        // bytes this token occupies in the literals stream, not counting an extended literal run itself
        const u32 adv = act ? ((need ? 1 : litn) + 2 + (mln == 15 ? 1 : 0)) : 0;
        u32 tot_adv = 0;
        const u32 A = W::excl_scan(adv, &tot_adv);
        // Serial chain over the tokens that carry a length extension (literal length and/or match length): only
        // these make a token's position in the literals stream data dependent.  E = bytes not yet counted in A.
        const bool needm = act && mln == 15;
        u32 my_lit = 0, my_lx = 0, my_mlv = 0, my_mx = 0;          // literal length / its field size, ml-ext value / size
        bool slow = false;
        u32 tot_ext = 0;
        long tokpos = 0;
        if ((V & 2) == 0) {
            u32 pending = W::ballot(need || needm), E = 0;
            const u32 needl_mask = W::ballot(need), needm_mask = W::ballot(needm);
            while (pending) {
                const u32 k = ctz32(pending); pending &= pending - 1;
                const long base = c.lp + (long)W::shfl(A, k) + (long)E;     // first stream byte of token k
                long pm;                                                     // where its match-length field would sit
                if ((needl_mask >> k) & 1) {
                    u32 v, sz;
                    if (base > nl - 5 || !ext_field(s.lits, nl, base, &v, &sz)) { slow = true; break; }
                    if (lane == k) { my_lit = 15 + v; my_lx = sz; }
                    E += 15 + v + (sz - 1);
                    pm = base + sz + 15 + v + 2;
                } else pm = base + (long)W::shfl(litn, k) + 2;
                if ((needm_mask >> k) & 1) {
                    u32 v, sz;
                    if (pm > nl - 5 || !ext_field(s.lits, nl, pm, &v, &sz)) { slow = true; break; }
                    if (lane == k) { my_mlv = v; my_mx = sz; }
                    E += sz - 1;
                }
            }
            if (!slow) {
                const u32 Eex = W::excl_scan((need ? my_lit + (my_lx - 1) : 0u) + (needm ? my_mx - 1 : 0u), &tot_ext);
                tokpos = c.lp + (long)A + (long)Eex;
            }
        } else {
            const u32 pendmask = W::ballot(need || needm);
            const u32 npend = popc32(pendmask), myidx = popc32(pendmask & ((1u << lane) - 1));
            if (LZB_DEC_CHAIN_WIN) {
                if (need || needm) chain_set_ent(cm, myidx, A | (litn << 16) | (need ? 1u << 24 : 0u) | (needm ? 1u << 25 : 0u));
                slow = !ext_chain_win<W>(s.lits, (u32)nl, (u32)c.lp, npend, cm, cwa, 15, 5, 2, &tot_ext);
                W::sync();                                      // the window is the copy descriptors' memory: all lanes are done with it
                if (!slow) {
                    ChainRec r; r.epre = tot_ext; r.vl = r.vm = 0;
                    if (myidx < npend) r = chain_get(cm, myidx);
                    tokpos = c.lp + (long)A + (long)r.epre;
                    if (need) { my_lit = 15 + (r.vl & 0xffffffu); my_lx = r.vl >> 24; }
                    if (needm) { my_mlv = r.vm & 0xffffffu; my_mx = r.vm >> 24; }
                }
            } else {
            if (need || needm) sh->chain.ent[myidx] = A | (litn << 16) | (need ? 1u << 24 : 0u) | (needm ? 1u << 25 : 0u);
            W::sync();
            slow = !ext_chain<W>(s.lits, nl, c.lp, npend, sh->chain.ent, sh->chain.epre, 15, 5, 2, &tot_ext);
            if (!slow) {
                W::sync();
                tokpos = c.lp + (long)A + (long)(myidx < npend ? sh->chain.epre[myidx] : tot_ext);
                // every lane reads its own fields (the chain has checked that they are inside the stream)
                if (need) { u32 v = 0, sz = 1; ext_field(s.lits, nl, tokpos, &v, &sz); my_lit = 15 + v; my_lx = sz; }
                if (needm) { u32 v = 0, sz = 1; ext_field(s.lits, nl, tokpos + (need ? (long)(my_lx + my_lit) : (long)litn) + 2, &v, &sz); my_mlv = v; my_mx = sz; }
            }
            }
        }
        if (!slow) {
            const u32 lit_len = need ? my_lit : (act ? litn : 0);
            const long lit_src = tokpos + (need ? (long)my_lx : 0);
            const long off_pos = lit_src + lit_len;
            bool bad = false;
            u32 ml = 0, off = 0;
            if (act) {
                if (lit_src + (long)lit_len > nl - 18) bad = true;
                else {
                    off = rd_le16(s.lits + off_pos);
                    ml = (needm ? 15 + my_mlv : mln) + kMinMatch;
                }
            }
            u32 tot_out = 0;
            const u32 O = W::excl_scan((act && !bad) ? lit_len + ml : 0, &tot_out);
            const long opos = c.op + (long)O;
            bool xl = false, xm = false;                                // kPartial: the reference stops after this token's literals / match
            if (act && !bad) {
                if (opos + (long)lit_len > oend - 16) bad = true;
                else if (kPartial && opos + (long)lit_len >= oexit) xl = true;
                else if ((long)off > opos + (long)lit_len + reach) bad = true;
                else if (opos + (long)lit_len + (long)ml > oend - 16) bad = true;
                else if (kPartial && opos + (long)lit_len + (long)ml >= oexit) xm = true;
            }
            if (kPartial) {
                // The first lane that reaches oexit ends the block.  Its position is exact when no earlier lane failed a check
                // (a failed lane adds nothing to the scan): then the batch shrinks to the tokens up to it, and failures behind
                // it are never looked at.  Otherwise the serial path below meets the earlier error, or the exit, itself.
                const u32 xs = W::ballot(xl || xm);
                if (xs != 0) {
                    const u32 e = ctz32(xs);
                    if ((W::ballot(bad) & ((2u << e) - 1u)) == 0) {
                        if (xl) ml = 0;                                 // lane e: literals only; the lanes behind it do not run
                        const u32 end = W::shfl(O + lit_len + ml, e);
                        if ((V & 1) == 0) run_batch_copies<W>(dst, s.lits, e + 1, (u32)lit_src, lit_len, (u32)opos, off, ml, sh->desc);
                        else run_batch_copies_pool<W, kDict>(dst, s.lits, e + 1, (u32)lit_src, lit_len, (u32)opos, off, ml, sh->desc, dw);
                        W::sync();
                        return (int)(c.op + (long)end - (long)op0);
                    }
                }
            }
            if (W::ballot(bad) == 0) {
                LZB_COUNT_FAST(W::lane() == 0 ? nb : 0);
                if (LZB_DEC_LIT_PF_NEXT) { const long nx = c.lp + (long)tot_adv + (long)tot_ext + 128 * (long)lane; if (lane < LZB_DEC_LIT_PF_LINES && nx < nl) W::prefetch(s.lits + nx); }
#if LZB_DEC_LIT_PF_LOAD && defined(__CUDA_ARCH__)
                asm volatile("" :: "r"(warm));
#endif
                if ((V & 1) == 0) run_batch_copies<W>(dst, s.lits, nb, (u32)lit_src, lit_len, (u32)opos, off, ml, sh->desc);
                else run_batch_copies_pool<W, kDict>(dst, s.lits, nb, (u32)lit_src, lit_len, (u32)opos, off, ml, sh->desc, dw);
                c.fp += nb; c.lp += (long)tot_adv + (long)tot_ext; c.op += (long)tot_out;
                continue;
            }
        }
        LZB_COUNT_SLOW(W::lane() == 0 ? nb : 0);
        const int e = lz4_serial<W, kPartial, kDict>(s, dst, oend, c, nb, oexit, dw);
        if (e < 0) return e;
        if (kPartial && e > 0) return (int)(c.op - (long)op0);
    }
    const long rest = nl - c.lp;
    if (rest < 0 || c.op + rest > oend) return -(int)c.fp - 1;
    if (V != 0 && rest >= (long)kWideMinBytes) lanes_copy_wide<W>(dst + c.op, s.lits + c.lp, (u32)rest, false);
    else lanes_copy<W>(dst + c.op, s.lits + c.lp, (u32)rest);
    W::sync();
    c.op += rest;
    return (int)(c.op - (long)op0);
}

// LIZv1 codewords (lib/lizard_decompress_liz.h:14-220)
// kPartial: the loop of Lizard_decompress_safe_partial, which returns in front of the first token that starts at or behind
// `oexit` (op0 + the target); once the flags run out, the block's last literals are copied whatever the target.
// kDict: as decode_tokens_lz4.
template <class W, int V, bool kPartial, bool kDict = false>
LZ_HD int decode_tokens_lizv1(const Streams& s, u8* dst, u32 op0, u32 oend_u, DecWarpShared* sh, long oexit, DictWin dw = DictWin())
{
    static_assert(!kDict || (V & 1) != 0, "dictionary matches need the pooled copy sweeps");
    const long nl = (long)s.nlits, oend = (long)oend_u;
    const long reach = kDict ? (long)dw.reach : 0;
    const u32 NL = W::lanes(), lane = W::lane();
    if (oend_u - op0 == 0) return (s.nflags == 1 && s.flags[0] == 0) ? 0 : -1;
    TokCursor c; c.fp = 0; c.lp = 0; c.op = op0; c.p16 = c.p24 = 0; c.last_off = 0;
    while (c.fp < s.nflags) {
        const u32 nb = s.nflags - c.fp < NL ? s.nflags - c.fp : NL;
        const bool act = lane < nb;
        if ((!LZB_DEC_LIT_PF_NEXT || c.fp == 0) && lane < LZB_DEC_LIT_PF_LINES && c.lp + LZB_DEC_LIT_PF_DIST + 128 * (long)lane < nl)
            W::prefetch(s.lits + c.lp + LZB_DEC_LIT_PF_DIST + 128 * (long)lane);
        const ChainMem cm = chain_mem(sh->chainw, sh->desc);
        u32 cwa = 0;
        if (LZB_DEC_CHAIN_WIN && (V & 2) != 0) cwa = chain_win_issue<W>(cm, s.lits, (u32)nl, (u32)(size_t)s.lits, (u32)c.lp);
        const u32 tok = act ? s.flags[c.fp + lane] : 32;           // inactive lanes: an empty short token
        const bool shortf = tok >= 32;                              // [r_MMMM_LLL] with a 16-bit or repeated offset
        const u32 litn = shortf ? (tok & 7) : 0;
        const u32 mln = shortf ? ((tok >> 3) & 15) : tok;
        const bool need = act && shortf && litn == 7;
        const bool mlext = act && ((shortf && mln == 15) || (!shortf && tok == kLastLongOff));
        const bool new16 = act && shortf && (tok >> 7) == 0;
        const u32 adv = act ? ((need ? 1 : litn) + (mlext ? 1 : 0)) : 0;
        u32 tot_adv = 0, tot16 = 0, tot24 = 0;
        const u32 A = W::excl_scan(adv, &tot_adv);
        const u32 P16 = W::excl_scan(new16 ? 2u : 0u, &tot16);
        const u32 P24 = W::excl_scan((act && !shortf) ? 3u : 0u, &tot24);
        u32 my_lit = 0, my_lx = 0, my_mlv = 0, my_mx = 0;
        bool slow = false;
        u32 tot_ext = 0;
        long tokpos = 0;
        if ((V & 2) == 0) {
            u32 pending = W::ballot(need || mlext), E = 0;
            const u32 needl_mask = W::ballot(need), needm_mask = W::ballot(mlext);
            while (pending) {
                const u32 k = ctz32(pending); pending &= pending - 1;
                const long base = c.lp + (long)W::shfl(A, k) + (long)E;
                long pm;
                if ((needl_mask >> k) & 1) {
                    u32 v, sz;
                    if (base > nl - 1 || !ext_field(s.lits, nl, base, &v, &sz)) { slow = true; break; }
                    if (lane == k) { my_lit = 7 + v; my_lx = sz; }
                    E += 7 + v + (sz - 1);
                    pm = base + sz + 7 + v;
                } else pm = base + (long)W::shfl(litn, k);
                if ((needm_mask >> k) & 1) {
                    u32 v, sz;
                    if (pm > nl - 1 || !ext_field(s.lits, nl, pm, &v, &sz)) { slow = true; break; }
                    if (lane == k) { my_mlv = v; my_mx = sz; }
                    E += sz - 1;
                }
            }
            if (!slow) {
                const u32 Eex = W::excl_scan((need ? my_lit + (my_lx - 1) : 0u) + (mlext ? my_mx - 1 : 0u), &tot_ext);
                tokpos = c.lp + (long)A + (long)Eex;
            }
        } else {
            const u32 pendmask = W::ballot(need || mlext);
            const u32 npend = popc32(pendmask), myidx = popc32(pendmask & ((1u << lane) - 1));
            if (LZB_DEC_CHAIN_WIN) {
                if (need || mlext) chain_set_ent(cm, myidx, A | (litn << 16) | (need ? 1u << 24 : 0u) | (mlext ? 1u << 25 : 0u));
                slow = !ext_chain_win<W>(s.lits, (u32)nl, (u32)c.lp, npend, cm, cwa, 7, 1, 0, &tot_ext);
                W::sync();
                if (!slow) {
                    ChainRec r; r.epre = tot_ext; r.vl = r.vm = 0;
                    if (myidx < npend) r = chain_get(cm, myidx);
                    tokpos = c.lp + (long)A + (long)r.epre;
                    if (need) { my_lit = 7 + (r.vl & 0xffffffu); my_lx = r.vl >> 24; }
                    if (mlext) { my_mlv = r.vm & 0xffffffu; my_mx = r.vm >> 24; }
                }
            } else {
            if (need || mlext) sh->chain.ent[myidx] = A | (litn << 16) | (need ? 1u << 24 : 0u) | (mlext ? 1u << 25 : 0u);
            W::sync();
            slow = !ext_chain<W>(s.lits, nl, c.lp, npend, sh->chain.ent, sh->chain.epre, 7, 1, 0, &tot_ext);
            if (!slow) {
                W::sync();
                tokpos = c.lp + (long)A + (long)(myidx < npend ? sh->chain.epre[myidx] : tot_ext);
                if (need) { u32 v = 0, sz = 1; ext_field(s.lits, nl, tokpos, &v, &sz); my_lit = 7 + v; my_lx = sz; }
                if (mlext) { u32 v = 0, sz = 1; ext_field(s.lits, nl, tokpos + (need ? (long)(my_lx + my_lit) : (long)litn), &v, &sz); my_mlv = v; my_mx = sz; }
            }
            }
        }
        if (!slow) {
            const u32 lit_len = need ? my_lit : (act ? litn : 0);
            const long lit_src = tokpos + (need ? (long)my_lx : 0);
            bool bad = false;
            u32 ml = 0, off = 0;
            if (act) {
                if (shortf) {
                    if (lit_src > nl - 16 || lit_src + (long)lit_len > nl) bad = true;
                    else if (c.p16 + P16 + (new16 ? 2u : 0u) > s.noff16) bad = true;
                    else {
                        if (new16) off = rd_le16(s.off16 + c.p16 + P16);
                        ml = mlext ? 15 + my_mlv : mln;
                    }
                } else {
                    ml = (tok == kLastLongOff) ? my_mlv + kLastLongOff + kMmLongOff : tok + kMmLongOff;
                    if ((long)(c.p24 + P24) > (long)s.noff24 - 3) bad = true;
                    else off = rd_le24(s.off24 + c.p24 + P24);
                }
            }
            // repeat-offset tokens take the offset of the closest earlier token that carried one
            const bool has_off = act && (new16 || !shortf);
            const u32 carriers = W::ballot(has_off);
            const u32 before = carriers & ((lane == 0) ? 0u : (0xffffffffu >> (32 - lane)));
            const u32 src_lane = before ? highbit32(before) : lane;
            const u32 inherited = W::shfl(off, src_lane);
            if (act && !has_off) off = before ? inherited : c.last_off;
            u32 tot_out = 0;
            const u32 O = W::excl_scan((act && !bad) ? lit_len + ml : 0, &tot_out);
            const long opos = c.op + (long)O;
            if (act && !bad) {
                if (shortf && opos + (long)lit_len > oend - 16) bad = true;
                else if ((long)off > opos + (long)lit_len + reach) bad = true;
                else if (opos + (long)lit_len + (long)ml > oend - 16) bad = true;
            }
            if (kPartial) {
                // The first lane that starts at or behind oexit ends the block before its token is read.  Its position is exact
                // when no earlier lane failed a check: then only the lanes in front of it run.  Otherwise the serial path below
                // meets the earlier error, or the exit, itself.
                const u32 xs = W::ballot(act && opos >= oexit);
                if (xs != 0) {
                    const u32 e = ctz32(xs);
                    if ((W::ballot(bad) & ((1u << e) - 1u)) == 0) {
                        const u32 end = W::shfl(O, e);
                        if (e > 0) {
                            if ((V & 1) == 0) run_batch_copies<W>(dst, s.lits, e, (u32)lit_src, lit_len, (u32)opos, off, ml, sh->desc);
                            else run_batch_copies_pool<W, kDict>(dst, s.lits, e, (u32)lit_src, lit_len, (u32)opos, off, ml, sh->desc, dw);
                            W::sync();
                        }
                        return (int)(c.op + (long)end - (long)op0);
                    }
                }
            }
            if (W::ballot(bad) == 0) {
                LZB_COUNT_FAST(W::lane() == 0 ? nb : 0);
                if (LZB_DEC_LIT_PF_NEXT) { const long nx = c.lp + (long)tot_adv + (long)tot_ext + 128 * (long)lane; if (lane < LZB_DEC_LIT_PF_LINES && nx < nl) W::prefetch(s.lits + nx); }
                if ((V & 1) == 0) run_batch_copies<W>(dst, s.lits, nb, (u32)lit_src, lit_len, (u32)opos, off, ml, sh->desc);
                else run_batch_copies_pool<W, kDict>(dst, s.lits, nb, (u32)lit_src, lit_len, (u32)opos, off, ml, sh->desc, dw);
                c.fp += nb; c.lp += (long)tot_adv + (long)tot_ext; c.op += (long)tot_out;
                c.p16 += tot16; c.p24 += tot24;
                c.last_off = W::shfl(off, nb - 1);
                continue;
            }
        }
        LZB_COUNT_SLOW(W::lane() == 0 ? nb : 0);
        const int e = lizv1_serial<W, kPartial, kDict>(s, dst, oend, c, nb, oexit, dw);
        if (e < 0) return e;
        if (kPartial && e > 0) return (int)(c.op - (long)op0);
    }
    const long rest = nl - c.lp;
    if (rest < 0 || c.op + rest > oend) return -(int)c.fp - 1;
    if (V != 0 && rest >= (long)kWideMinBytes) lanes_copy_wide<W>(dst + c.op, s.lits + c.lp, (u32)rest, false);
    else lanes_copy<W>(dst + c.op, s.lits + c.lp, (u32)rest);
    W::sync();
    c.op += rest;
    return (int)(c.op - (long)op0);
}

// Token loop of a block the token pre-pass has parsed: lane i of a batch loads record i, one scan gives the output
// positions, the pooled sweeps move the bytes.  Every bound was checked when the records were written.
template <class W> LZ_HD int decode_block_from_records(const Streams& s, u8* dst, u32 op0, const UnitSeq* us, const PoolRun* recs,
                                                       DecWarpShared* sh)
{
    const u32 NL = W::lanes(), lane = W::lane();
    const PoolRun* const mine = recs + us->off;
    u32 op = op0;
    for (u32 t = 0; t < us->nseq; t += NL) {
        const u32 nb = us->nseq - t < NL ? us->nseq - t : NL;
        PoolRun r; r.a = r.b = r.c = r.d = 0;
        if (lane < nb) r = mine[t + lane];
        if (lane < nb && (long)r.a + 2048 < (long)s.nlits) W::prefetch(s.lits + r.a + 2048);
        u32 tot = 0;
        const u32 O = W::excl_scan(r.b + r.d, &tot);
        run_batch_copies_pool<W>(dst, s.lits, nb, r.a, r.b, op + O, r.c, r.d, sh->desc);
        op += tot;
    }
    const u32 rest = s.nlits - us->final_lp;
    if (rest >= kWideMinBytes) lanes_copy_wide<W>(dst + op, s.lits + us->final_lp, rest, false);
    else lanes_copy<W>(dst + op, s.lits + us->final_lp, rest);
    W::sync();
    return (int)(op + rest - op0);
}

// One stream header.  Returns 1 on success, 0 on failure (Lizard_readStream, lizard_decompress.c:72-112).
// `ip` is an offset into the unit.
template <class W> LZ_HD int read_stream(bool huff, const u8* src, long csize, long& ip, u8* scratch, const u8** ptr, u32* len,
                                        DecWarpCore* sh, const u8* expanded = nullptr)
{
    if (!huff) {
        if (ip > csize - 3) return 0;
        *ptr = src + ip + 3;
        *len = rd_le24(src + ip);
        ip += 3 + (long)*len;
        return 1;
    }
    if (ip > csize - 6) return 0;
    const u32 n = rd_le24(src + ip), c = rd_le24(src + ip + 3);
    if (n > kBlockSize || ip + (long)c > csize - 6) return 0;
    if (expanded) { ip += (long)c + 6; *ptr = expanded; *len = n; return 1; }      // done by the pre-pass
    const int r = huf_decompress_lanes<W>(scratch, n, src + ip + 6, c, sh);
    if (r < 0 || (u32)r != n) return 0;
    ip += (long)c + 6;
    *ptr = scratch; *len = n;
    return 1;
}

// Lizard_decompress_safe for one unit; every lane returns the same value.
// kPartial: Lizard_decompress_safe_partial with targetOutputSize = `target` (lib/lizard_decompress.c:272-275).  The unit stops
// after the inner block that brings its output to `target` or beyond (:175 for a raw block, :249), and each block's token
// loop stops at its own start + `target`.  Nothing behind the stopping point is read.  Partial units never use the pre-passes.
// kDict: Lizard_decompress_safe_usingDict with the dictionary `dw` (its reach 0: none).  The Huffman pre-pass may have expanded
// the streams (`up`); the token pre-pass, which checks offsets against the unit start, is never used.
template <class W, int V, bool kPartial = false, bool kDict = false>
LZ_HD int decode_unit(const u8* src, u32 csize_u, u8* dst, u32 cap, u8* scratch, DecWarpShared* sh,
                      const UnitPre* up = nullptr, const u8* arena = nullptr,
                      const UnitSeq* us = nullptr, const PoolRun* recs = nullptr, int target = 0, DictWin dw = DictWin())
{
    const long csize = (long)csize_u;
    if (csize < 1) return 0;
    const int level = src[0];
    if (level < (int)kMinLevel || level > (int)kMaxLevel) return -1;
    const bool lizv1 = level_is_lizv1(level);
    long ip = 1;
    long op = 0;
    while (ip < csize) {
        const long ip0 = ip;                   // 1 for the unit's first inner block
        const u32 hdr = src[ip++];
        if (hdr == kFlagRaw) {
            if (ip > csize - 3) return -1;
            const u32 len = rd_le24(src + ip); ip += 3;
            if (ip + (long)len > csize || op + (long)len > (long)cap) return -1;
            if (V != 0 && len >= kWideMinBytes) lanes_copy_wide<W>(dst + op, src + ip, len, false);
            else lanes_copy<W>(dst + op, src + ip, len);
            W::sync();
            op += len; ip += len;
            if (kPartial && op >= (long)target) break;
            continue;
        }
        if (hdr & kFlagLen) return -1;
        if (ip > csize - 15) return -1;
        {   // lengths stream: always raw, always empty from this encoder, but honour its size field
            const long len_len = (long)rd_le24(src + ip);
            const long len_end = ip + 3 + len_len;
            if (len_end > csize - 3) return -1;
            ip = len_end;
        }
        Streams s;
        s.src_begin = src; s.src_end = src + csize;
        if (!read_stream<W>(hdr & kFlagOff16, src, csize, ip, scratch + 3 * kDecStreamScratch, &s.off16, &s.noff16, sh)) return -1;
        if (!read_stream<W>(hdr & kFlagOff24, src, csize, ip, scratch + 2 * kDecStreamScratch, &s.off24, &s.noff24, sh)) return -1;
        // streams of the unit's first inner block may have been expanded by the pre-pass already
        const bool first = up != nullptr && ip0 == 1;
        const u8* const pre_flags = (first && up->state[kSlotFlags] == kPreDone) ? arena + up->off[kSlotFlags] : nullptr;
        const u8* const pre_lits = (first && up->state[kSlotLiterals] == kPreDone) ? arena + up->off[kSlotLiterals] : nullptr;
        if (!read_stream<W>(hdr & kFlagFlags, src, csize, ip, scratch + 1 * kDecStreamScratch, &s.flags, &s.nflags, sh, pre_flags)) return -1;
        if (!read_stream<W>(hdr & kFlagLiterals, src, csize, ip, scratch, &s.lits, &s.nlits, sh, pre_lits)) return -1;
        if (ip > csize) return -1;
        int res;
        if (!kPartial && !kDict && us != nullptr && ip0 == 1 && us->state == kPreDone) res = decode_block_from_records<W>(s, dst, (u32)op, us, recs, sh);
        else res = lizv1 ? decode_tokens_lizv1<W, V, kPartial, kDict>(s, dst, (u32)op, cap, sh, op + target, dw)
                         : decode_tokens_lz4<W, V, kPartial, kDict>(s, dst, (u32)op, cap, sh, op + target, dw);
        if (res <= 0) return res;
        op += res;
        if (kPartial && op >= (long)target) break;
    }
    return (int)op;
}

}  // namespace lzb
