// host_shim.cpp -- TEST-ONLY host build of the lane-generic codec code.
// Compiled with g++ into lizard_b200/libhostshim.so so the CPU test-suite can pin the
// __host__ __device__ code (entropy_dec.cuh / entropy_enc.cuh / encode_core.cuh, instantiated with the
// one-lane policy HostLanes) against the reference library without a GPU.  Nothing in the product
// path links or loads this file; liblizard_b200.so has no CPU code path.
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>
#define LZB_SHIM_CHECK(cond) do { if (!(cond)) { fprintf(stderr, "host shim check failed: %s (%s:%d)\n", #cond, __FILE__, __LINE__); abort(); } } while (0)
#define LZB_DICT_STATS 1          /* count the dictionary decoder's matches (lzb_dict_stats) */
#define LZB_LP_STATS 1            /* count the lowestPrice parser's rare paths (lzb_lp_stats) */
#define LZB_OPT_STATS 1           /* count the optimal parser's reference behaviours (lzb_opt_stats) */
#define LZB_DICT_ENC_STATS 1      /* count priceFast matches that start in a dictionary (lzb_dict_enc_stats) */
#include "entropy_dec.cuh"
#include "encode_core.cuh"
#include "encode_lp.cuh"
#include "encode_opt.cuh"
#include "decode.cuh"
#include "decode2.cuh"
#include "frame_device.cuh"
#include <stdlib.h>

extern "C" int lzb_host_huf_decompress(unsigned char* dst, unsigned n, const unsigned char* src, unsigned c)
{
    lzb::HufDecScratch* ws = (lzb::HufDecScratch*)malloc(sizeof(lzb::HufDecScratch));
    int r = lzb::huf_decompress_serial(dst, n, src, c, ws);
    free(ws);
    return r;
}

// same choice as the device kernel: packed 17-bit entries when the unit is a single inner block and the table
// would live in shared memory, plain 32-bit entries otherwise (the buffer is big enough for either form)
// tests: 1 = plain 32-bit entries even where the packed form would do (on the device the warps of a CTA that have no
// shared-memory table run small-table levels on the plain form, with its in-entry tags)
static int g_force_plain = 0;
extern "C" void lzb_force_plain_table(int on) { g_force_plain = on; }

static lzb::HashTable make_table(lzb::u32* buf, int n, const lzb::LevelParams& lp)
{
    const lzb::u32 hash_log = lp.hashLog;
    lzb::HashTable T;
    const bool single = (lzb::u32)n <= lzb::kBlockSize;
    if (single && hash_log <= 14 && !g_force_plain) {
        T.t32 = nullptr; T.lo = (lzb::u16*)buf; T.hi = buf + ((size_t)1 << hash_log) / 2;
        T.tag = lzb::enc_tagged(lp) ? (lzb::u8*)buf + lzb::hash_packed_bytes(hash_log, false) : nullptr;   // 3.125 of the buffer's 4 bytes per entry
        T.tagged = 0;
    } else { T.t32 = buf; T.lo = nullptr; T.hi = nullptr; T.tag = nullptr; T.tagged = (single && lzb::enc_tagged_plain(lp)) ? 1u : 0u; }
    return T;
}

unsigned long long lzb::g_lp_stats[lzb::kLpStats];
extern "C" void lzb_lp_stats(unsigned long long* out, int reset)
{
    for (int k = 0; k < lzb::kLpStats; ++k) { if (out) out[k] = lzb::g_lp_stats[k]; if (reset) lzb::g_lp_stats[k] = 0; }
}

// the lowestPrice levels' scratch as the device kernel sets it up: a zero map (epoch 1), and for units of several inner
// blocks a zero big slot
struct LpScratch {
    lzb::LpWork* work; lzb::u8* big;
    explicit LpScratch(int n)
    {
        work = (lzb::LpWork*)malloc(sizeof(lzb::LpWork));
        memset(work->map, 0, sizeof work->map);
        work->huf.seg_count = (lzb::u32 (*)[256])malloc(4 * 256 * sizeof(lzb::u32));
        big = (lzb::u32)n > lzb::kBlockSize ? (lzb::u8*)calloc(1, lzb::kLpBigSlotBytes) : nullptr;
    }
    ~LpScratch()
    {
        if (big) {   // the unit must leave its table zero for the next holder of the slot
            const lzb::u32* t = (const lzb::u32*)big;
            for (size_t i = 0; i < lzb::kLpBigTableBytes / 4; ++i) LZB_SHIM_CHECK(t[i] == 0);
        }
        free(work->huf.seg_count); free(work); free(big);
    }
};

unsigned long long lzb::g_opt_stats[lzb::kOptStats];
extern "C" void lzb_opt_stats(unsigned long long* out, int reset)
{
    for (int k = 0; k < lzb::kOptStats; ++k) { if (out) out[k] = lzb::g_opt_stats[k]; if (reset) lzb::g_opt_stats[k] = 0; }
}

// the optimal levels' scratch as the device kernel sets it up: a zero map (epoch 1), and for units of several inner blocks a
// zero big slot; the tree, opt[] and the token statistics start as garbage, as they do on a warp
struct OptScratch {
    lzb::OptWork* work; lzb::u8* big; lzb::OptStats* stats;
    explicit OptScratch(int n)
    {
        work = (lzb::OptWork*)malloc(sizeof(lzb::OptWork));
        memset(work->lp.chain, 0xA5, sizeof work->lp.chain);
        memset(work->opt, 0x5A, sizeof work->opt);
        memset(work->lp.map, 0, sizeof work->lp.map);
        work->lp.huf.seg_count = (lzb::u32 (*)[256])malloc(4 * 256 * sizeof(lzb::u32));
        stats = (lzb::OptStats*)malloc(sizeof(lzb::OptStats));
        memset(stats, 0x3C, sizeof *stats);
        big = (lzb::u32)n > lzb::kBlockSize ? (lzb::u8*)calloc(1, lzb::kLpBigSlotBytes) : nullptr;
    }
    ~OptScratch()
    {
        if (big) {   // the unit must leave its table zero for the next holder of the slot
            const lzb::u32* t = (const lzb::u32*)big;
            for (size_t i = 0; i < lzb::kLpBigTableBytes / 4; ++i) LZB_SHIM_CHECK(t[i] == 0);
        }
        free(work->lp.huf.seg_count); free(work); free(stats); free(big);
    }
};

extern "C" int lzb_host_compress(const unsigned char* src, int n, unsigned char* dst, int cap, int level)
{
    if (n < 0 || cap < 0) return 0;
    if (level > 49) level = 49;
    if (level < 10) level = 17;
    if (lzb::lp_level(level)) {
        LpScratch sc(n);
        return lzb::encode_unit_lp<lzb::HostLanes>(src, (lzb::u32)n, dst, (lzb::u32)cap, level, sc.work, 1, sc.big);
    }
    if (lzb::opt_level(level)) {
        OptScratch sc(n);
        return lzb::encode_unit_opt<lzb::HostLanes>(src, (lzb::u32)n, dst, (lzb::u32)cap, level, sc.work, 1, sc.big, sc.stats);
    }
    lzb::LevelParams lp = lzb::level_params(level);
    if (lp.parser == lzb::kParserUnsupported) return 0;
    lzb::u32* table = (lzb::u32*)malloc(sizeof(lzb::u32) << lp.hashLog);
    lzb::EncWork* work = (lzb::EncWork*)malloc(sizeof(lzb::EncWork));
    work->huf.seg_count = (lzb::u32 (*)[256])malloc(4 * 256 * sizeof(lzb::u32));
    lzb::HashTable T = make_table(table, n, lp);
    int r = lzb::encode_unit<lzb::HostLanes>(src, (lzb::u32)n, dst, (lzb::u32)cap, level, T, work);
    free(work->huf.seg_count); free(table); free(work);
    return r;
}

// which schedule the decoder entry points below run (bit 0 pooled copies, bit 1 compact chain; device default 3)
static int g_dec_variant = 3;
extern "C" void lzb_set_decode_variant(int v) { g_dec_variant = v; }

// Lizard_decompress_safe through the one-lane instantiation of the device decoder
extern "C" int lzb_host_decompress(const unsigned char* src, int csize, unsigned char* dst, int cap)
{
    if (csize < 1) return 0;
    if (cap < 0) return -1;
    unsigned char* scratch = (unsigned char*)malloc(lzb::kDecScratchPerWarp);
    lzb::DecWarpShared* sh = (lzb::DecWarpShared*)malloc(sizeof(lzb::DecWarpShared));
    sh->big_table = (lzb::u16*)(scratch + 4 * lzb::kDecStreamScratch);
    int r;
    switch (g_dec_variant & 3) {
    case 0: r = lzb::decode_unit<lzb::HostLanes, 0>(src, (lzb::u32)csize, dst, (lzb::u32)cap, scratch, sh); break;
    case 1: r = lzb::decode_unit<lzb::HostLanes, 1>(src, (lzb::u32)csize, dst, (lzb::u32)cap, scratch, sh); break;
    case 2: r = lzb::decode_unit<lzb::HostLanes, 2>(src, (lzb::u32)csize, dst, (lzb::u32)cap, scratch, sh); break;
    default: r = lzb::decode_unit<lzb::HostLanes, 3>(src, (lzb::u32)csize, dst, (lzb::u32)cap, scratch, sh); break;
    }
    free(scratch); free(sh);
    return r;
}

// Lizard_decompress_safe_partial through the one-lane instantiation of the partial decoder (the schedule the device's
// partial kernel runs, without pre-passes)
extern "C" int lzb_host_decompress_partial(const unsigned char* src, int csize, unsigned char* dst, int target, int cap)
{
    if (csize < 1) return 0;
    if (cap < 0) return -1;
    unsigned char* scratch = (unsigned char*)malloc(lzb::kDecScratchPerWarp);
    lzb::DecWarpShared* sh = (lzb::DecWarpShared*)malloc(sizeof(lzb::DecWarpShared));
    sh->big_table = (lzb::u16*)(scratch + 4 * lzb::kDecStreamScratch);
    const int r = lzb::decode_unit<lzb::HostLanes, 3, true>(src, (lzb::u32)csize, dst, (lzb::u32)cap, scratch, sh,
                                                            nullptr, nullptr, nullptr, nullptr, target);
    free(scratch); free(sh);
    return r;
}

// Lizard_decompress_safe_usingDict through the one-lane instantiation of the dictionary decoder (the device's dictionary
// kernel without the Huffman pre-pass): the `avail` bytes in front of dict_end are the dictionary, `reach` how far below the
// unit start a match may start (dict_reach; 0xffffffff = unchecked)
extern "C" int lzb_host_decompress_dict(const unsigned char* src, int csize, unsigned char* dst, int cap,
                                        const unsigned char* dict_end, unsigned avail, unsigned reach)
{
    if (csize < 1) return 0;
    if (cap < 0) return -1;
    unsigned char* scratch = (unsigned char*)malloc(lzb::kDecScratchPerWarp);
    lzb::DecWarpShared* sh = (lzb::DecWarpShared*)malloc(sizeof(lzb::DecWarpShared));
    sh->big_table = (lzb::u16*)(scratch + 4 * lzb::kDecStreamScratch);
    lzb::DictWin dw; dw.end = dict_end; dw.avail = avail; dw.reach = reach;
    const int r = lzb::decode_unit<lzb::HostLanes, 3, false, true>(src, (lzb::u32)csize, dst, (lzb::u32)cap, scratch, sh,
                                                                   nullptr, nullptr, nullptr, nullptr, 0, dw);
    free(scratch); free(sh);
    return r;
}

// matches the dictionary decoders above and below have read from the dictionary alone / across its end since the last reset
extern "C" void lzb_dict_stats(unsigned long long* only, unsigned long long* straddle, int reset)
{
    *only = lzb::g_dict_only; *straddle = lzb::g_dict_straddle;
    if (reset) lzb::g_dict_only = lzb::g_dict_straddle = 0;
}

// The Huffman pre-pass (huf_expand.cuh) as the device runs it, serially: plan the unit's first inner block, expand the
// planned streams into an arena with the same per-segment function, hand the result to the token decoder.
struct HostPre { lzb::UnitPre up; unsigned char* arena; int jobs; };
static void host_prepass(const unsigned char* src, int csize, HostPre* hp, int sabotage)
{
    hp->up.state[0] = hp->up.state[1] = lzb::kPreNone; hp->up.off[0] = hp->up.off[1] = 0;
    hp->arena = (unsigned char*)malloc(2 * (size_t)lzb::pre_slot_bytes(lzb::kBlockSize));
    lzb::HufJob jobs[2];
    const lzb::u32 nj = lzb::plan_unit(src, (lzb::u32)csize, jobs);
    hp->jobs = (int)nj;
    lzb::HufJobScratch* ws = (lzb::HufJobScratch*)malloc(sizeof(lzb::HufJobScratch));
    lzb::HufCompact* table = (lzb::HufCompact*)malloc(sizeof(lzb::HufCompact));
    size_t cursor = 0;
    for (lzb::u32 i = 0; i < nj; ++i) {
        lzb::HufJob& j = jobs[i];
        j.dst = cursor; cursor += (size_t)lzb::pre_slot_bytes(j.n);
        lzb::u32 h = 0;
        bool ok = lzb::huf_job_prepare(src + j.src, j.c, j.n, table, ws, &h);
        lzb::u32 ring[lzb::kHufRingWords];
        for (lzb::u32 k = 0; ok && k < 4; ++k)
            ok = lzb::huf_job_segment(hp->arena + j.dst, j.n, src + j.src + h, j.c - h, k, *table, ring);
        if (sabotage && ok) memset(hp->arena + j.dst, 0x5A, j.n);     // tests: proves the token decoder reads the arena
        hp->up.off[j.slot] = j.dst;
        hp->up.state[j.slot] = ok ? lzb::kPreDone : lzb::kPreNone;
    }
    free(ws); free(table);
}
// HufCompact (two-level table of the Huffman pre-pass) against the reference-layout table built from the same weights:
// number of indices (all 1 << tl, three fillings of the bits below the index) whose lookup differs.
extern "C" int lzb_huf_compact_check(const unsigned char* weights, int nsym, int tl)
{
    lzb::u32 rank_a[lzb::kHufTableLogMax + 1] = {0}, rank_b[lzb::kHufTableLogMax + 1] = {0};
    for (int s = 0; s < nsym; ++s) { rank_a[weights[s]]++; rank_b[weights[s]]++; }
    lzb::u16* full = (lzb::u16*)malloc(sizeof(lzb::u16) << tl);
    lzb::HufCompact* c = (lzb::HufCompact*)malloc(sizeof(lzb::HufCompact));
    lzb::huf_fill_dtable(full, weights, rank_a, (lzb::u32)nsym, (lzb::u32)tl);
    lzb::huf_fill_compact(c, weights, rank_b, (lzb::u32)nsym, (lzb::u32)tl);
    lzb::HufFull f; f.t = full; f.down = 32u - (lzb::u32)tl;
    int bad = 0;
    const lzb::u32 low[3] = { 0u, 0xFFFFFFFFu, 0x5A5A5A5Au };
    for (lzb::u32 idx = 0; idx < (1u << tl); ++idx)
        for (int k = 0; k < 3; ++k) {
            const lzb::u32 hi = (idx << (32 - tl)) | (low[k] >> tl);
            if (f.look(hi) != lzb::huf_view(c).look(hi)) ++bad;
        }
    free(full); free(c);
    return bad;
}

// bit 0 of `mode`: 32 emulated lanes instead of one; bit 1: overwrite the expanded streams (negative control);
// bit 2: also run the token pre-pass (one-lane parse of the first inner block into sequence records).
// *jobs_done = streams the Huffman pre-pass expanded + 16 if the token pre-pass parsed the block.
extern "C" int lzb_decompress_with_prepass(const unsigned char* src, int csize, unsigned char* dst, int cap, int mode, int* jobs_done);

extern "C" void lzb_host_token_stats(unsigned long long* fast, unsigned long long* slow)
{
#if defined(LZB_STATS)
    *fast = lzb::g_tok_fast; *slow = lzb::g_tok_slow;
#else
    *fast = 0; *slow = 0;
#endif
}

// =====================================================================================================
// 32-lane warp emulator (TEST-ONLY).  The lane-parallel code paths (ballot / shuffle / match_any based)
// only exist for 32 lanes, and there is no GPU in the build container, so the CPU suite runs them on 32
// cooperative coroutines (ucontext): every collective is a rendezvous of all lanes, exactly the
// warp-synchronous model the kernels are written in.  Shared data (hash table, streams) is ordinary memory.
// =====================================================================================================
#include <ucontext.h>
#include <vector>

namespace emu {
constexpr int kLanes = 32;
struct Warp {
    ucontext_t sched;
    ucontext_t ctx[kLanes];
    std::vector<char> stack[kLanes];
    int cur = 0;
    bool done[kLanes];
    unsigned long long slot[kLanes];
    int arrived = 0, readers = 0;
    unsigned gen = 0, gen2 = 0;
    void (*body)(void*) = nullptr;
    void* arg = nullptr;
};
static Warp* g = nullptr;
static int g_order = 0;          // 0 forward, 1 reverse, 2 shuffled per round

static void yield() { swapcontext(&g->ctx[g->cur], &g->sched); }

// all lanes deposit a value; returns when every lane has deposited; out[] is a private copy
static void exchange(unsigned long long v, unsigned long long* out)
{
    Warp* w = g;
    const int me = w->cur;
    w->slot[me] = v;
    {   unsigned my = w->gen;
        if (++w->arrived == kLanes) { w->arrived = 0; w->gen++; }
        else while (w->gen == my) yield(); }
    for (int i = 0; i < kLanes; ++i) out[i] = w->slot[i];
    {   unsigned my = w->gen2;
        if (++w->readers == kLanes) { w->readers = 0; w->gen2++; }
        else while (w->gen2 == my) yield(); }
}

static void trampoline()
{
    Warp* w = g;
    w->body(w->arg);
    w->done[w->cur] = true;
    swapcontext(&w->ctx[w->cur], &w->sched);
}

static void run(void (*body)(void*), void* arg)
{
    Warp w;
    g = &w;
    w.body = body; w.arg = arg;
    for (int i = 0; i < kLanes; ++i) {
        w.done[i] = false;
        w.stack[i].resize(256 * 1024);
        getcontext(&w.ctx[i]);
        w.ctx[i].uc_stack.ss_sp = w.stack[i].data();
        w.ctx[i].uc_stack.ss_size = w.stack[i].size();
        w.ctx[i].uc_link = &w.sched;
        makecontext(&w.ctx[i], (void (*)())trampoline, 0);
    }
    unsigned rng = 12345u;
    for (;;) {
        bool any = false;
        // lane order inside a round: forward, reverse, or shuffled -- code that is missing a barrier between a write
        // by one lane and a read by another only fails under SOME orders, so the tests run all three
        int order[kLanes];
        for (int i = 0; i < kLanes; ++i) order[i] = g_order == 1 ? kLanes - 1 - i : i;
        if (g_order == 2)
            for (int i = kLanes - 1; i > 0; --i) {
                rng = rng * 1664525u + 1013904223u;
                const int j = (int)((rng >> 8) % (unsigned)(i + 1));
                const int t = order[i]; order[i] = order[j]; order[j] = t;
            }
        for (int n = 0; n < kLanes; ++n) {
            const int i = order[n];
            if (w.done[i]) continue;
            any = true;
            w.cur = i;
            swapcontext(&w.sched, &w.ctx[i]);
        }
        if (!any) break;
    }
    g = nullptr;
}
}  // namespace emu

extern "C" void lzb_emu_lane_order(int o) { emu::g_order = o; }

struct EmuLanes {
    static constexpr bool kDevice = false;
    static constexpr lzb::u32 kLanes = emu::kLanes;
    static lzb::u32 lane() { return (lzb::u32)emu::g->cur; }
    static lzb::u32 lanes() { return emu::kLanes; }
    static void sync() { unsigned long long t[emu::kLanes]; emu::exchange(0, t); }
    static int bcast(int v) { unsigned long long t[emu::kLanes]; emu::exchange((unsigned long long)(unsigned)v, t); return (int)(unsigned)t[0]; }
    static lzb::u32 sum(lzb::u32 v) { unsigned long long t[emu::kLanes]; emu::exchange(v, t); lzb::u32 s = 0; for (auto x : t) s += (lzb::u32)x; return s; }
    static lzb::u32 excl_scan(lzb::u32 v, lzb::u32* total)
    {
        unsigned long long t[emu::kLanes]; emu::exchange(v, t);
        lzb::u32 pre = 0, tot = 0;
        for (int i = 0; i < emu::kLanes; ++i) { if (i < emu::g->cur) pre += (lzb::u32)t[i]; tot += (lzb::u32)t[i]; }
        *total = tot; return pre;
    }
    static lzb::u32 ballot(bool p)
    {
        unsigned long long t[emu::kLanes]; emu::exchange(p ? 1 : 0, t);
        lzb::u32 m = 0; for (int i = 0; i < emu::kLanes; ++i) if (t[i]) m |= 1u << i; return m;
    }
    static lzb::u32 shfl(lzb::u32 v, lzb::u32 src)
    {
        unsigned long long t[emu::kLanes]; emu::exchange(v, t); return (lzb::u32)t[src & 31];
    }
    static void prefetch(const void*) {}
    static lzb::u32 red_or(lzb::u32 v)
    {
        unsigned long long t[emu::kLanes]; emu::exchange(v, t);
        lzb::u32 m = 0; for (int i = 0; i < emu::kLanes; ++i) m |= (lzb::u32)t[i]; return m;
    }
    static lzb::u32 match_any(lzb::u32 v)
    {
        unsigned long long t[emu::kLanes]; emu::exchange(v, t);
        lzb::u32 m = 0; for (int i = 0; i < emu::kLanes; ++i) if ((lzb::u32)t[i] == v) m |= 1u << i; return m;
    }
};

struct EmuCompressArgs { const unsigned char* src; int n; unsigned char* dst; int cap; int level; lzb::HashTable T; lzb::EncWork* work; int result; };
static void emu_compress_body(void* p)
{
    EmuCompressArgs* a = (EmuCompressArgs*)p;
    int r = lzb::encode_unit<EmuLanes>(a->src, (lzb::u32)a->n, a->dst, (lzb::u32)a->cap, a->level, a->T, a->work);
    if (EmuLanes::lane() == 0) a->result = r;
}

struct EmuLpArgs { const unsigned char* src; int n; unsigned char* dst; int cap; int level; LpScratch* sc; int result; };
static void emu_lp_body(void* p)
{
    EmuLpArgs* a = (EmuLpArgs*)p;
    int r = lzb::encode_unit_lp<EmuLanes>(a->src, (lzb::u32)a->n, a->dst, (lzb::u32)a->cap, a->level, a->sc->work, 1, a->sc->big);
    if (EmuLanes::lane() == 0) a->result = r;
}

struct EmuOptArgs { const unsigned char* src; int n; unsigned char* dst; int cap; int level; lzb::OptWork* work; lzb::u8* big;
                    lzb::OptStats* stats; unsigned epoch; int result; };
static void emu_opt_body(void* p)
{
    EmuOptArgs* a = (EmuOptArgs*)p;
    int r = lzb::encode_unit_opt<EmuLanes>(a->src, (lzb::u32)a->n, a->dst, (lzb::u32)a->cap, a->level, a->work, a->epoch, a->big, a->stats);
    if (EmuLanes::lane() == 0) a->result = r;
}

// Lizard_compress through the 32-lane emulation of the device code path
extern "C" int lzb_emu_compress(const unsigned char* src, int n, unsigned char* dst, int cap, int level)
{
    if (n < 0 || cap < 0) return 0;
    if (level > 49) level = 49;
    if (level < 10) level = 17;
    if (lzb::lp_level(level)) {
        LpScratch sc(n);
        EmuLpArgs a = { src, n, dst, cap, level, &sc, 0 };
        emu::run(emu_lp_body, &a);
        return a.result;
    }
    if (lzb::opt_level(level)) {
        OptScratch sc(n);
        EmuOptArgs a = { src, n, dst, cap, level, sc.work, sc.big, sc.stats, 1, 0 };
        emu::run(emu_opt_body, &a);
        return a.result;
    }
    lzb::LevelParams lp = lzb::level_params(level);
    if (lp.parser == lzb::kParserUnsupported) return 0;
    EmuCompressArgs a;
    a.src = src; a.n = n; a.dst = dst; a.cap = cap; a.level = level; a.result = 0;
    lzb::u32* table = (lzb::u32*)malloc(sizeof(lzb::u32) << lp.hashLog);
    a.T = make_table(table, n, lp);
    a.work = (lzb::EncWork*)malloc(sizeof(lzb::EncWork));
    a.work->huf.seg_count = (lzb::u32 (*)[256])malloc(4 * 256 * sizeof(lzb::u32));
    emu::run(emu_compress_body, &a);
    free(a.work->huf.seg_count); free(table); free(a.work);
    return a.result;
}

// ---- lowestPrice on persistent, poisoned scratch ------------------------------------------------------------------------
// A device warp does not get clean scratch per unit: its LpWork keeps whatever the previous unit (of this launch, or of
// another encoder that shares the workspace) left, its map holds entries of earlier epochs, and a big slot's chain is
// never cleared.  These entry points keep one such scratch across calls, so the tests can run sequences of units on it.
struct LpPersist { lzb::LpWork* work; lzb::u8* big; lzb::u32 (*seg)[256]; };
static lzb::u32 lp_rand(lzb::u32& s) { s = s * 1664525u + 1013904223u; return s ^ (s >> 15); }
static void lp_fill(void* p, size_t n, lzb::u32 seed)
{
    lzb::u32* w = (lzb::u32*)p;
    for (size_t i = 0; i < n / 4; ++i) w[i] = lp_rand(seed);
}
// garbage in the sequence list, chain, streams and Huffman scratch; a big slot whose table is zero and whose chain is garbage
extern "C" void* lzb_lp_scratch_new(unsigned seed)
{
    LpPersist* sc = (LpPersist*)malloc(sizeof(LpPersist));
    sc->work = (lzb::LpWork*)malloc(sizeof(lzb::LpWork));
    sc->seg = (lzb::u32 (*)[256])malloc(4 * 256 * sizeof(lzb::u32));
    lp_fill(sc->work, offsetof(lzb::LpWork, map), seed);
    lp_fill(sc->seg, 4 * 256 * sizeof(lzb::u32), seed + 1);
    sc->work->huf.seg_count = sc->seg;
    memset(sc->work->map, 0, sizeof sc->work->map);
    sc->big = (lzb::u8*)calloc(1, lzb::kLpBigSlotBytes);
    lp_fill(sc->big + lzb::kLpBigTableBytes, lzb::kLpBigChainBytes, seed + 2);
    return sc;
}
extern "C" void lzb_lp_scratch_free(void* p)
{
    LpPersist* sc = (LpPersist*)p;
    free(sc->seg); free(sc->work); free(sc->big); free(sc);
}
// A map as a warp may find it before a unit at `epoch`, filled with entries of other epochs (0, epoch - 1, epoch + 1 and
// kLpEpochMax, in turn):
//  * every slot holds a stale bucket whose home it is (at `hash_log`), with a random position;
//  * with `src`, the stale entries of the next unit's own buckets, placed where the map's probing would find them: for each
//    position p that the unit inserts, bucket(p) -> p - k (k = 1..7).  Taken for a current entry, such an entry lies within
//    8 bytes below p, so Lizard_Insert's "replace unless within 8" rule keeps it instead of p, and the parse loses matches.
// A map that counts every slot of another epoch as empty gives the unit the reference's bytes.
static void poison_map(lzb::u64* const map, unsigned epoch, unsigned hash_log, unsigned seed, const unsigned char* src, int n,
                       unsigned mls)
{
    const lzb::u32 shift = hash_log - lzb::kLpMapLog, mx = lzb::kLpEpochMax, mask = (1u << lzb::kLpMapLog) - 1;
    lzb::u32 other[4] = { 0u, (epoch - 1) & mx, (epoch + 1) & mx, mx };
    for (lzb::u32& e : other)
        if (e == epoch) e = (epoch + 2) & mx;          // epoch 1: epoch - 1 is 0; kLpEpochMax: epoch + 1 wraps to 0
    for (lzb::u32 i = 0; i <= mask; ++i) {
        const lzb::u32 bucket = (i << shift) | (lp_rand(seed) & ((1u << shift) - 1));
        const lzb::u32 pos1 = 1 + lp_rand(seed) % lzb::kBlockSize;
        map[i] = (lzb::u64)other[i & 3] << 41 | (lzb::u64)bucket << 18 | pos1;
    }
    if (!src || n <= (int)lzb::kMfLimit) return;
    std::vector<unsigned char> placed(mask + 1, 0);
    for (lzb::u32 q = 1; q < (lzb::u32)n - lzb::kMfLimit && q < lzb::kBlockSize; ++q) {
        const lzb::u32 h = lzb::hc_hash(src + q, hash_log, mls);
        lzb::u32 i = h >> shift;
        bool dup = false;
        for (; placed[i]; i = (i + 1) & mask)
            if ((lzb::u32)(map[i] >> 18 & 0x7FFFFFu) == h) { dup = true; break; }
        if (dup) continue;
        const lzb::u32 k = 1 + lp_rand(seed) % 7, stale = q > k ? q - k : 0;
        map[i] = (lzb::u64)other[q & 3] << 41 | (lzb::u64)h << 18 | (stale + 1);
        placed[i] = 1;
    }
}
extern "C" void lzb_lp_scratch_poison_map(void* p, unsigned epoch, unsigned hash_log, unsigned seed,
                                          const unsigned char* src, int n, unsigned mls)
{
    poison_map(((LpPersist*)p)->work->map, epoch, hash_log, seed, src, n, mls);
}
// the kernel's rule when a warp's epoch reaches kLpEpochMax: clear the map, go on at epoch 1
extern "C" void lzb_lp_scratch_clear_map(void* p) { memset(((LpPersist*)p)->work->map, 0, sizeof ((LpPersist*)p)->work->map); }
// 1 if the big slot's table is zero, as every unit must leave it
extern "C" int lzb_lp_scratch_big_clean(void* p)
{
    const lzb::u32* t = (const lzb::u32*)((LpPersist*)p)->big;
    for (size_t i = 0; i < lzb::kLpBigTableBytes / 4; ++i) if (t[i]) return 0;
    return 1;
}

struct EmuLpOnArgs { const unsigned char* src; int n; unsigned char* dst; int cap; int level; LpPersist* sc; unsigned epoch; int result; };
static void emu_lp_on_body(void* p)
{
    EmuLpOnArgs* a = (EmuLpOnArgs*)p;
    int r = lzb::encode_unit_lp<EmuLanes>(a->src, (lzb::u32)a->n, a->dst, (lzb::u32)a->cap, a->level, a->sc->work, a->epoch, a->sc->big);
    if (EmuLanes::lane() == 0) a->result = r;
}
// one unit at a lowestPrice level on the persistent scratch under `epoch` (1 .. kLpEpochMax); emu = 32 emulated lanes
extern "C" int lzb_lp_compress_on(void* p, const unsigned char* src, int n, unsigned char* dst, int cap, int level,
                                  unsigned epoch, int emu)
{
    LpPersist* sc = (LpPersist*)p;
    if (n < 0 || cap < 0 || !lzb::lp_level(level) || epoch < 1 || epoch > lzb::kLpEpochMax) return 0;
    if (!emu) return lzb::encode_unit_lp<lzb::HostLanes>(src, (lzb::u32)n, dst, (lzb::u32)cap, level, sc->work, epoch, sc->big);
    EmuLpOnArgs a = { src, n, dst, cap, level, sc, epoch, 0 };
    emu::run(emu_lp_on_body, &a);
    return a.result;
}

// ---- the optimal parser on persistent, poisoned scratch -------------------------------------------------------------
// As above for levels 18, 19 and 39: the warp's tree, opt[], match list, sequence list, streams and token statistics keep
// garbage (or the previous unit's contents), its map entries of other epochs, its big slot a zero table.
struct OptPersist { lzb::OptWork* work; lzb::u8* big; lzb::u32 (*seg)[256]; lzb::OptStats* stats; };
extern "C" void* lzb_opt_scratch_new(unsigned seed)
{
    OptPersist* sc = (OptPersist*)malloc(sizeof(OptPersist));
    sc->work = (lzb::OptWork*)malloc(sizeof(lzb::OptWork));
    sc->seg = (lzb::u32 (*)[256])malloc(4 * 256 * sizeof(lzb::u32));
    sc->stats = (lzb::OptStats*)malloc(sizeof(lzb::OptStats));
    lp_fill(sc->work, sizeof(lzb::OptWork), seed);
    lp_fill(sc->seg, 4 * 256 * sizeof(lzb::u32), seed + 1);
    lp_fill(sc->stats, sizeof(lzb::OptStats), seed + 2);
    sc->work->lp.huf.seg_count = sc->seg;
    memset(sc->work->lp.map, 0, sizeof sc->work->lp.map);
    sc->big = (lzb::u8*)calloc(1, lzb::kLpBigSlotBytes);
    lp_fill(sc->big + lzb::kLpBigTableBytes, lzb::kLpBigChainBytes, seed + 3);
    return sc;
}
extern "C" void lzb_opt_scratch_free(void* p)
{
    OptPersist* sc = (OptPersist*)p;
    free(sc->seg); free(sc->work); free(sc->stats); free(sc->big); free(sc);
}
// garbage again in the tree (every 16th node a (U32)-1 link), opt[] and the match list, as another launch may leave them
extern "C" void lzb_opt_scratch_poison(void* p, unsigned seed)
{
    OptPersist* sc = (OptPersist*)p;
    lp_fill(sc->work->lp.chain, sizeof sc->work->lp.chain, seed);
    for (size_t i = 0; i < sizeof sc->work->lp.chain / 4; i += 16) sc->work->lp.chain[i] = lzb::kOptNoLink;
    lp_fill(sc->work->opt, sizeof sc->work->opt, seed + 1);
    lp_fill(sc->work->match, sizeof sc->work->match, seed + 2);
}
// the map poisoned as lzb_lp_scratch_poison_map does it (hash4 buckets)
extern "C" void lzb_opt_scratch_poison_map(void* p, unsigned epoch, unsigned hash_log, unsigned seed, const unsigned char* src, int n)
{
    poison_map(((OptPersist*)p)->work->lp.map, epoch, hash_log, seed, src, n, 4);
}
extern "C" void lzb_opt_scratch_clear_map(void* p) { memset(((OptPersist*)p)->work->lp.map, 0, sizeof ((OptPersist*)p)->work->lp.map); }
extern "C" int lzb_opt_scratch_big_clean(void* p)
{
    const lzb::u32* t = (const lzb::u32*)((OptPersist*)p)->big;
    for (size_t i = 0; i < lzb::kLpBigTableBytes / 4; ++i) if (t[i]) return 0;
    return 1;
}
// one unit at level 18, 19 or 39 on the persistent scratch under `epoch` (1 .. kLpEpochMax); emu = 32 emulated lanes
extern "C" int lzb_opt_compress_on(void* p, const unsigned char* src, int n, unsigned char* dst, int cap, int level,
                                   unsigned epoch, int emu)
{
    OptPersist* sc = (OptPersist*)p;
    if (n < 0 || cap < 0 || !lzb::opt_level(level) || epoch < 1 || epoch > lzb::kLpEpochMax) return 0;
    if (!emu) return lzb::encode_unit_opt<lzb::HostLanes>(src, (lzb::u32)n, dst, (lzb::u32)cap, level, sc->work, epoch, sc->big, sc->stats);
    EmuOptArgs a = { src, n, dst, cap, level, sc->work, sc->big, sc->stats, epoch, 0 };
    emu::run(emu_opt_body, &a);
    return a.result;
}

unsigned long long lzb::g_lp_probe[lzb::kLpProbeStats];
// longest probe run, slots probed past the home slot, probes that wrapped past the map's last slot
extern "C" void lzb_lp_probe_stats(unsigned long long* out, int reset)
{
    for (int k = 0; k < lzb::kLpProbeStats; ++k) { if (out) out[k] = lzb::g_lp_probe[k]; if (reset) lzb::g_lp_probe[k] = 0; }
}

struct EmuDecompressArgs { const unsigned char* src; int csize; unsigned char* dst; int cap; unsigned char* scratch; lzb::DecWarpShared* sh; int result;
                           const lzb::UnitPre* up; const unsigned char* arena; const lzb::UnitSeq* us; const lzb::PoolRun* recs; };
static void emu_decompress_body(void* p)
{
    EmuDecompressArgs* a = (EmuDecompressArgs*)p;
    int r;
    switch (g_dec_variant & 3) {
    case 0: r = lzb::decode_unit<EmuLanes, 0>(a->src, (lzb::u32)a->csize, a->dst, (lzb::u32)a->cap, a->scratch, a->sh, a->up, a->arena, a->us, a->recs); break;
    case 1: r = lzb::decode_unit<EmuLanes, 1>(a->src, (lzb::u32)a->csize, a->dst, (lzb::u32)a->cap, a->scratch, a->sh, a->up, a->arena, a->us, a->recs); break;
    case 2: r = lzb::decode_unit<EmuLanes, 2>(a->src, (lzb::u32)a->csize, a->dst, (lzb::u32)a->cap, a->scratch, a->sh, a->up, a->arena, a->us, a->recs); break;
    default: r = lzb::decode_unit<EmuLanes, 3>(a->src, (lzb::u32)a->csize, a->dst, (lzb::u32)a->cap, a->scratch, a->sh, a->up, a->arena, a->us, a->recs); break;
    }
    if (EmuLanes::lane() == 0) a->result = r;
}

// Lizard_decompress_safe through the 32-lane emulation of the device code path
extern "C" int lzb_emu_decompress(const unsigned char* src, int csize, unsigned char* dst, int cap)
{
    if (csize < 1) return 0;
    if (cap < 0) return -1;
    EmuDecompressArgs a;
    a.src = src; a.csize = csize; a.dst = dst; a.cap = cap; a.result = -1; a.up = nullptr; a.arena = nullptr; a.us = nullptr; a.recs = nullptr;
    a.scratch = (unsigned char*)malloc(lzb::kDecScratchPerWarp);
    a.sh = (lzb::DecWarpShared*)malloc(sizeof(lzb::DecWarpShared));
    a.sh->big_table = (lzb::u16*)(a.scratch + 4 * lzb::kDecStreamScratch);
    emu::run(emu_decompress_body, &a);
    free(a.scratch); free(a.sh);
    return a.result;
}

struct EmuPartialArgs { const unsigned char* src; int csize; unsigned char* dst; int target; int cap; unsigned char* scratch;
                        lzb::DecWarpShared* sh; int result; };
static void emu_partial_body(void* p)
{
    EmuPartialArgs* a = (EmuPartialArgs*)p;
    const int r = lzb::decode_unit<EmuLanes, 3, true>(a->src, (lzb::u32)a->csize, a->dst, (lzb::u32)a->cap, a->scratch, a->sh,
                                                      nullptr, nullptr, nullptr, nullptr, a->target);
    if (EmuLanes::lane() == 0) a->result = r;
}

// Lizard_decompress_safe_partial through the 32-lane emulation of the device's partial kernel
extern "C" int lzb_emu_decompress_partial(const unsigned char* src, int csize, unsigned char* dst, int target, int cap)
{
    if (csize < 1) return 0;
    if (cap < 0) return -1;
    EmuPartialArgs a;
    a.src = src; a.csize = csize; a.dst = dst; a.target = target; a.cap = cap; a.result = -1;
    a.scratch = (unsigned char*)malloc(lzb::kDecScratchPerWarp);
    a.sh = (lzb::DecWarpShared*)malloc(sizeof(lzb::DecWarpShared));
    a.sh->big_table = (lzb::u16*)(a.scratch + 4 * lzb::kDecStreamScratch);
    emu::run(emu_partial_body, &a);
    free(a.scratch); free(a.sh);
    return a.result;
}

struct EmuDictArgs { const unsigned char* src; int csize; unsigned char* dst; int cap; lzb::DictWin dw; unsigned char* scratch;
                     lzb::DecWarpShared* sh; int result; };
static void emu_dict_body(void* p)
{
    EmuDictArgs* a = (EmuDictArgs*)p;
    const int r = lzb::decode_unit<EmuLanes, 3, false, true>(a->src, (lzb::u32)a->csize, a->dst, (lzb::u32)a->cap, a->scratch, a->sh,
                                                             nullptr, nullptr, nullptr, nullptr, 0, a->dw);
    if (EmuLanes::lane() == 0) a->result = r;
}

// Lizard_decompress_safe_usingDict through the 32-lane emulation of the device's dictionary kernel (arguments as
// lzb_host_decompress_dict)
extern "C" int lzb_emu_decompress_dict(const unsigned char* src, int csize, unsigned char* dst, int cap,
                                       const unsigned char* dict_end, unsigned avail, unsigned reach)
{
    if (csize < 1) return 0;
    if (cap < 0) return -1;
    EmuDictArgs a;
    a.src = src; a.csize = csize; a.dst = dst; a.cap = cap; a.result = -1;
    a.dw.end = dict_end; a.dw.avail = avail; a.dw.reach = reach;
    a.scratch = (unsigned char*)malloc(lzb::kDecScratchPerWarp);
    a.sh = (lzb::DecWarpShared*)malloc(sizeof(lzb::DecWarpShared));
    a.sh->big_table = (lzb::u16*)(a.scratch + 4 * lzb::kDecStreamScratch);
    emu::run(emu_dict_body, &a);
    free(a.scratch); free(a.sh);
    return a.result;
}

extern "C" int lzb_decompress_with_prepass(const unsigned char* src, int csize, unsigned char* dst, int cap, int mode, int* jobs_done)
{
    if (csize < 1) return 0;
    if (cap < 0) return -1;
    HostPre hp;
    host_prepass(src, csize, &hp, mode & 2);
    if (jobs_done) *jobs_done = (hp.up.state[0] == lzb::kPreDone) + (hp.up.state[1] == lzb::kPreDone);
    lzb::UnitSeq us; us.off = 0; us.nseq = 0; us.state = lzb::kPreNone; us.final_lp = us.final_op = 0;
    lzb::PoolRun* recs = nullptr;
    if (mode & 4) {
        lzb::Streams st; int lizv1 = 0;
        if (lzb::locate_first_block(src, (lzb::u32)csize, &hp.up, hp.arena, &st, &lizv1)) {
            recs = (lzb::PoolRun*)malloc(sizeof(lzb::PoolRun) * (st.nflags + 1));
            const bool ok = lizv1 ? lzb::parse_block_lizv1(st, 0, (lzb::u32)cap, recs, &us.final_lp, &us.final_op)
                                  : lzb::parse_block_lz4(st, 0, (lzb::u32)cap, recs, &us.final_lp, &us.final_op);
            if (ok) { us.nseq = st.nflags; us.state = lzb::kPreDone; if (jobs_done) *jobs_done += 16; }
        }
    }
    unsigned char* scratch = (unsigned char*)malloc(lzb::kDecScratchPerWarp);
    lzb::DecWarpShared* sh = (lzb::DecWarpShared*)malloc(sizeof(lzb::DecWarpShared));
    sh->big_table = (lzb::u16*)(scratch + 4 * lzb::kDecStreamScratch);
    int r;
    if (mode & 1) {
        EmuDecompressArgs a;
        a.src = src; a.csize = csize; a.dst = dst; a.cap = cap; a.result = -1; a.up = &hp.up; a.arena = hp.arena;
        a.us = (mode & 4) ? &us : nullptr; a.recs = recs;
        a.scratch = scratch; a.sh = sh;
        emu::run(emu_decompress_body, &a);
        r = a.result;
    } else r = lzb::decode_unit<lzb::HostLanes, 3>(src, (lzb::u32)csize, dst, (lzb::u32)cap, scratch, sh, &hp.up, hp.arena,
                                                   (mode & 4) ? &us : nullptr, recs);
    free(scratch); free(sh); free(hp.arena); free(recs);
    return r;
}


// ---- second-generation decoder (decode2.cuh): parser + copier through the in-line sink -------------------------------
// mode bit 0: 32 emulated lanes instead of one.  `span` = most literals-stream bytes per published batch (the device uses
// ~4 KB; tests also run tiny values to exercise the prefix / split paths).  `dst` may be unaligned: the copier works in the
// aligned space of dst & ~15 and must not touch a byte outside [dst, dst + result).
template <class W> static int decode2_run(const unsigned char* src, int csize, unsigned char* dst, int cap, unsigned span,
                                          unsigned char* scratch, lzb::DecWarpCore* core, lzb::CopyShared* cs)
{
    lzb::InlineSink<W> sk;
    sk.cs = cs; sk.lits.p = nullptr; sk.nrec_total = 0; sk.span_limit = span; sk.out_pos = 0;
    sk.st.unit_lo = (lzb::u32)((size_t)dst & 15);
    sk.st.dst_al = dst - sk.st.unit_lo;
    sk.resync(sk.st.unit_lo);
    return lzb::decode_unit2<W>(src, (lzb::u32)csize, dst, (lzb::u32)cap, scratch, core, sk);
}
struct EmuDecode2Args { const unsigned char* src; int csize; unsigned char* dst; int cap; unsigned span; unsigned char* scratch;
                        lzb::DecWarpCore* core; lzb::CopyShared* cs; int result; };
static void emu_decode2_body(void* p)
{
    EmuDecode2Args* a = (EmuDecode2Args*)p;
    const int r = decode2_run<EmuLanes>(a->src, a->csize, a->dst, a->cap, a->span, a->scratch, a->core, a->cs);
    if (EmuLanes::lane() == 0) a->result = r;
}
extern "C" int lzb_host_decompress2(const unsigned char* src, int csize, unsigned char* dst, int cap, int mode, unsigned span)
{
    if (csize < 1) return 0;
    if (cap < 0) return -1;
    unsigned char* scratch = (unsigned char*)malloc(lzb::kDecScratchPerWarp);
    lzb::DecWarpCore* core = (lzb::DecWarpCore*)malloc(sizeof(lzb::DecWarpCore));
    lzb::CopyShared* cs = (lzb::CopyShared*)malloc(sizeof(lzb::CopyShared));
    memset(cs, 0xA5, sizeof *cs);
    core->big_table = (lzb::u16*)(scratch + 4 * lzb::kDecStreamScratch);
    int r;
    if (mode & 1) {
        EmuDecode2Args a; a.src = src; a.csize = csize; a.dst = dst; a.cap = cap; a.span = span; a.scratch = scratch; a.core = core;
        a.cs = cs; a.result = -1;
        emu::run(emu_decode2_body, &a);
        r = a.result;
    } else r = decode2_run<lzb::HostLanes>(src, csize, dst, cap, span, scratch, core, cs);
    free(scratch); free(core); free(cs);
    return r;
}

// ---- compression against a loaded dictionary (hashChain and priceFast levels) ------------------------------------------------------
// Lizard_createStream(level) + Lizard_loadDict(dict, dict_size) + Lizard_compress_continue(src, dst, n, cap), one lane or the
// 32-lane emulator: emu bit 0 runs the unit's parse on the emulator, bit 1 the dictionary's load too (the load is the
// emulator's slowest part and the same code for every unit).  dict + dict_size == src is the prefix layout.
// The device's scratch is not clean: the unit's chain and the loaded chain start as garbage, the overlay as garbage that the
// unit clears.  Levels without a dictionary path return 0.
unsigned long long lzb::g_dict_enc_stats[lzb::kDictEncStats];
extern "C" void lzb_dict_enc_stats(unsigned long long* out, int reset)
{
    for (int k = 0; k < lzb::kDictEncStats; ++k) { if (out) out[k] = lzb::g_dict_enc_stats[k]; if (reset) lzb::g_dict_enc_stats[k] = 0; }
}
struct DictCompressArgs { const unsigned char* src; int n; unsigned char* dst; int cap; int level; const unsigned char* dict;
                          lzb::u32 dsize; lzb::u32* ov; lzb::u32* sh; lzb::u16* dchain; lzb::EncWork* work; int emu_load; int result; };
template <class W> static void dict_compress_body(DictCompressArgs* a)
{
    const lzb::LevelParams lp = lzb::level_params(a->level);
    lzb::DictTable T = lzb::dict_view(a->src, (lzb::u32)a->n, a->dict, a->dsize);
    if (a->emu_load || W::kLanes == 1) lzb::dict_load<W>(a->dict, a->dsize >= 8 ? a->dsize - 7 : 0u, lp, a->sh, a->dchain);
    else if (W::lane() == 0) lzb::dict_load<lzb::HostLanes>(a->dict, a->dsize >= 8 ? a->dsize - 7 : 0u, lp, a->sh, a->dchain);
    W::sync();
    T.ov = a->ov; T.sh = a->sh; T.dchain = a->dchain;
    const int r = lzb::encode_unit_dict<W>(a->src - a->dsize, (lzb::u32)a->n, a->dst, (lzb::u32)a->cap, a->level, T, a->work);
    if (W::lane() == 0) a->result = r;
}
static void emu_dict_compress_body(void* p) { dict_compress_body<EmuLanes>((DictCompressArgs*)p); }

extern "C" int lzb_dict_compress(const unsigned char* src, int n, unsigned char* dst, int cap, int level,
                                 const unsigned char* dict, int dict_size, int emu)
{
    if (n < 0 || cap < 0 || dict_size < 0) return 0;
    if (level > 49) level = 49;
    if (level < 10) level = 17;
    const lzb::LevelParams lp = lzb::level_params(level);
    if (!lzb::dict_parser(lp)) return 0;
    if (dict_size > (int)lzb::kDictSize) { dict += dict_size - (int)lzb::kDictSize; dict_size = (int)lzb::kDictSize; }   // :429-432
    DictCompressArgs a;
    a.src = src; a.n = n; a.dst = dst; a.cap = cap; a.level = level; a.dict = dict; a.dsize = (lzb::u32)dict_size; a.emu_load = emu & 2; a.result = 0;
    a.ov = (lzb::u32*)malloc(sizeof(lzb::u32) << lp.hashLog);
    a.sh = (lzb::u32*)malloc(sizeof(lzb::u32) << lp.hashLog);
    a.dchain = (lzb::u16*)malloc(sizeof(lzb::u16) << 16);
    a.work = (lzb::EncWork*)malloc(sizeof(lzb::EncWork));
    a.work->huf.seg_count = (lzb::u32 (*)[256])malloc(4 * 256 * sizeof(lzb::u32));
    memset(a.ov, 0x3C, sizeof(lzb::u32) << lp.hashLog);
    memset(a.sh, 0x3C, sizeof(lzb::u32) << lp.hashLog);
    memset(a.dchain, 0x5A, sizeof(lzb::u16) << 16);
    memset(a.work->chain, 0xA5, sizeof a.work->chain);
    if (emu & 1) emu::run(emu_dict_compress_body, &a);
    else dict_compress_body<lzb::HostLanes>(&a);
    free(a.work->huf.seg_count); free(a.work); free(a.dchain); free(a.sh); free(a.ov);
    return a.result;
}

// XXH32 as the frame kernels compute it (frame_device.cuh), one thread
extern "C" unsigned lzb_host_xxh32(const unsigned char* p, unsigned long long n, unsigned seed) { return lzb::xxh32_serial(p, n, seed); }

// LizardB200_decompressFrames for one frame on the host: the index kernel's walk, each compressed block through the one-lane
// decoder at the frame's maximum block size, frame_settle, placement and the checksum.  Returns the result as a size_t
// (LizardF error codes are negated); `blocks_out` = number of complete blocks the walk found.
extern "C" unsigned long long lzb_host_frame_decode(const unsigned char* src, unsigned long long n, unsigned char* dst,
                                                    unsigned long long cap, unsigned* blocks_out)
{
    lzb::FrameInfoRec fi;
    lzb::frame_walk(src, n, &fi, nullptr, 0);
    if (blocks_out) *blocks_out = fi.n_blocks;
    const unsigned nb = fi.verdict == lzb::kFwOk && !fi.skippable ? fi.n_blocks : 0;
    lzb::FrameBlockRec* blocks = (lzb::FrameBlockRec*)malloc((nb + 1) * sizeof(lzb::FrameBlockRec));
    int* decoded = (int*)calloc(nb + 1, sizeof(int));
    lzb::u64* place = (lzb::u64*)malloc((nb + 1) * 8);
    unsigned char** staged = (unsigned char**)calloc(nb + 1, sizeof(unsigned char*));
    if (nb) lzb::frame_walk(src, n, &fi, blocks, nb);
    for (unsigned k = 0; k < nb; ++k) {
        if (blocks[k].raw) continue;
        staged[k] = (unsigned char*)malloc(fi.max_block + 64);
        decoded[k] = lzb_host_decompress(src + blocks[k].src, (int)blocks[k].csize, staged[k], (int)fi.max_block);
    }
    lzb::u64 out = 0; lzb::u32 check = 0;
    lzb::u32 v = lzb::frame_settle(fi, blocks, decoded, cap, place, &out, &check);
    if (v == lzb::kFwOk && !fi.skippable) {
        for (unsigned k = 0; k < nb; ++k) {
            if (blocks[k].raw) memcpy(dst + place[k], src + blocks[k].src, blocks[k].csize);
            else if (decoded[k] > 0) memcpy(dst + place[k], staged[k], (size_t)decoded[k]);
        }
        if (check) v = lzb::frame_settle_hash(fi, lzb::xxh32_serial(dst, out, 0));
    }
    for (unsigned k = 0; k < nb; ++k) free(staged[k]);
    free(staged); free(place); free(decoded); free(blocks);
    if (v != lzb::kFwOk) return (unsigned long long)-(long long)v;
    return fi.skippable ? 0 : out;
}

// the staging arena LizardB200_decompressFramesAsync sizes for (max_blocks, stage_bytes)
extern "C" unsigned long long lzb_host_frame_stage_limit(unsigned max_blocks, unsigned long long stage_bytes)
{
    return lzb::frame_stage_limit(max_blocks, stage_bytes);
}

// LizardB200_decompressFramesAsync's planning (frame_async_kernels.cuh) serially: frame i takes blocks[i] blocks and, if it
// passes the block bound, slots[i] bytes of slots; ok[i] = 0 marks a frame whose header check failed.  Writes adm[i] and, for
// admitted frames, the block base and slot base the kernels give them.
// The stage bound is clamped first, as LizardB200_decompressFramesAsync clamps it (frame_stage_limit).
extern "C" void lzb_host_frame_async_plan(unsigned n, const unsigned long long* blocks, const unsigned long long* slots,
                                          const unsigned* ok, unsigned max_blocks, unsigned long long stage_bytes,
                                          unsigned* adm, unsigned long long* base, unsigned long long* slot)
{
    stage_bytes = lzb::frame_stage_limit(max_blocks, stage_bytes);
    std::vector<lzb::FrameInfoRec> fi(n);
    for (unsigned i = 0; i < n; ++i) {
        memset(&fi[i], 0, sizeof fi[i]);
        fi[i].verdict = ok[i] ? lzb::kFwOk : lzb::kFwFrameType;
        fi[i].n_blocks = (lzb::u32)blocks[i];
    }
    lzb::u64 before = 0;
    for (unsigned i = 0; i < n; ++i) {                                       // step 1: blocks
        const lzb::u64 v = lzb::frame_plan_blocks(fi[i]);
        adm[i] = lzb::frame_admit_blocks(before, v, max_blocks);
        base[i] = before;
        before += v;
    }
    before = 0;
    for (unsigned i = 0; i < n; ++i) {                                       // step 2: slots of the frames that passed step 1
        const lzb::u64 v = adm[i] && lzb::frame_plan_blocks(fi[i]) ? slots[i] : 0;     // as frame_plan_slots
        adm[i] = adm[i] && lzb::frame_admit_slots(before, v, stage_bytes);
        slot[i] = before;
        before += v;
    }
}

// One frame through LizardB200_decompressFramesAsync's layout: the walk, blocks decoded by the one-lane decoder into slots
// of the maximum block size behind each other in one staging arena, frame_settle_entries, the moves its gather entries
// describe (staged, then raw), the checksum.  Same return convention as lzb_host_frame_decode.
extern "C" unsigned long long lzb_host_frame_async_decode(const unsigned char* src, unsigned long long n, unsigned char* dst,
                                                          unsigned long long cap)
{
    lzb::FrameInfoRec fi;
    lzb::frame_walk(src, n, &fi, nullptr, 0);
    const unsigned nb = (unsigned)lzb::frame_plan_blocks(fi);
    std::vector<lzb::FrameBlockRec> blocks(nb + 1);
    if (nb) lzb::frame_walk(src, n, &fi, blocks.data(), nb);
    const lzb::u64 slots = lzb::frame_plan_slots(fi, blocks.data());
    std::vector<unsigned char> stage(slots + 64);
    std::vector<int> res(nb + 1, 0);
    std::vector<lzb::u64> at(nb + 1, 0), s_off(nb + 1), s_dst(nb + 1), r_off(nb + 1), r_dst(nb + 1);
    std::vector<int> s_len(nb + 1), r_len(nb + 1);
    lzb::u64 slot = 0;
    for (unsigned k = 0; k < nb; ++k) {
        if (blocks[k].raw) continue;
        at[k] = slot;
        res[k] = lzb_host_decompress(src + blocks[k].src, (int)blocks[k].csize, stage.data() + slot, (int)fi.max_block);
        slot += fi.max_block;
    }
    const lzb::FrameGather g{ s_off.data(), s_dst.data(), s_len.data(), r_off.data(), r_dst.data(), r_len.data() };
    lzb::u64 out = 0; lzb::u32 check = 0;
    lzb::u32 v = lzb::frame_settle_entries(fi, blocks.data(), res.data(), at.data(), 0, 0, cap, g, &out, &check);
    for (unsigned k = 0; k < nb; ++k) if (s_len[k] > 0) memcpy(dst + s_dst[k], stage.data() + s_off[k], (size_t)s_len[k]);
    for (unsigned k = 0; k < nb; ++k) if (r_len[k] > 0) memcpy(dst + r_dst[k], src + r_off[k], (size_t)r_len[k]);
    if (check) v = lzb::frame_settle_hash(fi, lzb::xxh32_serial(dst, out, 0));
    if (v != lzb::kFwOk) return (unsigned long long)-(long long)v;
    return fi.skippable ? 0 : out;
}

// LizardB200_compressFramesAsync's per-frame decisions (frame_device.cuh: frame_compress_plan) for a frame of src bytes with
// cap bytes of room under the given preference fields.  Returns the verdict; hdr (16 bytes) gets the header, out[0..4] the
// header length, block size, block count, staging bytes and checksum flag.
extern "C" unsigned lzb_host_frame_compress_plan(unsigned bsid, unsigned block_mode, unsigned ccksum, unsigned auto_flush,
                                                 unsigned long long content_size, int level_ok, unsigned long long src,
                                                 unsigned long long cap, unsigned char* hdr, unsigned long long* out)
{
    const lzb::FramePrefs p{ bsid, block_mode, ccksum, auto_flush, content_size };
    lzb::FrameCompressPlan pl;
    lzb::frame_compress_plan(p, level_ok != 0, src, cap, hdr, &pl);
    out[0] = pl.hdr_len; out[1] = pl.block_size; out[2] = pl.n_blocks; out[3] = pl.stage; out[4] = pl.ccksum;
    return pl.verdict;
}

// the staging arena LizardB200_compressFramesAsync sizes for (max_blocks, the preferences' block size ID, stage_bytes)
extern "C" unsigned long long lzb_host_frame_compress_stage_limit(unsigned max_blocks, unsigned bsid, unsigned long long stage_bytes)
{
    return lzb::frame_compress_stage_limit(max_blocks, bsid, stage_bytes);
}

// LizardB200_compressFramesAsync's planning (frame_compress_async_kernels.cuh) serially over n frames of sizes[i] bytes with
// caps[i] bytes of room: the plan of each frame, its demands and the admission on the two exclusive sums, after the stage
// clamp.  Writes adm[i], the block base first[i] and the staging base sbase[i].
extern "C" void lzb_host_frame_compress_admit(unsigned n, const unsigned long long* sizes, const unsigned long long* caps,
                                              unsigned bsid, unsigned block_mode, unsigned ccksum, unsigned long long content_size,
                                              int level_ok, unsigned max_blocks, unsigned long long stage_bytes, unsigned* adm,
                                              unsigned long long* first, unsigned long long* sbase)
{
    const lzb::FramePrefs p{ bsid, block_mode, ccksum, 0, content_size };
    stage_bytes = lzb::frame_compress_stage_limit(max_blocks, bsid, stage_bytes);
    lzb::u64 bb = 0, sb = 0;
    unsigned char hdr[16];
    for (unsigned i = 0; i < n; ++i) {
        lzb::FrameCompressPlan pl;
        lzb::frame_compress_plan(p, level_ok != 0, sizes[i], caps[i], hdr, &pl);
        const lzb::u64 b = lzb::frame_compress_demand_blocks(pl, max_blocks), s = lzb::frame_compress_demand_stage(pl);
        adm[i] = lzb::frame_admit_blocks(bb, b, max_blocks) && lzb::frame_admit_slots(sb, s, stage_bytes);
        first[i] = bb; sbase[i] = sb;
        bb += b; sb += s;
    }
}

// ---- LizardB200_decompressStream on the host (frame_stream.h): the state machine and StreamIO over host memory, the walk
// and the one-lane decoder standing in for the kernels, so the CPU tests compare a stream call for call with the reference.
#include "frame_stream.h"
namespace {
struct HostStreamExec {
    std::vector<lzb::u8> stage;
    lzb::u64 rounds = 0;
    void read(void* to, const void* p, size_t n) { memcpy(to, p, n); }
    void copy(void* to, const void* from, size_t n) { memmove(to, from, n); }
    void sync() {}
    void round(const lzb::u8* p, lzb::u64 n, lzb::u32 mb, const lzb::u8* carry, lzb::u32 carry_len, lzb::u32 max_recs,
               lzb::u32 slots, lzb::StreamWalk* walk, lzb::StreamWalkRec* recs, int* res, lzb::u8** st)
    {
        ++rounds;
        const size_t U = (size_t)slots + 1;
        std::vector<lzb::u64> u_src(U, 0);
        std::vector<lzb::u32> u_len(U, 0);
        *walk = lzb::frame_stream_walk(p, n, mb, recs, max_recs, slots, u_src.data(), u_len.data());
        u_src[0] = (lzb::u64)(size_t)carry; u_len[0] = carry_len;
        stage.assign(U * mb + 64, 0);
        for (size_t k = 0; k < U; ++k)
            res[k] = k <= walk->n_units ? lzb_host_decompress((const unsigned char*)(size_t)u_src[k], (int)u_len[k], stage.data() + k * mb, (int)mb) : 0;
        *st = stage.data();
    }
    void gather(const std::vector<lzb::StreamSeg>& segs) { for (const lzb::StreamSeg& g : segs) memcpy((void*)(size_t)g.dst, (const void*)(size_t)g.src, g.len); }
    void hash(const std::vector<lzb::StreamSeg>& segs, lzb::StreamHashState* h)
    {
        for (const lzb::StreamSeg& g : segs) lzb::xx_stream_update(h, (const lzb::u8*)(size_t)g.src, g.len);
    }
    void hash_reset(lzb::StreamHashState* h) { lzb::xx_stream_reset(h); }
    lzb::u32 digest(lzb::StreamHashState* h) { return lzb::xx_stream_digest(h); }
    void buffers(lzb::StreamBuffers& sb, size_t block)
    {
        if (block <= sb.block) return;
        free(sb.carry); free(sb.tmp_out);
        sb.carry = (lzb::u8*)malloc(block + 16); sb.tmp_out = (lzb::u8*)malloc(block + 64);
        if (!sb.carry || !sb.tmp_out) throw std::bad_alloc();
        sb.block = block; sb.tmp_at = sb.tmp_out;
    }
};
struct HostStream { lzb::FrameDState d; lzb::StreamBuffers sb; lzb::StreamHashState h; HostStreamExec x; };
}  // namespace

extern "C" void* lzb_host_stream_new()
{
    HostStream* s = new HostStream();
    s->d.reset();
    s->sb.hash = &s->h;
    lzb::xx_stream_reset(&s->h);
    return s;
}
extern "C" void lzb_host_stream_free(void* p)
{
    HostStream* s = (HostStream*)p;
    free(s->sb.carry); free(s->sb.tmp_out);
    delete s;
}
// one LizardB200_decompressStream call; *rounds (if not null) gets the rounds (walk + decode) the call ran
extern "C" size_t lzb_host_stream_call(void* p, unsigned char* dst, size_t* dst_size, const unsigned char* src, size_t* src_size,
                                       unsigned long long* rounds)
{
    HostStream* s = (HostStream*)p;
    const lzb::u64 r0 = s->x.rounds;
    size_t r;
    try { r = lzb::frame_stream_call(s->x, s->sb, &s->d, dst, dst_size, src, src_size); }
    catch (const std::bad_alloc&) { r = lzb::ferr(lzb::FE_allocation_failed); }
    if (rounds) *rounds = s->x.rounds - r0;
    return r;
}
// the walk of one round (frame_stream_walk): records as (pos, word, unit) triples, and the summary (records, stop, units)
extern "C" void lzb_host_stream_walk(const unsigned char* p, unsigned long long n, unsigned max_block, unsigned max_recs,
                                     unsigned slots, unsigned long long* pos, unsigned* word, int* unit, unsigned* summary)
{
    std::vector<lzb::StreamWalkRec> rec(max_recs);
    std::vector<lzb::u64> u_src((size_t)slots + 1);
    std::vector<lzb::u32> u_len((size_t)slots + 1);
    const lzb::StreamWalk w = lzb::frame_stream_walk(p, n, max_block, rec.data(), max_recs, slots, u_src.data(), u_len.data());
    for (lzb::u32 i = 0; i < w.n_recs; ++i) { pos[i] = rec[i].pos; word[i] = rec[i].word; unit[i] = rec[i].unit; }
    summary[0] = w.n_recs; summary[1] = w.stop; summary[2] = w.n_units;
}

// ---- LizardB200_compressStream* on the host (frame_cstream.h): the shared runs over host memory with the one-lane encoder in
// place of the kernels, so the CPU tests compare them call for call with the reference's LizardF_compressBegin / Update / flush /
// End.  Records are written as frame.inl's frame_compress_blocks and the assembly kernel write them (frame_record_payload).
#include "frame_cstream.h"
namespace {
struct HostCStream { lzb::FrameCState st; std::vector<lzb::u8> carry; lzb::StreamHashState h; };
struct ShimCompressIO {
    HostCStream* cs;
    bool ready() { return true; }
    bool level_ok(int level)
    {
        return lzb::level_params(level).parser != lzb::kParserUnsupported || lzb::lp_level(level) || lzb::opt_level(level);
    }
    void begin(lzb::u8* dst, const lzb::u8* hdr, lzb::u32 n, size_t bs)
    {
        memcpy(dst, hdr, n);
        lzb::xx_stream_reset(&cs->h);
        if (cs->carry.size() < bs) cs->carry.resize(bs);
    }
    void hash_begin(const lzb::u8*, size_t) {}
    void hash_end(const lzb::u8* p, size_t n) { lzb::xx_stream_update(&cs->h, p, n); }
    void hash_abort() {}
    void carry(size_t at, const lzb::u8* p, size_t n) { memcpy(cs->carry.data() + at, p, n); }
    size_t compress_carry(lzb::u8* dst, size_t cap, size_t n, int level) { return compress(dst, cap, cs->carry.data(), n, level); }
    size_t compress(lzb::u8* dst, size_t cap, const lzb::u8* p, size_t n, int level)
    {
        const size_t bs = cs->st.block_size;
        std::vector<lzb::u8> enc(bs + 64);
        size_t o = 0;
        for (size_t at = 0; at < n; at += bs) {
            const lzb::u32 len = (lzb::u32)(n - at < bs ? n - at : bs);
            const int r = lzb_host_compress(p + at, (int)len, enc.data(), (int)len - 1, level);
            const lzb::u32 payload = lzb::frame_record_payload(len, r);
            if (o + 4 + payload > cap) return lzb::ferr(lzb::FE_dstMaxSize_tooSmall);
            if (len == 1) lzb::frame_one_byte_record(dst + o, level, p[at]);
            else {
                lzb::wr_le32(dst + o, r > 0 ? (lzb::u32)r : (len | 0x80000000u));
                memcpy(dst + o + 4, r > 0 ? enc.data() : p + at, payload);
            }
            o += 4 + payload;
        }
        return o;
    }
    void end_mark(lzb::u8* dst, bool ccksum) { lzb::wr_le32(dst, 0); if (ccksum) lzb::wr_le32(dst + 4, lzb::xx_stream_digest(&cs->h)); }
};
}  // namespace

extern "C" void* lzb_host_cstream_new()
{
    HostCStream* s = new HostCStream();
    s->st.reset();
    lzb::xx_stream_reset(&s->h);
    return s;
}
extern "C" void lzb_host_cstream_free(void* p) { delete (HostCStream*)p; }
extern "C" size_t lzb_host_cstream_begin(void* p, unsigned char* dst, size_t cap, const LizardF_preferences_t* prefs)
{
    HostCStream* s = (HostCStream*)p;
    ShimCompressIO io{ s };
    return lzb::frame_cbegin_run(&s->st, io, dst, cap, prefs);
}
extern "C" size_t lzb_host_cstream_update(void* p, unsigned char* dst, size_t cap, const unsigned char* src, size_t n)
{
    HostCStream* s = (HostCStream*)p;
    ShimCompressIO io{ s };
    return lzb::frame_cupdate_run(&s->st, io, dst, cap, src, n);
}
extern "C" size_t lzb_host_cstream_flush(void* p, unsigned char* dst, size_t cap)
{
    HostCStream* s = (HostCStream*)p;
    ShimCompressIO io{ s };
    return lzb::frame_cflush_run(&s->st, io, dst, cap);
}
extern "C" size_t lzb_host_cstream_end(void* p, unsigned char* dst, size_t cap)
{
    HostCStream* s = (HostCStream*)p;
    ShimCompressIO io{ s };
    return lzb::frame_cend_run(&s->st, io, dst, cap);
}
// the planning kernel's unit k (cstream_unit): out = source address, length, encoder slot, capacity
extern "C" void lzb_host_cstream_unit(unsigned k, unsigned long long carry, unsigned long long carry_len, unsigned long long p,
                                      unsigned long long n, unsigned long long bs, unsigned long long stride, unsigned long long* out)
{
    lzb::u64 src, enc;
    lzb::u32 len, cap;
    lzb::cstream_unit(k, carry, carry_len, p, n, bs, stride, &src, &len, &enc, &cap);
    out[0] = src; out[1] = len; out[2] = enc; out[3] = cap;
}
// an Update's split of a chunk (frame_cupdate_plan): out = take, whole, rest, carry_block
extern "C" void lzb_host_cupdate_plan(unsigned long long carry, unsigned long long bs, unsigned auto_flush, unsigned long long n,
                                      unsigned long long* out)
{
    const lzb::CUpdatePlan pl = lzb::frame_cupdate_plan(carry, bs, auto_flush, n);
    out[0] = pl.take; out[1] = pl.whole; out[2] = pl.rest; out[3] = pl.carry_block;
}
