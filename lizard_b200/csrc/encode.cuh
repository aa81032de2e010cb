// encode.cuh -- device kernel around encode_core.cuh: one warp per independent unit
// (= one Lizard_compress call, normally one 128 KiB frame block), persistent grid, atomic work queue.
//
// The kernel is one template, lizard_encode_units_kernel<kFam>, instantiated per parser family (enc_family() in
// encode_core.cuh): Fast (levels 10/11: 72 registers, no stack), FastBig (20) and Generic (the rest, Huffman stage
// included).  Every instance has the same launch bounds, table setup and frame packing; encode_launch() runs the level's.
// Level 10 on an H100 SXM 80 GB at a 400 W limit: 11.7 ms per GiB (12.2 with one kernel for all levels).
//
// Memory placement per warp (launch shape per level: encode_shape() below):
//   shared : the PACKED hash table (16-bit entries + a bit plane for position bit 16 + one tag byte per entry for the fast
//            parsers: 12.5 KiB at level 10/30, 34 KiB untagged at 20/21/40/41) for as many of a CTA's 14 warps as the
//            measured shape gives one (7 at level 10, 3 at 30, 2 at 20/21, 1 at 40/41), + 4 KiB of per-segment byte
//            histograms for the Huffman stage
//   global : for the other warps the plain 32-bit table in their scratch (tags in the spare bits of an entry; 16 KiB at
//            hashLog 12, 64 KiB at 14, 1 MiB at 18 or for multi-inner-block units), the sequence list of the block being
//            parsed, the flags / literals streams when an entropy stage follows, the Huffman build scratch
#pragma once
#include "common.cuh"
#include "encode_core.cuh"
#include "decode.cuh"       // Progress hand-shake
#include "frame_device.cuh" // the block record rule (frame_record_payload)
#include <cuda_runtime.h>
#include <cstdlib>
#include <cmath>
#include <cstdio>

namespace lzb {

// Frame packing fused into the encoder (LizardF block records, lib/lizard_frame.c:455-476): once a unit is encoded
// its warp learns where the record goes from a decoupled look-back over the units before it (units are handed out
// in ascending order, so every predecessor is running or done), writes the 4-byte block header and moves the payload
// (the compressed bytes, or the source bytes when the block did not shrink) to its final place.  The warp that
// completes a chunk publishes the chunk's end offset next to the done flag, and the host copies that byte range out.
struct FramePack {
    u8*           out;             // packed records, contiguous; null = no packing
    u64*          state;           // [n_units] look-back words, zero before launch
    volatile u64* host_chunk_end;  // mapped pinned: [n_chunks] end offset of the chunk's last record
};
#define kPackAgg (1ull << 62)
#define kPackIncl (1ull << 63)
#define kPackMask ((1ull << 62) - 1)

struct EncodeBatch {
    const u8*  src_base;  const u64* src_off;  const u32* src_len;
    u8*        dst_base;  const u64* dst_off;  const u32* dst_cap;
    int*       result;    // [n] Lizard_compress return value (0 = failed / does not fit)
    u32        n_units;
    int        level;
    u8*        scratch;   // grid_warps * per_warp_bytes
    u32*       counter;
    Progress   progress;
    FramePack  pack;
};

// byte-exact warp copy with 4-byte stores once dst is aligned (src may have any alignment)
__device__ __forceinline__ void warp_copy_words(u8* dst, const u8* src, u32 n, u32 lane)
{
    u32 head = (u32)((4 - ((size_t)dst & 3)) & 3);
    if (head > n) head = n;
    if (lane < head) dst[lane] = src[lane];
    dst += head; src += head; n -= head;
    const u32 words = n >> 2;
    const size_t sa = (size_t)src;
    const u32* sq = (const u32*)(sa & ~(size_t)3);
    const u32 sh = (u32)(sa & 3) * 8;
    u32* dq = (u32*)dst;
    if (sh == 0) { for (u32 i = lane; i < words; i += 32) dq[i] = sq[i]; }
    else {
        u32 i = lane;
        for (; i + 96 < words; i += 128) {                   // four independent words in flight per lane
            const u32 a0 = sq[i], a1 = sq[i + 1], b0 = sq[i + 32], b1 = sq[i + 33];
            const u32 c0 = sq[i + 64], c1 = sq[i + 65], d0 = sq[i + 96], d1 = sq[i + 97];
            dq[i] = __funnelshift_r(a0, a1, sh); dq[i + 32] = __funnelshift_r(b0, b1, sh);
            dq[i + 64] = __funnelshift_r(c0, c1, sh); dq[i + 96] = __funnelshift_r(d0, d1, sh);
        }
        for (; i < words; i += 32) dq[i] = __funnelshift_r(sq[i], sq[i + 1], sh);
    }
    const u32 tail = n & 3;
    if (lane < tail) dst[words * 4 + lane] = src[words * 4 + lane];
}

// Exclusive prefix of the record sizes of units [0, unit): decoupled look-back, 32 predecessors per step.
__device__ __forceinline__ u64 pack_lookback(volatile u64* state, u32 unit, u64 rec, u32 lane)
{
    if (unit == 0) {
        if (lane == 0) { __threadfence(); state[0] = kPackIncl | rec; }
        return 0;
    }
    if (lane == 0) { __threadfence(); state[unit] = kPackAgg | rec; }
    u64 excl = 0;
    long hi = (long)unit - 1;                                 // next predecessor to look at
    for (;;) {
        const long idx = hi - (long)lane;
        u64 w = 0;
        for (;;) {
            w = idx >= 0 ? state[idx] : kPackIncl;            // before unit 0: inclusive prefix 0
            if (__all_sync(0xffffffffu, (w & (kPackAgg | kPackIncl)) != 0)) break;
            __nanosleep(100);
        }
        const u32 incl = __ballot_sync(0xffffffffu, (w & kPackIncl) != 0);
        const u32 stop = incl ? (u32)(__ffs((int)incl) - 1) : 32;   // nearest predecessor with an inclusive prefix
        u64 v = lane <= stop ? (w & kPackMask) : 0;
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        excl += v;
        if (incl) break;
        hi -= 32;
    }
    if (lane == 0) { __threadfence(); state[unit] = kPackIncl | (excl + rec); }
    return excl;
}

__device__ __forceinline__ void pack_unit(const EncodeBatch& b, u32 unit, u32 len, int r, u32 lane)
{
    const u32 payload = frame_record_payload(len, r);
    const u64 at = pack_lookback(b.pack.state, unit, 4 + (u64)payload, lane);
    u8* o = b.pack.out + at;
    const u8* src = b.src_base + b.src_off[unit];
    if (len == 1) {
        if (lane == 0) frame_one_byte_record(o, b.level, src[0]);
        return;
    }
    const u32 word = r > 0 ? (u32)r : (len | 0x80000000u);
    if (lane < 4) o[lane] = (u8)(word >> (8 * lane));
    warp_copy_words(o + 4, r > 0 ? b.dst_base + b.dst_off[unit] : src, payload, lane);
}

// chunk bookkeeping with packing: the warp that finishes a chunk reports where the chunk's records end
__device__ __forceinline__ void pack_done(const EncodeBatch& b, u32 unit, u32 lane)
{
    const Progress& pg = b.progress;
    if (pg.done_count && lane == 0) {
        __threadfence();
        u32 first, cnt;
        const u32 c = progress_chunk(pg, unit, &first, &cnt);
        if (atomicAdd(&pg.done_count[c], 1u) == cnt - 1) {
            __threadfence();
            volatile u64* st = b.pack.state;
            const u64 w = st[first + cnt - 1];                // inclusive: that unit finished, so it is published
            b.pack.host_chunk_end[c] = w & kPackMask;
            __threadfence_system();
            pg.host_done[c] = 1u;
        }
    }
}

struct EncodeConfig {
    int    sm_count = 0;
    size_t per_warp_small = 0;    // EncWork only
    size_t per_warp_big = 0;      // EncWork + 1 MiB table
    int    max_warps = 0;         // upper bound on resident warps (sizes the scratch)
    size_t scratch_bytes = 0;
};

constexpr u32 kEncBigTableBytes = 4u << 18;          // plain 32-bit table for hashLog 18 or multi-inner-block units
// Residency: registers allow 28 warps per SM (72 registers/thread), the register limit.  The grid therefore runs CTAs of
// 14 warps, two per SM; how many of the 14 keep their hash table in shared memory is the launch shape (encode_shape()),
// the others use the plain table in their global scratch (L1/L2-resident, slower).  On 132 SMs the 8192-block workload is
// 2.2 rounds of the 3696 resident warps; the atomic work queue hands the last blocks to whichever warps finish first.
constexpr int kEncWarpsPerCta = 14, kEncCtasPerSM = 2, kEncMaxWarpsPerSM = kEncWarpsPerCta * kEncCtasPerSM;

#if !defined(LZB_ENC_OPAQUE)
#define LZB_ENC_OPAQUE 2
#endif
// One instance per parser family (enc_family(), encode_core.cuh); the launch picks the level's instance.
template <int kFam>
__global__ void __launch_bounds__(32 * kEncWarpsPerCta, kEncCtasPerSM)
lizard_encode_units_kernel(EncodeBatch b, u32 smem_tables, u32 table_bytes, u32 hist_bytes, size_t per_warp_bytes)
{
    extern __shared__ __align__(16) unsigned char enc_smem[];
    const u32 lane = WarpLanes::lane(), wic = threadIdx.x >> 5, wpc = blockDim.x >> 5;
    const size_t my_off = ((size_t)blockIdx.x * wpc + wic) * per_warp_bytes;
    // shared layout: [smem_tables packed hash tables][per-warp 4 KiB segment histograms, entropy levels only]
    const bool packed_ok = wic < smem_tables;
    u32* seg_hist = reinterpret_cast<u32*>(enc_smem + (size_t)smem_tables * table_bytes + (size_t)wic * hist_bytes);
    if (lane == 0) reinterpret_cast<EncWork*>(b.scratch + my_off)->huf.seg_count = reinterpret_cast<u32 (*)[256]>(seg_hist);
    __syncwarp();
    for (;;) {
        u32 unit = 0;
        if (lane == 0) unit = atomicAdd(b.counter, 1u);
        unit = __shfl_sync(0xffffffffu, unit, 0);
        if (unit >= b.n_units) break;
        progress_wait(b.progress, unit, lane);
        const u32 len = b.src_len[unit];
        // The level's parameters, the warp's scratch base and its table base are derived per unit: kept for the whole
        // kernel they took local-memory slots.  The two bases are then held in registers for the unit: left to itself
        // the compiler re-derives them (a 64-bit multiply-add) in front of every access.
        const LevelParams klp = level_params(b.level);
        const bool tagged = enc_tagged(klp), tagged_plain = enc_tagged_plain(klp);
        u8* my = b.scratch + my_off;
        u8* tab = enc_smem + (size_t)wic * table_bytes;
#if LZB_ENC_OPAQUE
        asm volatile("" : "+l"(my));
#endif
#if LZB_ENC_OPAQUE >= 2
        asm volatile("" : "+l"(tab));            // (generic instead of shared-space accesses to the packed table then)
#endif
        EncWork* work = reinterpret_cast<EncWork*>(my);
        // 17-bit packed entries need every position of the unit below 2^17
        HashTable T;
        if (packed_ok && len <= kBlockSize) {
            T.t32 = nullptr; T.lo = reinterpret_cast<u16*>(tab);
            T.hi = reinterpret_cast<u32*>(tab + ((size_t)2 << klp.hashLog));
            T.tag = tagged ? tab + hash_packed_bytes(klp.hashLog, false) : nullptr; T.tagged = 0;
        } else {
            T.t32 = reinterpret_cast<u32*>(my + sizeof(EncWork)); T.lo = nullptr; T.hi = nullptr; T.tag = nullptr;
            T.tagged = (tagged_plain && len <= kBlockSize) ? 1u : 0u;      // 7 spare bits per entry when positions stay below 2^17
        }
        const int r = encode_unit_fam<WarpLanes, kFam>(b.src_base + b.src_off[unit], len,
                                                       b.dst_base + b.dst_off[unit], b.dst_cap[unit], b.level, T, work);
        if (lane == 0) b.result[unit] = r;
        __syncwarp();
        if (b.pack.out) { pack_unit(b, unit, len, r, lane); __syncwarp(); pack_done(b, unit, lane); }
        else progress_done(b.progress, unit, lane);
    }
}

inline size_t enc_align(size_t v) { return (v + 255) / 256 * 256; }

typedef void (*EncodeKernel)(EncodeBatch, u32, u32, u32, size_t);
inline EncodeKernel encode_kernel(int fam)
{
    switch (fam) {
    case kEncFamFast:    return lizard_encode_units_kernel<kEncFamFast>;
    case kEncFamFastBig: return lizard_encode_units_kernel<kEncFamFastBig>;
    default:             return lizard_encode_units_kernel<kEncFamGeneric>;
    }
}

inline int encode_context_init(EncodeConfig& c, int sm_count, int)
{
    c.sm_count = sm_count;
    c.per_warp_small = enc_align(sizeof(EncWork) + kEncBigTableBytes);
    c.per_warp_big = c.per_warp_small;
    for (int f = 0; f < kEncFamilies; ++f)
        if (cudaFuncSetAttribute(encode_kernel(f), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 227 * 1024) != cudaSuccess) return -1;
    c.max_warps = sm_count * kEncMaxWarpsPerSM;
    c.scratch_bytes = (size_t)c.max_warps * c.per_warp_small;
    return 0;
}

// Launch shape for a level: warps per CTA, how many of them own a shared-memory table, dynamic shared bytes.
struct EncodeShape { int warps, smem_tables; size_t table_bytes, hist_bytes, smem; int ctas_per_sm; };
inline EncodeShape encode_shape(const LevelParams& lp)
{
    EncodeShape sh;
    sh.table_bytes = lp.hashLog <= 14 ? hash_packed_bytes(lp.hashLog, enc_tagged(lp)) : 0;
    sh.hist_bytes = lp.huffman ? 4096 : 0;
    const size_t sm_max = 228 * 1024, cta_reserved = 1024, cta_max = 227 * 1024;
    // Shared memory and L1 are one 256 KB array per SM, and the 14-warp shapes do better when they do not take all of it:
    // their tables are sized for the 196 KB carve-out step, which leaves the L1 60 KB for the input and the match
    // candidates (H100 SXM at a 400 W limit, 1 GiB, level 10: 14,7,2 12.2 ms against 14.0 ms for 14,11,2 in the 228 KB step;
    // level 21: 14,2,2 61.9 ms, 14,3,2 61.7, 14,1,2 65.7).
    const size_t sm_pref = 196 * 1024;
    // Three shapes, picked from measurements (tools/dec_bench.py --enc-shapes):
    //   A. 2 CTAs x 14 warps when at least 8 of the 14 could get a shared-memory table (level 10-style small tables),
    //      or when there is no shared-memory table at all (hashLog 18: everything global anyway);
    //   B. one warp per CTA, every warp on a shared-memory table, when that keeps >= 16 warps resident;
    //   C. otherwise 2 CTAs x 14 warps with as many shared-memory tables as fit the preferred carve-out.
    auto tabs_for = [&](int warps, int ctas, size_t sm_bytes) -> int {
        const size_t budget = sm_bytes / ctas < cta_max + cta_reserved ? sm_bytes / ctas - cta_reserved : cta_max;
        const size_t hist = (size_t)warps * sh.hist_bytes;
        if (hist > budget) return -1;
        if (!sh.table_bytes) return 0;
        int t = (int)((budget - hist) / sh.table_bytes);
        return t > warps ? warps : t;
    };
    EncodeShape best = sh;
    auto set = [&](int warps, int tabs, int ctas) {
        best.warps = warps; best.smem_tables = tabs; best.ctas_per_sm = ctas;
        best.smem = (size_t)tabs * sh.table_bytes + (size_t)warps * sh.hist_bytes;
    };
    const int fit14 = tabs_for(kEncWarpsPerCta, kEncCtasPerSM, sm_max);       // tables that fit at all
    int tabs14 = tabs_for(kEncWarpsPerCta, kEncCtasPerSM, sm_pref);           // tables we give the 14-warp shapes
    if (tabs14 < 0) tabs14 = fit14 < 0 ? -1 : 0;
    int solo = 0;                                                   // shape B: resident single-warp CTAs
    for (int ctas = kEncMaxWarpsPerSM; ctas >= 1; --ctas) if (tabs_for(1, ctas, sm_max) >= (sh.table_bytes ? 1 : 0)) { solo = ctas; break; }
    // every table the preferred step holds pays for itself (H100, 1 GiB, level 10: 14,7,2 12.2 ms; 14,5,2 15.0; 14,3,2 19.4;
    // 14,2,2 22.0; level 41, one 34 KiB table beside the histograms: 14,1,2 72.0 ms against 78.4 for 14,0,2)
    if (!sh.table_bytes || fit14 >= 8) set(kEncWarpsPerCta, tabs14 < 0 ? 0 : tabs14, kEncCtasPerSM);
    else if (solo >= 16) set(1, 1, solo);
    else if (tabs14 >= 0) set(kEncWarpsPerCta, tabs14, kEncCtasPerSM);
    else set(1, 1, solo >= 1 ? solo : 1);
    return best;
}

// The shape a launch uses: encode_shape(), unless LIZARDB200_ENC_SHAPE="warps,tables,ctas" is set and valid (diagnostics and
// tests: "14,0,2" runs every warp on the plain global table, "1,1,1" one warp per SM on a shared-memory table).  Levels
// without a shared-memory table keep 0 tables whatever the variable asks.  The CTAs per SM are an upper bound the launch
// lowers to what the device can hold.
inline EncodeShape encode_shape_in_effect(const LevelParams& lp)
{
    EncodeShape sh = encode_shape(lp);
    if (const char* e = getenv("LIZARDB200_ENC_SHAPE")) {
        int w = 0, t = 0, k = 0;
        if (sscanf(e, "%d,%d,%d", &w, &t, &k) == 3 && w >= 1 && w <= kEncWarpsPerCta && t >= 0 && t <= w && k >= 1) {
            sh.warps = w; sh.smem_tables = sh.table_bytes ? t : 0; sh.ctas_per_sm = k;
            sh.smem = (size_t)sh.smem_tables * sh.table_bytes + (size_t)w * sh.hist_bytes;
        }
    }
    return sh;
}

inline cudaError_t encode_launch(const EncodeConfig& c, const EncodeBatch& b, cudaStream_t s, int* launches)
{
    const LevelParams lp = level_params(b.level);
    const EncodeShape sh = encode_shape_in_effect(lp);
    const EncodeKernel kern = encode_kernel(enc_family(lp));
    const size_t per_warp = c.per_warp_small;
    int per_sm = 0;
    // the occupancy query honours the kernel's current carve-out preference, which the previous launch (possibly of
    // another level) left behind: ask with the whole array available, then set what this launch uses
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 32 * sh.warps, sh.smem);
    if (e != cudaSuccess) return e;
    if (per_sm < 1) per_sm = 1;
    if (per_sm > sh.ctas_per_sm) per_sm = sh.ctas_per_sm;
    size_t grid = (size_t)c.sm_count * per_sm;
    const size_t need = (b.n_units + sh.warps - 1) / sh.warps;
    if (grid > need) grid = need;
    if (grid * sh.warps * per_warp > c.scratch_bytes) grid = c.scratch_bytes / (per_warp * sh.warps);
    {   // shared memory and L1 share one array: ask for the carve-out the resident CTAs use, no more (see api.cu)
        const size_t total = 228 * 1024, use = (size_t)per_sm * (sh.smem + 1024);
        int pct = (int)((use * 100 + total - 1) / total);
        if (pct > 100) pct = 100;
        cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, pct);
    }
    kern<<<(unsigned)grid, 32 * sh.warps, sh.smem, s>>>(b, (u32)sh.smem_tables, (u32)sh.table_bytes, (u32)sh.hist_bytes, per_warp);
    *launches = 1;
    return cudaGetLastError();
}

}  // namespace lzb
