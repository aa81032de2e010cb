// encode_dict_kernel.cuh -- compression against a loaded dictionary at the hashChain (13-17 / 34-38) and priceFast (21, 22,
// 41, 42) levels: each unit is
// Lizard_createStream(level) + Lizard_loadDict(dict) + Lizard_compress_continue(unit), byte for byte (encode_unit_dict in
// encode_core.cuh).  One launch of lizard_encode_dict_kernel: one warp per unit on the encoder's persistent grid, unit queue and
// progress hand-shake.
//   * Each distinct dictionary (end offset and size, after the trim to the last 2^24 bytes) gets a slot through an
//     open-addressed map.  The warp whose unit claims a new key takes the next slot and replays Lizard_Insert over the
//     dictionary into the slot's table (2^hashLog u32) and chain (2^16 u16) (dict_load), then marks it ready.  Warps whose
//     units find the key wait until the slot is ready.  A loader waits on nothing, so every wait ends.  All dictionaries below
//     8 bytes share one key: Lizard_loadDict inserts nothing then, so their slot's table is empty.
//   * The unit reads its slot's table through its own overlay (the plain 1 MiB table of its EncWork scratch) and never copies it.
// Workspace (the encoder's, which does not grow): [map + slot flags][slots x kDictSlotBytes][grid warps x per-warp scratch].
// Units whose dictionary gets no slot (more distinct dictionaries than the workspace holds: dict_shape()) are not run and get
// the result -1.  Slots go to keys in the order warps claim them, so which units those are depends on scheduling.
// The table is 2^18 entries whatever the level's hashLog (14 or 18); dict_load clears and fills the level's 2^hashLog.
#pragma once
#include "encode.cuh"

namespace lzb {

constexpr int kDictWarpsPerCta = 4;
constexpr int kDictMaxRegs = 96;
constexpr size_t kDictSlotBytes = ((size_t)4 << 18) + ((size_t)2 << 16);   // table at hashLog 18 + chain

struct DictBatch {
    const u8* dict_base; const u64* dict_off; const u32* dict_len;
    u64* keys;                                // (end, size) -> map entry; 0 = empty entry
    u32* ids;                                 // per map entry: slot + 1 once published, 0 before
    u32* ready;                               // per slot: 1 once its table is loaded
    u32* n_slots;                             // slots handed out
    u32 map_mask, max_slots;
    u8* slots;
};

__device__ __forceinline__ u32 dict_hash(u64 key, u32 mask) { return (u32)((key * 0x9E3779B97F4A7C15ull) >> 40) & mask; }

// the unit's slot, loading it first if the unit is the first of its dictionary; >= max_slots: no slot
__device__ __forceinline__ u32 dict_acquire(const DictBatch& d, u64 off, u32 len, int level, u32 lane)
{
    const u64 key = len < 8 ? 1ull : ((off + len) << 25 | len) + 2;
    u32 slot = 0, load = 0;
    if (lane == 0) {
        u32 h = dict_hash(key, d.map_mask);
        for (;; h = (h + 1) & d.map_mask) {
            const u64 prev = atomicCAS(reinterpret_cast<unsigned long long*>(&d.keys[h]), 0ull, (unsigned long long)key);
            if (prev == 0) {
                slot = atomicAdd(d.n_slots, 1u);
                load = slot < d.max_slots;
                atomicExch(&d.ids[h], slot + 1);
                break;
            }
            if (prev == key) {
                volatile u32* id = d.ids + h;
                while ((slot = *id) == 0) __nanosleep(200);
                --slot;
                if (slot < d.max_slots) { volatile u32* r = d.ready + slot; while (*r == 0) __nanosleep(500); }
                __threadfence();
                break;
            }
        }
    }
    slot = __shfl_sync(0xffffffffu, slot, 0);
    load = __shfl_sync(0xffffffffu, load, 0);
    if (load) {
        u8* p = d.slots + (size_t)slot * kDictSlotBytes;
        dict_load<WarpLanes>(d.dict_base + off, len >= 8 ? len - 7 : 0u, level_params(level),
                             reinterpret_cast<u32*>(p), reinterpret_cast<u16*>(p + ((size_t)4 << 18)));
        __syncwarp();
        if (lane == 0) { __threadfence(); atomicExch(&d.ready[slot], 1u); }
    }
    return slot;
}

__global__ void __maxnreg__(kDictMaxRegs)
lizard_encode_dict_kernel(EncodeBatch b, DictBatch d, size_t per_warp_bytes)
{
    __shared__ u32 seg_hist[kDictWarpsPerCta][4][256];
    const u32 lane = WarpLanes::lane(), wic = threadIdx.x >> 5;
    u8* const my = b.scratch + ((size_t)blockIdx.x * kDictWarpsPerCta + wic) * per_warp_bytes;
    EncWork* const work = reinterpret_cast<EncWork*>(my);
    if (lane == 0) work->huf.seg_count = seg_hist[wic];
    __syncwarp();
    for (;;) {
        u32 unit = 0;
        if (lane == 0) unit = atomicAdd(b.counter, 1u);
        unit = __shfl_sync(0xffffffffu, unit, 0);
        if (unit >= b.n_units) break;
        progress_wait(b.progress, unit, lane);
        u64 off = d.dict_off[unit]; u32 len = d.dict_len[unit];
        if (len > kDictSize) { off += len - kDictSize; len = kDictSize; }          // lib/lizard_compress.c:429-432
        const u32 slot = dict_acquire(d, off, len, b.level, lane);
        int r = -1;
        if (slot < d.max_slots) {
            const u8* unit_src = b.src_base + b.src_off[unit];
            const u32 n = b.src_len[unit];
            const u8* dict = d.dict_base + off;
            DictTable T = dict_view(unit_src, n, dict, len);
            const u8* sp = d.slots + (size_t)slot * kDictSlotBytes;
            T.ov = reinterpret_cast<u32*>(my + sizeof(EncWork));
            T.sh = reinterpret_cast<const u32*>(sp);
            T.dchain = reinterpret_cast<const u16*>(sp + ((size_t)4 << 18));
            r = encode_unit_dict<WarpLanes>(unit_src - len, n, b.dst_base + b.dst_off[unit], b.dst_cap[unit], b.level, T, work);
        }
        if (lane == 0) b.result[unit] = r;
        __syncwarp();
        progress_done(b.progress, unit, lane);
    }
}

// Workspace split for n units: the map and slot flags first, then as many warps as registers allow (capped by the units), then
// every remaining byte as slots (at most n).
struct DictShape { size_t meta_bytes, grid, per_warp; u32 map_mask, max_slots; };
inline DictShape dict_shape(const EncodeConfig& c, u32 n)
{
    DictShape sh;
    u32 map = 16; while (map < 2 * n) map <<= 1;
    sh.map_mask = map - 1;
    sh.per_warp = c.per_warp_small;
    const size_t per_sm = 65536 / (kDictMaxRegs * 32 * kDictWarpsPerCta);
    sh.grid = (size_t)c.sm_count * per_sm;
    const size_t need = (n + kDictWarpsPerCta - 1) / kDictWarpsPerCta;
    if (sh.grid > need) sh.grid = need;
    sh.meta_bytes = enc_align((size_t)map * 12 + (size_t)n * 4 + 256);
    const size_t warps_bytes = sh.grid * kDictWarpsPerCta * sh.per_warp;
    const size_t rest = c.scratch_bytes > sh.meta_bytes + warps_bytes ? c.scratch_bytes - sh.meta_bytes - warps_bytes : 0;
    size_t slots = rest / kDictSlotBytes;
    if (slots > (size_t)n) slots = (size_t)n;
    sh.max_slots = (u32)slots;
    return sh;
}

inline cudaError_t dict_encode_launch(const EncodeConfig& c, EncodeBatch b, const u8* dict_base, const u64* dict_off,
                                      const u32* dict_len, cudaStream_t s, int* launches)
{
    const DictShape sh = dict_shape(c, b.n_units);
    if (sh.max_slots < 1) return cudaErrorMemoryAllocation;
    u8* const ws = b.scratch;
    DictBatch d;
    d.dict_base = dict_base; d.dict_off = dict_off; d.dict_len = dict_len;
    d.keys = reinterpret_cast<u64*>(ws);
    d.ids = reinterpret_cast<u32*>(d.keys + (sh.map_mask + 1));
    d.ready = d.ids + (sh.map_mask + 1);
    d.n_slots = d.ready + b.n_units;
    d.map_mask = sh.map_mask; d.max_slots = sh.max_slots;
    d.slots = ws + sh.meta_bytes;
    b.scratch = d.slots + (size_t)sh.max_slots * kDictSlotBytes;
    const cudaError_t e = cudaMemsetAsync(ws, 0, sh.meta_bytes, s);
    if (e != cudaSuccess) return e;
    lizard_encode_dict_kernel<<<(unsigned)sh.grid, 32 * kDictWarpsPerCta, 0, s>>>(b, d, sh.per_warp);
    *launches = 1;
    return cudaGetLastError();
}

}  // namespace lzb
