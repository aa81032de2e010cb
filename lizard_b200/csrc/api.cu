// api.cu -- C-ABI shim of liblizard_b200.so (see include/lizard_b200.h): context, workspaces, kernel
// launches, host staging.  Host-side logic only; the codec lives in decode.cuh / encode.cuh.
#include "../../include/lizard_b200.h"
#include "decode.cuh"
#include "decode2.cuh"
#include "prepass.cuh"
#include "encode.cuh"
#include "encode_lp_kernel.cuh"
#include "encode_opt_kernel.cuh"
#include "encode_dict_kernel.cuh"
#include "frame_device_kernels.cuh"
#include "frame_async_kernels.cuh"
#include "frame_compress_async_kernels.cuh"
#include "frame_stream_kernels.cuh"
#include "frame_stream.h"
#include "frame_cstream_kernels.cuh"
#include "frame_cstream.h"

#include <cuda_runtime.h>
#include <mutex>
#include <thread>
#include <functional>
#include <vector>
#include <unordered_map>
#include <map>
#include <utility>
#include <string>
#include <atomic>
#include <cstring>
#include <cstdio>
#include <cstdlib>
#include <chrono>
#include <new>

using namespace lzb;

namespace {

#if !defined(LZB_DEC_SH_OPAQUE)
#define LZB_DEC_SH_OPAQUE 1
#endif
#if !defined(LZB_DEC_WARPS)
#define LZB_DEC_WARPS 8
#endif
constexpr int kDecWarps = LZB_DEC_WARPS;     // warps per CTA in the decode kernel (x 4 CTAs per SM)
constexpr int kMaxDevices = 16;

// Body of the first-generation decode kernels: a persistent set of warps, one unit per warp at a time.
// kPartial: Lizard_decompress_safe_partial with the unit's b.target instead of Lizard_decompress_safe.
// kDict: Lizard_decompress_safe_usingDict with the unit's dictionary (b.dict_*).
template <int V, bool kPartial, bool kDict = false> __device__ __forceinline__ void decode_units(const DecodeBatch& b)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const u32 warp = threadIdx.x >> 5, lane = WarpLanes::lane();
    DecWarpShared* sh = reinterpret_cast<DecWarpShared*>(smem_raw) + warp;
#if LZB_DEC_SH_OPAQUE
    // one register for the warp's block: left to itself the compiler re-derives `base + warp * size` in front of every access
    // (10 % of the kernel's instructions); the price is generic instead of shared-space loads
    asm volatile("" : "+l"(sh));
#endif
    const size_t gwarp = (size_t)blockIdx.x * kDecWarps + warp;
    u8* scratch = b.scratch + gwarp * kDecScratchPerWarp;
    if (lane == 0) sh->big_table = reinterpret_cast<u16*>(scratch + 4 * kDecStreamScratch);
    __syncwarp();
    for (;;) {
        u32 unit = 0;
        if (lane == 0) unit = atomicAdd(b.counter, 1u);
        unit = __shfl_sync(LZB_FULL, unit, 0);
        if (unit >= b.n_units) break;
        progress_wait(b.progress, unit, lane);
        int r;
        if constexpr (kPartial) r = decode_unit<WarpLanes, V, true>(b.src_base + b.src_off[unit], b.src_len[unit],
                                                          b.dst_base + b.dst_off[unit], b.dst_cap[unit], scratch, sh,
                                                          nullptr, nullptr, nullptr, nullptr, b.target[unit]);
        else if constexpr (kDict) {
            u8* const dst = b.dst_base + b.dst_off[unit];
            const u32 dl = b.dict_len[unit];
            DictWin dw;
            dw.end = b.dict_base + b.dict_off[unit] + dl;
            dw.avail = dl;
            dw.reach = b.dict_reach ? b.dict_reach[unit] : dict_reach(dl, dw.end == dst);
            r = decode_unit<WarpLanes, V, false, true>(b.src_base + b.src_off[unit], b.src_len[unit], dst, b.dst_cap[unit], scratch, sh,
                                                       b.pre ? b.pre + unit : nullptr, b.arena, nullptr, nullptr, 0, dw);
        }
        else r = decode_unit<WarpLanes, V>(b.src_base + b.src_off[unit], b.src_len[unit],
                                           b.dst_base + b.dst_off[unit], b.dst_cap[unit], scratch, sh,
                                           b.pre ? b.pre + unit : nullptr, b.arena,
                                           b.seq ? b.seq + unit : nullptr, b.recs);
        if (lane == 0) b.result[unit] = r;
        __syncwarp();
        progress_done(b.progress, unit, lane);
    }
}

// V = schedule of the token loops, two bits: 1 = pooled copy sweeps, 2 = compact length-extension chain (default 3 = both;
// LIZARDB200_DEC_VARIANT=0..3 or LizardB200_setDecodeVariant select the others for A/B runs)
template <int V> __global__ void __launch_bounds__(kDecWarps * 32, 4)
lizard_decode_units_kernel(DecodeBatch b)
{
    decode_units<V, false>(b);
}

// Partial decode (LizardB200_decompress_partial_*): a kernel of its own, so that the full decode above keeps its code.  It runs
// the default schedule and never the pre-passes, which expand or parse whole streams that a partial unit may never reach.
constexpr int kDecDefaultSchedule = 3;
__global__ void __launch_bounds__(kDecWarps * 32, 4) lizard_decode_partial_units_kernel(DecodeBatch b)
{
    decode_units<kDecDefaultSchedule, true>(b);
}

// Decoding against dictionaries (LizardB200_decompress_dict_*, Lizard_decompress_safe_usingDict / _continue): a kernel of its
// own as well, on the default schedule.  The Huffman pre-pass may run ahead of it (it reads only the compressed streams); the
// token pre-pass and the second generation never do, whatever the decode variant: both check offsets against the unit start.
__global__ void __launch_bounds__(kDecWarps * 32, 4) lizard_decode_dict_units_kernel(DecodeBatch b)
{
    decode_units<kDecDefaultSchedule, false, true>(b);
}

// Variable-length segments to their places in another arena (segment i: src_off[i], len[i] -> dst_off[i]): what the frame
// layer's "payloads back to back" (lib/lizard_frame.c:544-549 writes each block behind the previous one) is on the device
// when the units were produced at a fixed stride.  One CTA per segment, warps take 4 KiB tiles, destination-aligned 16-byte
// stores (lanes_copy_wide).  Segments with len <= 0 (failed units) are skipped.
__global__ void __launch_bounds__(256) lizard_gather_segments_kernel(const u8* src, const u64* src_off, const int* len,
                                                                      u8* dst, const u64* dst_off, u32 n)
{
    const u32 warp = threadIdx.x >> 5;
    for (u32 i = blockIdx.x; i < n; i += gridDim.x) {
        const int L = len[i];
        if (L <= 0) continue;
        const u8* s = src + src_off[i];
        u8* d = dst + dst_off[i];
        for (u32 t = warp * 4096u; t < (u32)L; t += 8u * 4096u) {
            const u32 part = (u32)L - t < 4096u ? (u32)L - t : 4096u;
            lanes_copy_wide<WarpLanes, true, true>(d + t, s + t, part, false);
        }
    }
}

// Second generation (decode2.cuh): one CTA of two warps per unit -- warp 0 parses (tokens -> records, literals stream staged
// through shared memory by TMA bulk copies), warp 1 copies (records -> output tile -> coalesced 16-byte stores).
// kStages = stages of 2 KiB in the literals ring.
template <u32 kStages> __global__ void __launch_bounds__(64, kStages >= 8 ? 8 : 11)
lizard_decode2_units_kernel(DecodeBatch b)
{
    __shared__ PairShared<kStages> ps;
    const u32 warp = threadIdx.x >> 5, lane = WarpLanes::lane();
    if (threadIdx.x == 0) {
        for (u32 i = 0; i < kStages; ++i) mbar_init(&ps.full_bar[i], 1);
        for (u32 i = 0; i < kBatchSlots; ++i) { mbar_init(&ps.pub_bar[i], 1); mbar_init(&ps.free_bar[i], 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (warp == 1) { copier_loop<kStages>(&ps); return; }
    u8* scratch = b.scratch + (size_t)blockIdx.x * kDecScratchPerWarp;
    if (lane == 0) ps.dws.big_table = reinterpret_cast<u16*>(scratch + 4 * kDecStreamScratch);
    __syncwarp();
    PairSink<kStages> sk;
    sk.init(&ps);
    for (;;) {
        u32 unit = 0;
        if (lane == 0) unit = atomicAdd(b.counter, 1u);
        unit = __shfl_sync(LZB_FULL, unit, 0);
        if (unit >= b.n_units) break;
        progress_wait(b.progress, unit, lane);
        u8* const dst = b.dst_base + b.dst_off[unit];
        sk.begin_unit(dst);
        const int r = decode_unit2<WarpLanes>(b.src_base + b.src_off[unit], b.src_len[unit], dst, b.dst_cap[unit], scratch,
                                              &ps.dws, sk, b.pre ? b.pre + unit : nullptr, b.arena);
        sk.drain();
        if (lane == 0) b.result[unit] = r;
        __syncwarp();
        progress_done(b.progress, unit, lane);
    }
    sk.finish_stream();
    sk.exit_copier();
}

typedef void (*DecodeKernel)(DecodeBatch);
DecodeKernel decode2_kernel(int stages) { return stages >= 8 ? lizard_decode2_units_kernel<8> : lizard_decode2_units_kernel<4>; }
DecodeKernel decode_kernel(int v)
{
    switch (v & 3) {
    case 0: return lizard_decode_units_kernel<0>;
    case 1: return lizard_decode_units_kernel<1>;
    case 2: return lizard_decode_units_kernel<2>;
    default: return lizard_decode_units_kernel<3>;
    }
}

thread_local std::string g_last_error;
thread_local int g_device = 0;
std::atomic<unsigned long long> g_launches{0};

struct DeviceBuffer {
    void* p = nullptr; size_t bytes = 0;
    cudaError_t reserve(size_t n) {
        if (n <= bytes) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; bytes = 0;
        size_t want = n + n / 4;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { e = cudaMalloc(&p, n); want = n; }
        if (e == cudaSuccess) bytes = want;
        return e;
    }
};
struct PinnedBuffer {
    void* p = nullptr; size_t bytes = 0;
    cudaError_t reserve(size_t n) {
        if (n <= bytes) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr; bytes = 0;
        cudaError_t e = cudaMallocHost(&p, n);
        if (e == cudaSuccess) bytes = n;
        return e;
    }
};

struct Context {
    std::mutex mu;
    bool ready = false, failed = false;
    int device = 0, sm_count = 0;
    cudaStream_t stream = nullptr, s_in = nullptr, s_out = nullptr;   // compute / H2D / D2H
    int decp_grid = 0, decd_grid = 0;         // grids of the partial-decode and dictionary-decode kernels
    int dec_grid = 0, dec_variant = 7;        // bits 0-1: schedule of the token loops, bit 2: Huffman pre-pass, bit 3: token pre-pass,
                                              // bit 4: second-generation kernel (parser + copier warp per unit)
    int dec2_grid = 0, dec2_stages = 4;
    int exp_ctas = 1;                         // CTAs per SM of the Huffman expand kernel
    DeviceBuffer pre_ws, pre_arena, pre_scratch, seq_ws, seq_recs;
    DeviceBuffer dec_scratch, enc_scratch, counters;
    u32 counter_slot = 0;
    // The kernels of one device share the library-owned workspaces (scratch per grid warp, pre-pass arena, sequence list).
    // Launches on ONE stream are ordered by the stream; a launch on a different stream than the previous one first waits
    // for the previous launch's completion event, so two streams never run on the same scratch at once.
    cudaEvent_t ws_done = nullptr; cudaStream_t ws_stream = nullptr; bool ws_used = false;
    // staging for the host-pointer entry points
    PinnedBuffer pin_in, pin_out, pin_tab, pin_flags;
    DeviceBuffer d_progress;
    DeviceBuffer d_in, d_out, d_tab, d_pack;
    DeviceBuffer fd_tab, fd_stage;            // tables and staged blocks of the device-memory frame calls (frame.inl)
    DeviceBuffer fa_tab, fa_stage;            // the same for LizardB200_decompressFramesAsync, kept apart: a captured graph holds them
    DeviceBuffer fc_tab, fc_stage;            // and for LizardB200_compressFramesAsync, apart from both for the same reason
    DeviceBuffer ds_tab, ds_stage, ds_seg;    // a LizardB200_decompressStream round's tables and staged blocks, its segment lists
    EncodeConfig enc_cfg;
};
Context g_ctx[kMaxDevices];

bool fail(const char* what, cudaError_t e)
{
    char buf[256];
    snprintf(buf, sizeof buf, "%s: %s", what, cudaGetErrorString(e));
    g_last_error = buf;
    return false;
}
#define CU_OK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { fail(#call, e_); return LIZARDB200_ERR_CUDA; } } while (0)

constexpr int kCounterSlots = 1024;

// bring the per-device context up (called with ctx.mu held)
int ensure_context(Context& c, int device)
{
    if (c.ready) { cudaSetDevice(device); return LIZARDB200_OK; }
    if (c.failed) return LIZARDB200_ERR_NO_DEVICE;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || device < 0 || device >= n) {
        c.failed = true;
        g_last_error = e != cudaSuccess ? std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e)
                                        : std::string("no such CUDA device");
        return LIZARDB200_ERR_NO_DEVICE;
    }
    cudaDeviceProp prop;
    if ((e = cudaSetDevice(device)) != cudaSuccess || (e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) {
        c.failed = true; fail("cudaSetDevice", e); return LIZARDB200_ERR_NO_DEVICE;
    }
    if (prop.major != 9 || prop.minor != 0) {   // the fatbin holds sm_90a SASS only
        c.failed = true;
        g_last_error = "liblizard_b200 is built for sm_90a (H100) only; found " + std::string(prop.name);
        return LIZARDB200_ERR_NO_DEVICE;
    }
    c.device = device;
    c.sm_count = prop.multiProcessorCount;
    if ((e = cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking)) != cudaSuccess ||
        (e = cudaStreamCreateWithFlags(&c.s_in, cudaStreamNonBlocking)) != cudaSuccess ||
        (e = cudaStreamCreateWithFlags(&c.s_out, cudaStreamNonBlocking)) != cudaSuccess) {
        c.failed = true; fail("cudaStreamCreate", e); return LIZARDB200_ERR_CUDA;
    }
    const size_t dec_smem = sizeof(DecWarpShared) * kDecWarps;
    if (const char* v = getenv("LIZARDB200_DEC_VARIANT")) c.dec_variant = atoi(v) & 31;
    // Shared memory and L1 share one 256 KB array per SM.  Left alone, the driver sizes the carve-out for as many CTAs as
    // the kernel's registers would allow, which leaves these kernels -- whose grids are sized by hand -- a 28 KB L1 for
    // hundreds of byte streams; ask for exactly what the resident CTAs use.
    auto carveout = [&](size_t smem_per_sm, const char* env) {
        if (const char* v = getenv(env)) return atoi(v);
        const size_t total = prop.sharedMemPerMultiprocessor;
        const size_t pct = (smem_per_sm * 100 + total - 1) / total;
        return (int)(pct > 100 ? 100 : pct);
    };
    e = cudaFuncSetAttribute(lizard_huf_expand_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(ExpWarpShared) * kExpWarps));
    {   // as many expand CTAs per SM as their tables allow, at most kExpCtasMax (1 GiB of 128 KiB blocks is ~14 warps of
        // bitstreams per SM; more CTAs than that find no work).  LIZARDB200_EXP_CTAS_PER_SM overrides.
        int fit = (int)(prop.sharedMemPerMultiprocessor / (sizeof(ExpWarpShared) * kExpWarps + 1024));
        if (fit < 1) fit = 1;
        c.exp_ctas = fit > (int)kExpCtasMax ? (int)kExpCtasMax : fit;
        if (const char* v = getenv("LIZARDB200_EXP_CTAS_PER_SM")) { const int w = atoi(v); if (w >= 1 && w <= fit) c.exp_ctas = w; }
    }
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(lizard_huf_expand_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                 carveout((size_t)c.exp_ctas * (sizeof(ExpWarpShared) * kExpWarps + 1024), "LIZARDB200_EXP_CARVEOUT"));
    if (e != cudaSuccess) { c.failed = true; fail("cudaFuncSetAttribute(expand)", e); return LIZARDB200_ERR_CUDA; }
    e = cudaSuccess;
    for (int v = 0; v < 4 && e == cudaSuccess; ++v)
        e = cudaFuncSetAttribute(decode_kernel(v), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dec_smem);
    if (e != cudaSuccess) { c.failed = true; fail("cudaFuncSetAttribute(decode)", e); return LIZARDB200_ERR_CUDA; }
    int per_sm = 0;
    for (int v = 0; v < 4; ++v) {          // all schedules share one launch shape (same registers and shared memory)
        int p = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&p, decode_kernel(v), kDecWarps * 32, dec_smem);
        if (v == 0 || p < per_sm) per_sm = p;
    }
    if (per_sm < 1) per_sm = 1;
    if (const char* v = getenv("LIZARDB200_DEC_CTAS_PER_SM")) {     // diagnostics: fewer units in flight (L2 residency sweeps)
        const int want = atoi(v);
        if (want >= 1 && want < per_sm) per_sm = want;
    }
    c.dec_grid = c.sm_count * per_sm;
    for (int v = 0; v < 4; ++v)
        cudaFuncSetAttribute(decode_kernel(v), cudaFuncAttributePreferredSharedMemoryCarveout,
                             carveout((size_t)per_sm * (dec_smem + 1024), "LIZARDB200_DEC_CARVEOUT"));
    {   // partial and dictionary decode: same launch shape and scratch as the full decode, kernels of their own
        const DecodeKernel own[2] = { lizard_decode_partial_units_kernel, lizard_decode_dict_units_kernel };
        int* const grid[2] = { &c.decp_grid, &c.decd_grid };
        for (int k = 0; k < 2; ++k) {
            int pp = 0;
            e = cudaFuncSetAttribute(own[k], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dec_smem);
            if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&pp, own[k], kDecWarps * 32, dec_smem);
            if (e != cudaSuccess) { c.failed = true; fail("cudaFuncSetAttribute(partial / dictionary decode)", e); return LIZARDB200_ERR_CUDA; }
            if (pp < 1) pp = 1;
            if (pp > per_sm) pp = per_sm;             // the scratch below is sized for dec_grid
            *grid[k] = c.sm_count * pp;
            cudaFuncSetAttribute(own[k], cudaFuncAttributePreferredSharedMemoryCarveout,
                                 carveout((size_t)pp * (dec_smem + 1024), "LIZARDB200_DEC_CARVEOUT"));
        }
    }
    {   // second generation: CTAs of two warps, static shared memory; as many per SM as fit (LIZARDB200_DEC2_CTAS_PER_SM caps it)
        if (const char* v = getenv("LIZARDB200_DEC2_STAGES")) c.dec2_stages = atoi(v) >= 8 ? 8 : 4;
        cudaFuncAttributes fa;
        int p2 = 0;
        if ((e = cudaFuncGetAttributes(&fa, decode2_kernel(c.dec2_stages))) != cudaSuccess) { c.failed = true; fail("cudaFuncGetAttributes(decode2)", e); return LIZARDB200_ERR_CUDA; }
        cudaFuncSetAttribute(decode2_kernel(c.dec2_stages), cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&p2, decode2_kernel(c.dec2_stages), 64, 0);
        if (p2 < 1) p2 = 1;
        if (const char* v = getenv("LIZARDB200_DEC2_CTAS_PER_SM")) { const int want = atoi(v); if (want >= 1 && want < p2) p2 = want; }
        c.dec2_grid = c.sm_count * p2;
        cudaFuncSetAttribute(decode2_kernel(c.dec2_stages), cudaFuncAttributePreferredSharedMemoryCarveout,
                             carveout((size_t)p2 * (fa.sharedSizeBytes + 1024), "LIZARDB200_DEC2_CARVEOUT"));
    }
    const size_t dec_scratch_units = (size_t)c.dec_grid * kDecWarps > (size_t)c.dec2_grid ? (size_t)c.dec_grid * kDecWarps : (size_t)c.dec2_grid;
    if ((e = c.dec_scratch.reserve(dec_scratch_units * kDecScratchPerWarp)) != cudaSuccess) {
        c.failed = true; fail("cudaMalloc(decode scratch)", e); return LIZARDB200_ERR_MEMORY;
    }
    if ((e = c.counters.reserve(kCounterSlots * sizeof(u32))) != cudaSuccess) {
        c.failed = true; fail("cudaMalloc(counters)", e); return LIZARDB200_ERR_MEMORY;
    }
    int er = encode_context_init(c.enc_cfg, c.sm_count, c.enc_scratch.p ? 0 : 0);
    if (er != 0) { c.failed = true; g_last_error = "encode kernel attribute setup failed"; return LIZARDB200_ERR_CUDA; }
    if ((e = c.enc_scratch.reserve(c.enc_cfg.scratch_bytes)) != cudaSuccess) {
        c.failed = true; fail("cudaMalloc(encode scratch)", e); return LIZARDB200_ERR_MEMORY;
    }
    c.ready = true;
    return LIZARDB200_OK;
}

// workspace hand-over between streams (see Context::ws_done)
// A stream being captured into a CUDA graph neither waits for nor records the hand-over event: an event recorded outside the
// capture cannot be waited on inside it, and the graph's launches are ordered by whoever launches the graph.
bool stream_capturing(cudaStream_t s)
{
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    return cudaStreamIsCapturing(s, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone;
}
void workspace_acquire(Context& c, cudaStream_t s)
{
    if (!c.ws_done) cudaEventCreateWithFlags(&c.ws_done, cudaEventDisableTiming);
    if (c.ws_used && c.ws_stream != s && c.ws_done && !stream_capturing(s)) cudaStreamWaitEvent(s, c.ws_done, 0);
}
void workspace_release(Context& c, cudaStream_t s)
{
    if (stream_capturing(s)) return;
    if (c.ws_done) cudaEventRecord(c.ws_done, s);
    c.ws_stream = s; c.ws_used = true;
}

// a fresh zeroed work-queue counter for one launch
u32* next_counter(Context& c, cudaStream_t s)
{
    u32* p = (u32*)c.counters.p + (c.counter_slot++ % kCounterSlots);
    cudaMemsetAsync(p, 0, sizeof(u32), s);
    return p;
}

// Huffman pre-pass (huf_expand.cuh / prepass.cuh): plan + expand kernels ahead of the token kernel, same stream.
// Worth two extra launches only for real batches; the streaming (progress) launches of the frame path keep the
// in-kernel expansion because their units arrive while the kernel is already running.
constexpr u32 kPrepassMinUnits = 32;
constexpr size_t kPrepassArenaPerUnit = 160u << 10;     // literals + flags of one 128 KiB block; overflow falls back in-kernel
constexpr size_t kPrepassArenaMax = (size_t)3 << 30;    // never more than this, however many units a batch has: the plan kernel
                                                        // hands out arena space by what the streams really need and leaves the
                                                        // rest to the in-kernel expansion (a batch of a million 4 KiB units must
                                                        // not ask for 160 KiB each)

// the pre-pass workspaces a batch of n units needs
void prepass_bytes(const Context& c, size_t n, size_t* ws_bytes, size_t* arena_bytes, size_t* scratch_bytes)
{
    *ws_bytes = 256 + n * sizeof(UnitPre) + 2 * n * sizeof(HufJob);
    *arena_bytes = n * kPrepassArenaPerUnit;
    if (*arena_bytes > kPrepassArenaMax) *arena_bytes = kPrepassArenaMax;
    *scratch_bytes = (size_t)c.sm_count * c.exp_ctas * kExpWarps * kExpJobs * sizeof(HufJobScratch);
}

int launch_prepass(Context& c, DecodeBatch& b, cudaStream_t s)
{
    const size_t n = b.n_units;
    size_t ws_bytes, arena_bytes, scratch_bytes;
    prepass_bytes(c, n, &ws_bytes, &arena_bytes, &scratch_bytes);
    if (ws_bytes > c.pre_ws.bytes || arena_bytes > c.pre_arena.bytes || scratch_bytes > c.pre_scratch.bytes) {
        // growing a workspace is the one place where an enqueue-only call synchronises (first call, or a larger batch than
        // ever before): an earlier launch may still be reading the buffers that are about to be replaced
        cudaStreamSynchronize(s);
        if (c.pre_ws.reserve(ws_bytes) != cudaSuccess || c.pre_arena.reserve(arena_bytes) != cudaSuccess ||
            c.pre_scratch.reserve(scratch_bytes) != cudaSuccess) {
            cudaGetLastError();                          // no room for the pre-pass: the token kernel expands the streams itself
            b.pre = nullptr; b.arena = nullptr;
            return LIZARDB200_OK;
        }
    }
    PrepassBatch p;
    p.src_base = b.src_base; p.src_off = b.src_off; p.src_len = b.src_len; p.n_units = b.n_units;
    p.hdr = (PreHeader*)c.pre_ws.p;
    p.pre = (UnitPre*)((u8*)c.pre_ws.p + 256);
    p.jobs = (HufJob*)((u8*)c.pre_ws.p + 256 + n * sizeof(UnitPre));
    p.arena = (u8*)c.pre_arena.p; p.arena_bytes = c.pre_arena.bytes;
    p.scratch = (HufJobScratch*)c.pre_scratch.p;
    CU_OK(cudaMemsetAsync(p.hdr, 0, sizeof(PreHeader), s));
    lizard_huf_plan_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(p);
    lizard_huf_expand_kernel<<<c.sm_count * c.exp_ctas, kExpWarps * 32, sizeof(ExpWarpShared) * kExpWarps, s>>>(p);
    g_launches += 2;
    CU_OK(cudaGetLastError());
    b.pre = p.pre; b.arena = p.arena;
    return LIZARDB200_OK;
}

// Token pre-pass (prepass.cuh: lizard_token_parse_kernel): one lane per unit parses the first inner block into sequence
// records; runs behind the Huffman pre-pass (it reads the expanded streams) and ahead of the token kernel.
constexpr size_t kSeqRecordsPerUnit = 2048;             // 32 KiB of records per unit on average; overflow falls back in-kernel

// the token pre-pass workspaces a batch of n units needs
void token_parse_bytes(size_t n, size_t* ws_bytes, size_t* rec_bytes)
{
    *ws_bytes = 64 + n * sizeof(UnitSeq);
    *rec_bytes = n * kSeqRecordsPerUnit * sizeof(PoolRun);
    if (*rec_bytes < ((size_t)64 << 20)) *rec_bytes = (size_t)64 << 20;
}

int launch_token_parse(Context& c, DecodeBatch& b, cudaStream_t s)
{
    const size_t n = b.n_units;
    size_t ws_bytes, rec_bytes;
    token_parse_bytes(n, &ws_bytes, &rec_bytes);
    if (ws_bytes > c.seq_ws.bytes || rec_bytes > c.seq_recs.bytes) {
        cudaStreamSynchronize(s);
        if (c.seq_ws.reserve(ws_bytes) != cudaSuccess || c.seq_recs.reserve(rec_bytes) != cudaSuccess) {
            cudaGetLastError();                          // optional pass: decode without it
            b.seq = nullptr; b.recs = nullptr;
            return LIZARDB200_OK;
        }
    }
    SeqBatch q;
    q.src_base = b.src_base; q.src_off = b.src_off; q.src_len = b.src_len; q.dst_cap = b.dst_cap; q.n_units = b.n_units;
    q.pre = b.pre; q.arena = b.arena;
    q.hdr = (SeqHeader*)c.seq_ws.p;
    q.seq = (UnitSeq*)((u8*)c.seq_ws.p + 64);
    q.recs = (PoolRun*)c.seq_recs.p; q.recs_cap = c.seq_recs.bytes / sizeof(PoolRun);
    CU_OK(cudaMemsetAsync(q.hdr, 0, sizeof(SeqHeader), s));
    lizard_token_parse_kernel<<<(unsigned)((n + 31) / 32), 32, 0, s>>>(q);
    g_launches++;
    CU_OK(cudaGetLastError());
    b.seq = q.seq; b.recs = q.recs;
    return LIZARDB200_OK;
}

// true when launch_decode of n units (no progress) finds every pre-pass workspace it will use large enough, so that it
// neither synchronises nor allocates (the condition for capturing it in a CUDA graph)
bool decode_workspace_fits(const Context& c, u32 n)
{
    if ((c.dec_variant & 4) && n >= kPrepassMinUnits) {
        size_t ws, arena, scratch;
        prepass_bytes(c, n, &ws, &arena, &scratch);
        if (ws > c.pre_ws.bytes || arena > c.pre_arena.bytes || scratch > c.pre_scratch.bytes) return false;
    }
    if ((c.dec_variant & 8) && !(c.dec_variant & 16) && n >= kPrepassMinUnits) {
        size_t ws, recs;
        token_parse_bytes(n, &ws, &recs);
        if (ws > c.seq_ws.bytes || recs > c.seq_recs.bytes) return false;
    }
    return true;
}

int launch_decode(Context& c, const void* dSrc, const u64* dSrcOff, const u32* dSrcLen,
                  void* dDst, const u64* dDstOff, const u32* dDstCap, int* dResult, u32 n, cudaStream_t s,
                  const Progress* pg = nullptr)
{
    if (n == 0) return LIZARDB200_OK;
    workspace_acquire(c, s);
    struct Release { Context& c; cudaStream_t s; ~Release() { workspace_release(c, s); } } release_on_exit{c, s};
    DecodeBatch b;
    if (pg) b.progress = *pg; else memset(&b.progress, 0, sizeof b.progress);
    b.src_base = (const u8*)dSrc; b.src_off = dSrcOff; b.src_len = dSrcLen;
    b.dst_base = (u8*)dDst; b.dst_off = dDstOff; b.dst_cap = dDstCap;
    b.result = dResult; b.n_units = n;
    b.scratch = (u8*)c.dec_scratch.p;
    b.counter = next_counter(c, s);
    b.pre = nullptr; b.arena = nullptr; b.seq = nullptr; b.recs = nullptr; b.target = nullptr;
    if ((c.dec_variant & 4) && pg == nullptr && n >= kPrepassMinUnits) {
        int st = launch_prepass(c, b, s);
        if (st != LIZARDB200_OK) return st;
    }
    if ((c.dec_variant & 8) && !(c.dec_variant & 16) && pg == nullptr && n >= kPrepassMinUnits) {
        int st = launch_token_parse(c, b, s);
        if (st != LIZARDB200_OK) return st;
    }
    if (c.dec_variant & 16) {
        const int grid2 = (int)n < c.dec2_grid ? (int)n : c.dec2_grid;
        decode2_kernel(c.dec2_stages)<<<grid2, 64, 0, s>>>(b);
        g_launches++;
        CU_OK(cudaGetLastError());
        return LIZARDB200_OK;
    }
    u32 warps_needed = n;
    int grid = (int)((warps_needed + kDecWarps - 1) / kDecWarps);
    if (grid > c.dec_grid) grid = c.dec_grid;
    decode_kernel(c.dec_variant)<<<grid, kDecWarps * 32, sizeof(DecWarpShared) * kDecWarps, s>>>(b);
    g_launches++;
    CU_OK(cudaGetLastError());
    return LIZARDB200_OK;
}

// Lizard_decompress_safe_partial for every unit, dTarget[i] = unit i's targetOutputSize: one launch of the partial kernel,
// whatever the decode variant (no pre-pass, no second generation).
int launch_decode_partial(Context& c, const void* dSrc, const u64* dSrcOff, const u32* dSrcLen,
                          void* dDst, const u64* dDstOff, const u32* dDstCap, const int* dTarget, int* dResult, u32 n,
                          cudaStream_t s)
{
    if (n == 0) return LIZARDB200_OK;
    workspace_acquire(c, s);
    struct Release { Context& c; cudaStream_t s; ~Release() { workspace_release(c, s); } } release_on_exit{c, s};
    DecodeBatch b;
    memset(&b, 0, sizeof b);
    b.src_base = (const u8*)dSrc; b.src_off = dSrcOff; b.src_len = dSrcLen;
    b.dst_base = (u8*)dDst; b.dst_off = dDstOff; b.dst_cap = dDstCap;
    b.result = dResult; b.n_units = n; b.target = dTarget;
    b.scratch = (u8*)c.dec_scratch.p;
    b.counter = next_counter(c, s);
    int grid = (int)((n + kDecWarps - 1) / kDecWarps);
    if (grid > c.decp_grid) grid = c.decp_grid;
    lizard_decode_partial_units_kernel<<<grid, kDecWarps * 32, sizeof(DecWarpShared) * kDecWarps, s>>>(b);
    g_launches++;
    CU_OK(cudaGetLastError());
    return LIZARDB200_OK;
}

// Lizard_decompress_safe_usingDict for every unit against the dictionary dDictLen[i] bytes at dDict + dDictOff[i]: one launch
// of the dictionary kernel, behind the Huffman pre-pass under the rule of launch_decode.  dDictReach: see DecodeBatch.
int launch_decode_dict(Context& c, const void* dSrc, const u64* dSrcOff, const u32* dSrcLen,
                       void* dDst, const u64* dDstOff, const u32* dDstCap, const void* dDict, const u64* dDictOff,
                       const u32* dDictLen, const u32* dDictReach, int* dResult, u32 n, cudaStream_t s)
{
    if (n == 0) return LIZARDB200_OK;
    workspace_acquire(c, s);
    struct Release { Context& c; cudaStream_t s; ~Release() { workspace_release(c, s); } } release_on_exit{c, s};
    DecodeBatch b;
    memset(&b, 0, sizeof b);
    b.src_base = (const u8*)dSrc; b.src_off = dSrcOff; b.src_len = dSrcLen;
    b.dst_base = (u8*)dDst; b.dst_off = dDstOff; b.dst_cap = dDstCap;
    b.result = dResult; b.n_units = n;
    b.dict_base = (const u8*)dDict; b.dict_off = dDictOff; b.dict_len = dDictLen; b.dict_reach = dDictReach;
    b.scratch = (u8*)c.dec_scratch.p;
    b.counter = next_counter(c, s);
    if ((c.dec_variant & 4) && n >= kPrepassMinUnits) {
        int st = launch_prepass(c, b, s);
        if (st != LIZARDB200_OK) return st;
    }
    int grid = (int)((n + kDecWarps - 1) / kDecWarps);
    if (grid > c.decd_grid) grid = c.decd_grid;
    lizard_decode_dict_units_kernel<<<grid, kDecWarps * 32, sizeof(DecWarpShared) * kDecWarps, s>>>(b);
    g_launches++;
    CU_OK(cudaGetLastError());
    return LIZARDB200_OK;
}

// levels the encoder implements: the parsers of level_params(), lowestPrice (23-25, 43-45) and the binary-tree optimal parser
// with LZ4 codewords (18, 19, 39), each in a kernel of its own
bool enc_level_ok(int level) { return level_params(level).parser != kParserUnsupported || lp_level(level) || opt_level(level); }

int launch_encode(Context& c, const void* dSrc, const u64* dSrcOff, const u32* dSrcLen,
                  void* dDst, const u64* dDstOff, const u32* dDstCap, int* dResult, u32 n, int level, cudaStream_t s,
                  const Progress* pg = nullptr, const FramePack* fp = nullptr, bool big_units = true)
{
    if (n == 0) return LIZARDB200_OK;
    if (!enc_level_ok(level)) { g_last_error = "compression level not implemented on the GPU"; return LIZARDB200_ERR_LEVEL; }
    workspace_acquire(c, s);
    struct Release { Context& c; cudaStream_t s; ~Release() { workspace_release(c, s); } } release_on_exit{c, s};
    EncodeBatch b;
    if (pg) b.progress = *pg; else memset(&b.progress, 0, sizeof b.progress);
    if (fp) b.pack = *fp; else memset(&b.pack, 0, sizeof b.pack);
    b.src_base = (const u8*)dSrc; b.src_off = dSrcOff; b.src_len = dSrcLen;
    b.dst_base = (u8*)dDst; b.dst_off = dDstOff; b.dst_cap = dDstCap;
    b.result = dResult; b.n_units = n; b.level = level;
    b.scratch = (u8*)c.enc_scratch.p;
    b.counter = next_counter(c, s);
    int launches = 0;
    cudaError_t e = lp_level(level) ? lp_encode_launch(c.enc_cfg, b, s, &launches, big_units)
                  : opt_level(level) ? opt_encode_launch(c.enc_cfg, b, s, &launches, big_units)
                  : encode_launch(c.enc_cfg, b, s, &launches);
    g_launches += (unsigned long long)launches;
    if (e != cudaSuccess) { fail("encode launch", e); return LIZARDB200_ERR_CUDA; }
    return LIZARDB200_OK;
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// levels with a dictionary path: the parsers that search a loaded dictionary through the table Lizard_loadDict fills
// (dict_parser(), encode_core.cuh; kernel: encode_dict_kernel.cuh)
bool enc_dict_level_ok(int level) { return dict_parser(level_params(level)); }
const char* const kNoDictLevel = "compression with a dictionary is implemented on the GPU at levels 13-17, 21-22, 34-38 and 41-42 only "
                                 "(the hashChain and priceFast parsers)";

int launch_encode_dict(Context& c, const void* dSrc, const u64* dSrcOff, const u32* dSrcLen,
                       void* dDst, const u64* dDstOff, const u32* dDstCap, const void* dDict, const u64* dDictOff,
                       const u32* dDictLen, int* dResult, u32 n, int level, cudaStream_t s)
{
    if (!enc_dict_level_ok(level)) { g_last_error = kNoDictLevel; return LIZARDB200_ERR_LEVEL; }
    if (n == 0) return LIZARDB200_OK;
    if (dict_shape(c.enc_cfg, n).max_slots < 1) {
        g_last_error = "the encode workspace has no room for a dictionary slot beside the warps' scratch";
        return LIZARDB200_ERR_MEMORY;
    }
    workspace_acquire(c, s);
    struct Release { Context& c; cudaStream_t s; ~Release() { workspace_release(c, s); } } release_on_exit{c, s};
    EncodeBatch b;
    memset(&b, 0, sizeof b);
    b.src_base = (const u8*)dSrc; b.src_off = dSrcOff; b.src_len = dSrcLen;
    b.dst_base = (u8*)dDst; b.dst_off = dDstOff; b.dst_cap = dDstCap;
    b.result = dResult; b.n_units = n; b.level = level;
    b.scratch = (u8*)c.enc_scratch.p;
    b.counter = next_counter(c, s);
    int launches = 0;
    const cudaError_t e = dict_encode_launch(c.enc_cfg, b, (const u8*)dDict, dDictOff, dDictLen, s, &launches);
    g_launches += (unsigned long long)launches;
    if (e != cudaSuccess) { fail("dictionary encode launch", e); return LIZARDB200_ERR_CUDA; }
    return LIZARDB200_OK;
}

// LizardB200_compress_dict_batch: every unit and its dictionary staged so that their relative placement survives: a unit that
// touches or overlaps its dictionary (the prefix layout, or an input inside its dictionary) is staged together with it as one
// range; other dictionaries are staged once per (end address, size).  Only the last 2^24 bytes of a dictionary are staged.
int run_host_compress_dict(const void* const* src, const int* srcSize, void* const* dst, const int* dstCap,
                           const void* const* dict, const int* dictSize, int* result, int n, int level)
{
    if (n < 0 || (n > 0 && (!src || !srcSize || !dst || !dstCap || !result || !dict || !dictSize))) return LIZARDB200_ERR_ARGUMENT;
    Context& c = g_ctx[g_device];
    std::lock_guard<std::mutex> lock(c.mu);
    int st = ensure_context(c, g_device);
    if (st != LIZARDB200_OK) return st;
    if (!enc_dict_level_ok(level)) { g_last_error = kNoDictLevel; return LIZARDB200_ERR_LEVEL; }
    if (n == 0) return LIZARDB200_OK;
    struct Range { const u8* lo; size_t bytes; u64 at; };
    std::vector<Range> ranges;
    std::map<std::pair<const u8*, u32>, size_t> shared;              // (end, size) -> range of a dictionary staged alone
    std::vector<size_t> unit_range(n), dict_range(n);
    std::vector<u32> dlen(n);
    std::vector<const u8*> dptr(n);
    size_t distinct = 0, out_total = 0;                               // dictionaries of 8 bytes or more; smaller ones share a slot
    bool small = false;
    std::vector<u64> out_off(n);
    for (int i = 0; i < n; ++i) {
        if (srcSize[i] < 0 || dstCap[i] < 0 || dictSize[i] < 0 || (srcSize[i] && !src[i]) || (dictSize[i] && !dict[i]))
            return LIZARDB200_ERR_ARGUMENT;
        const u8* s0 = (const u8*)src[i];
        const u8* d0 = (const u8*)dict[i];
        u32 dl = (u32)dictSize[i];
        if (dl > kDictSize) { d0 += dl - kDictSize; dl = kDictSize; }
        dptr[i] = d0; dlen[i] = dl;
        out_off[i] = out_total; out_total += align_up((size_t)dstCap[i] + 32, 16);
        small = small || dl < 8;
        if (dl && s0 <= d0 + dl && s0 + srcSize[i] >= d0) {
            const u8* lo = s0 < d0 ? s0 : d0;
            const u8* hi = s0 + srcSize[i] > d0 + dl ? s0 + srcSize[i] : d0 + dl;
            unit_range[i] = dict_range[i] = ranges.size();
            ranges.push_back(Range{lo, (size_t)(hi - lo), 0});
            distinct += dl >= 8;
            continue;
        }
        unit_range[i] = ranges.size();
        ranges.push_back(Range{s0, (size_t)srcSize[i], 0});
        if (!dl) continue;
        auto it = shared.find({d0 + dl, dl});
        if (it == shared.end()) {
            it = shared.emplace(std::make_pair(d0 + dl, dl), ranges.size()).first;
            ranges.push_back(Range{d0, dl, 0});
            distinct += dl >= 8;
        }
        dict_range[i] = it->second;
    }
    const DictShape shape = dict_shape(c.enc_cfg, (u32)n);
    if (distinct + (small ? 1 : 0) > shape.max_slots) {
        char buf[200];
        snprintf(buf, sizeof buf, "%zu distinct dictionaries of 8 bytes or more in one call; the encode workspace holds %u for %d units",
                 distinct, shape.max_slots - (small ? 1 : 0), n);
        g_last_error = buf;
        return LIZARDB200_ERR_MEMORY;
    }
    size_t in_total = 0;
    for (Range& r : ranges) { r.at = in_total; in_total = align_up(in_total + r.bytes + 16, 16); }
    const size_t tab_bytes = (size_t)n * (8 + 8 + 8 + 4 + 4 + 4 + 4);
    CU_OK(c.pin_in.reserve(in_total));
    CU_OK(c.pin_tab.reserve(tab_bytes));
    CU_OK(c.d_in.reserve(in_total));
    CU_OK(c.d_out.reserve(out_total));
    CU_OK(c.d_tab.reserve(tab_bytes));
    CU_OK(c.pin_out.reserve(out_total));
    u64* t_in_off = (u64*)c.pin_tab.p;
    u64* t_out_off = t_in_off + n;
    u64* t_dict_off = t_out_off + n;
    u32* t_in_len = (u32*)(t_dict_off + n);
    u32* t_out_cap = t_in_len + n;
    u32* t_dict_len = t_out_cap + n;
    int* t_res = (int*)(t_dict_len + n);
    for (const Range& r : ranges) if (r.bytes) memcpy((u8*)c.pin_in.p + r.at, r.lo, r.bytes);
    for (int i = 0; i < n; ++i) {
        const Range& ur = ranges[unit_range[i]];
        t_in_off[i] = ur.at + (u64)((const u8*)src[i] - ur.lo);
        t_out_off[i] = out_off[i];
        t_in_len[i] = (u32)srcSize[i]; t_out_cap[i] = (u32)dstCap[i];
        t_dict_len[i] = dlen[i];
        t_dict_off[i] = dlen[i] ? ranges[dict_range[i]].at + (u64)(dptr[i] - ranges[dict_range[i]].lo) : 0;
    }
    u8* dtab = (u8*)c.d_tab.p;
    cudaStream_t s = c.stream;
    CU_OK(cudaMemcpyAsync(c.d_in.p, c.pin_in.p, in_total, cudaMemcpyHostToDevice, s));
    CU_OK(cudaMemcpyAsync(dtab, c.pin_tab.p, tab_bytes - (size_t)n * 4, cudaMemcpyHostToDevice, s));
    const u64* d_in_off = (const u64*)dtab;
    const u64* d_out_off = d_in_off + n;
    const u64* d_dict_off = d_out_off + n;
    const u32* d_in_len = (const u32*)(d_dict_off + n);
    const u32* d_out_cap = d_in_len + n;
    const u32* d_dict_len = d_out_cap + n;
    int* d_res = (int*)(d_dict_len + n);
    st = launch_encode_dict(c, c.d_in.p, d_in_off, d_in_len, c.d_out.p, d_out_off, d_out_cap, c.d_in.p, d_dict_off, d_dict_len,
                            d_res, (u32)n, level, s);
    if (st != LIZARDB200_OK) return st;
    CU_OK(cudaMemcpyAsync(t_res, d_res, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    CU_OK(cudaMemcpyAsync(c.pin_out.p, c.d_out.p, out_total, cudaMemcpyDeviceToHost, s));
    CU_OK(cudaStreamSynchronize(s));
    for (int i = 0; i < n; ++i) {
        result[i] = t_res[i];
        if (result[i] > 0) memcpy(dst[i], (u8*)c.pin_out.p + out_off[i], (size_t)t_res[i]);
    }
    return LIZARDB200_OK;
}

// Shared body of the host-pointer batch calls: stage inputs + tables, run, fetch results + outputs.
// `target` (decode only): per-unit targetOutputSize of a partial decode, null for a full one.
// `dict` / `dictSize` (decode only): per-unit dictionary of Lizard_decompress_safe_usingDict, null for none.  Only the bytes
// a unit's matches can reach are staged (dict_window of its level), once per dictionary end address; a negative size gives
// the unit -1 without decoding it.  `dictReach`: the units' reaches, if not the ones their dictionaries imply (_continue).
template <bool kCompress>
int run_host_batch(const void* const* src, const int* srcSize, void* const* dst, const int* dstCap,
                   int* result, int n, int level, const int* target = nullptr,
                   const void* const* dict = nullptr, const int* dictSize = nullptr, const u32* dictReach = nullptr)
{
    if (n < 0 || (n > 0 && (!src || !srcSize || !dst || !dstCap || !result))) return LIZARDB200_ERR_ARGUMENT;
    if (n == 0) return LIZARDB200_OK;
    Context& c = g_ctx[g_device];
    std::lock_guard<std::mutex> lock(c.mu);
    int st = ensure_context(c, g_device);
    if (st != LIZARDB200_OK) return st;
    if (kCompress && !enc_level_ok(level)) {
        g_last_error = "compression level not implemented on the GPU";
        return LIZARDB200_ERR_LEVEL;
    }

    // layout: every unit 16-byte aligned in both arenas
    std::vector<u64> in_off(n), out_off(n);
    size_t in_total = 0, out_total = 0;
    for (int i = 0; i < n; ++i) {
        if (srcSize[i] < 0 || dstCap[i] < 0) return LIZARDB200_ERR_ARGUMENT;
        in_off[i] = in_total;   in_total += align_up((size_t)srcSize[i] + 16, 16);
        out_off[i] = out_total; out_total += align_up((size_t)dstCap[i] + 32, 16);
    }
    // dictionaries go behind the inputs, one staged copy per dictionary end address, as long as the longest reach of a unit
    // that uses it
    const int nd = dict ? n : 0;
    std::vector<u32> dict_avail(nd), dict_rch(nd);
    std::vector<u64> dict_at(nd);                                 // arena offset of unit i's first readable dictionary byte
    struct Staged { const u8* end; u32 bytes; u64 at; };
    std::vector<Staged> staged;
    if (dict) {
        std::unordered_map<const u8*, size_t> slot;
        std::vector<size_t> unit_slot(n);
        for (int i = 0; i < n; ++i) {
            dict_avail[i] = dict_rch[i] = 0; dict_at[i] = 0;
            if (dictSize[i] <= 0 || srcSize[i] < 1) continue;
            if (!dict[i]) return LIZARDB200_ERR_ARGUMENT;
            const u8* end = (const u8*)dict[i] + dictSize[i];
            const int lv = ((const u8*)src[i])[0];
            const u32 win = (lv >= (int)kMinLevel && lv <= (int)kMaxLevel) ? dict_window(lv) : 0u;
            dict_avail[i] = (u32)dictSize[i] < win ? (u32)dictSize[i] : win;
            dict_rch[i] = dictReach ? dictReach[i] : dict_reach((u32)dictSize[i], end == (const u8*)dst[i]);
            auto it = slot.find(end);
            if (it == slot.end()) { it = slot.emplace(end, staged.size()).first; staged.push_back(Staged{end, 0, 0}); }
            unit_slot[i] = it->second;
            if (staged[it->second].bytes < dict_avail[i]) staged[it->second].bytes = dict_avail[i];
        }
        for (Staged& d : staged) { d.at = in_total; in_total = align_up(in_total + d.bytes + 16, 16); }
        for (int i = 0; i < n; ++i)
            if (dict_avail[i]) { const Staged& d = staged[unit_slot[i]]; dict_at[i] = d.at + d.bytes - dict_avail[i]; }
    }
    const size_t tab_bytes = (size_t)n * (8 + 4 + 8 + 4 + (target ? 4 : 0) + (dict ? 8 + 4 + 4 : 0) + 4);
    CU_OK(c.pin_in.reserve(in_total));
    CU_OK(c.pin_tab.reserve(tab_bytes));
    CU_OK(c.d_in.reserve(in_total));
    CU_OK(c.d_out.reserve(out_total));
    CU_OK(c.d_tab.reserve(tab_bytes));
    CU_OK(c.pin_out.reserve(out_total));

    u8* tab = (u8*)c.pin_tab.p;
    u64* t_in_off = (u64*)tab;
    u64* t_out_off = t_in_off + n;
    u32* t_in_len = (u32*)(t_out_off + n);
    u32* t_out_cap = t_in_len + n;
    u64* t_dict_off = (u64*)(t_out_cap + n);                      // 8-byte aligned: 24 bytes per unit in front of it
    u32* t_dict_len = (u32*)(t_dict_off + nd);
    u32* t_dict_reach = t_dict_len + nd;
    int* t_target = (int*)(t_dict_reach + nd);
    int* t_res = t_target + (target ? n : 0);
    for (int i = 0; i < n; ++i) {
        memcpy((u8*)c.pin_in.p + in_off[i], src[i], (size_t)srcSize[i]);
        t_in_off[i] = in_off[i]; t_out_off[i] = out_off[i];
        t_in_len[i] = (u32)srcSize[i]; t_out_cap[i] = (u32)dstCap[i];
        if (target) t_target[i] = target[i];
        if (dict) { t_dict_off[i] = dict_at[i]; t_dict_len[i] = dict_avail[i]; t_dict_reach[i] = dict_rch[i]; }
    }
    for (const Staged& d : staged) memcpy((u8*)c.pin_in.p + d.at, d.end - d.bytes, d.bytes);
    u8* dtab = (u8*)c.d_tab.p;
    cudaStream_t s = c.stream;
    CU_OK(cudaMemcpyAsync(c.d_in.p, c.pin_in.p, in_total, cudaMemcpyHostToDevice, s));
    CU_OK(cudaMemcpyAsync(dtab, tab, tab_bytes - (size_t)n * 4, cudaMemcpyHostToDevice, s));
    const u64* d_in_off = (const u64*)dtab;
    const u64* d_out_off = d_in_off + n;
    const u32* d_in_len = (const u32*)(d_out_off + n);
    const u32* d_out_cap = d_in_len + n;
    const u64* d_dict_off = (const u64*)(d_out_cap + n);
    const u32* d_dict_len = (const u32*)(d_dict_off + nd);
    const u32* d_dict_reach = d_dict_len + nd;
    const int* d_target = (const int*)(d_dict_reach + nd);
    int* d_res = (int*)d_target + (target ? n : 0);
    if (kCompress) {
        bool big = false;                                         // a unit of several inner blocks (lowestPrice big slots)
        for (int i = 0; i < n; ++i) big = big || (u32)srcSize[i] > kBlockSize;
        st = launch_encode(c, c.d_in.p, d_in_off, d_in_len, c.d_out.p, d_out_off, d_out_cap, d_res, (u32)n, level, s, nullptr, nullptr, big);
    }
    else if (target) st = launch_decode_partial(c, c.d_in.p, d_in_off, d_in_len, c.d_out.p, d_out_off, d_out_cap, d_target, d_res, (u32)n, s);
    else if (dict) st = launch_decode_dict(c, c.d_in.p, d_in_off, d_in_len, c.d_out.p, d_out_off, d_out_cap, c.d_in.p, d_dict_off,
                                           d_dict_len, d_dict_reach, d_res, (u32)n, s);
    else           st = launch_decode(c, c.d_in.p, d_in_off, d_in_len, c.d_out.p, d_out_off, d_out_cap, d_res, (u32)n, s);
    if (st != LIZARDB200_OK) return st;
    CU_OK(cudaMemcpyAsync(t_res, d_res, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    CU_OK(cudaMemcpyAsync(c.pin_out.p, c.d_out.p, out_total, cudaMemcpyDeviceToHost, s));
    CU_OK(cudaStreamSynchronize(s));
    for (int i = 0; i < n; ++i) {
        result[i] = dict && dictSize[i] < 0 ? -1 : t_res[i];
        if (result[i] > 0) memcpy(dst[i], (u8*)c.pin_out.p + out_off[i], (size_t)t_res[i]);
    }
    return LIZARDB200_OK;
}

}  // namespace

// ================================================================================================
extern "C" {

int Lizard_versionNumber(void) { return LIZARD_B200_VERSION_NUMBER; }
int Lizard_compressBound(int isize) { return compress_bound(isize); }

int Lizard_sizeofState(int level)
{
    // lib/lizard_compress.c:311-323: struct + hash table + chain table + 5 stream buffers + Huffman bound.
    // The device keeps its own state; the figure is reproduced so callers that malloc it keep working.
    if (level > (int)kMaxLevel) level = kMaxLevel;
    if (level < (int)kMinLevel) level = kDefaultLevel;
    static const unsigned char hash_log[40] = {12,18,18,18,18,18,18,18,18,23, 14,14,18,18,23,23,23,23,23,23,
                                               12,18,14,18,18,18,18,18,18,23, 14,14,18,18,23,23,23,23,23,23};
    static const unsigned char content_log[40] = {0,0,0,16,16,16,16,16,17,17, 0,22,22,22,22,22,23,23,23,25,
                                                  0,0,0,0,16,16,16,16,16,17, 0,22,22,22,22,22,22,23,23,25};
    const size_t struct_bytes = 2384;   // sizeof(Lizard_stream_t) on LP64 (SURVEY.md section 8 a2)
    const size_t huf_bound = 129 + (kBlockSizePad + (kBlockSizePad >> 8) + 8);
    size_t total = struct_bytes + (size_t(4) << hash_log[level - 10]) + (size_t(4) << content_log[level - 10])
                 + 5 * (size_t)kBlockSizePad + huf_bound;
    return (int)total;
}

int LizardB200_setDevice(int device)
{
    if (device < 0 || device >= kMaxDevices) return LIZARDB200_ERR_ARGUMENT;
    g_device = device;
    Context& c = g_ctx[device];
    std::lock_guard<std::mutex> lock(c.mu);
    return ensure_context(c, device);
}
int LizardB200_available(void)
{
    Context& c = g_ctx[g_device];
    std::lock_guard<std::mutex> lock(c.mu);
    return ensure_context(c, g_device) == LIZARDB200_OK;
}
const char* LizardB200_lastError(void) { return g_last_error.c_str(); }
unsigned long long LizardB200_launchCount(void) { return g_launches.load(); }

// diagnostics: the encode kernel's launch shape for a level, LIZARDB200_ENC_SHAPE applied (pure host arithmetic, needs no
// device): warps per CTA, how many of them keep their hash table in shared memory, CTAs per SM, dynamic shared bytes per CTA
int LizardB200_encodeShape(int level, int* warpsPerCta, int* smemTables, int* ctasPerSM, int* smemBytes)
{
    if (lp_level(level) || opt_level(level)) {   // the lowestPrice / optimal kernels: no shared-memory tables, static histograms
        const LpShape sh = lp_level(level) ? lp_shape() : opt_shape();
        if (warpsPerCta) *warpsPerCta = sh.warps;
        if (smemTables) *smemTables = 0;
        if (ctasPerSM) *ctasPerSM = sh.ctas_per_sm;
        if (smemBytes) *smemBytes = 0;
        return LIZARDB200_OK;
    }
    const LevelParams lp = level_params(level);
    if (lp.parser == kParserUnsupported) return LIZARDB200_ERR_LEVEL;
    const EncodeShape sh = encode_shape_in_effect(lp);
    if (warpsPerCta) *warpsPerCta = sh.warps;
    if (smemTables) *smemTables = sh.smem_tables;
    if (ctasPerSM) *ctasPerSM = sh.ctas_per_sm;
    if (smemBytes) *smemBytes = (int)sh.smem;
    return LIZARDB200_OK;
}

// diagnostics (tools/dec_bench.py): batch schedule of the decode kernel on this thread's device, see lizard_decode_units_kernel
int LizardB200_setDecodeVariant(int variant)
{
    Context& c = g_ctx[g_device];
    std::lock_guard<std::mutex> lk(c.mu);
    int st = ensure_context(c, g_device);
    if (st != LIZARDB200_OK) return st;
    c.dec_variant = variant & 31;
    return LIZARDB200_OK;
}

int LizardB200_decompress_device(const void* dSrc, const uint64_t* dSrcOff, const uint32_t* dSrcLen,
                                 void* dDst, const uint64_t* dDstOff, const uint32_t* dDstCap,
                                 int* dResult, unsigned nUnits, void* stream)
{
    Context& c = g_ctx[g_device];
    std::lock_guard<std::mutex> lock(c.mu);
    int st = ensure_context(c, g_device);
    if (st != LIZARDB200_OK) return st;
    return launch_decode(c, dSrc, (const u64*)dSrcOff, dSrcLen, dDst, (const u64*)dDstOff, dDstCap, dResult, nUnits, (cudaStream_t)stream);
}
int LizardB200_decompress_partial_device(const void* dSrc, const uint64_t* dSrcOff, const uint32_t* dSrcLen,
                                         void* dDst, const uint64_t* dDstOff, const uint32_t* dDstCap,
                                         const int* dTarget, int* dResult, unsigned nUnits, void* stream)
{
    if (nUnits > 0 && !dTarget) return LIZARDB200_ERR_ARGUMENT;
    Context& c = g_ctx[g_device];
    std::lock_guard<std::mutex> lock(c.mu);
    int st = ensure_context(c, g_device);
    if (st != LIZARDB200_OK) return st;
    return launch_decode_partial(c, dSrc, (const u64*)dSrcOff, dSrcLen, dDst, (const u64*)dDstOff, dDstCap, dTarget, dResult, nUnits,
                                 (cudaStream_t)stream);
}
int LizardB200_decompress_dict_device(const void* dSrc, const uint64_t* dSrcOff, const uint32_t* dSrcLen,
                                      void* dDst, const uint64_t* dDstOff, const uint32_t* dDstCap,
                                      const void* dDict, const uint64_t* dDictOff, const uint32_t* dDictLen,
                                      int* dResult, unsigned nUnits, void* stream)
{
    if (nUnits > 0 && (!dDictOff || !dDictLen)) return LIZARDB200_ERR_ARGUMENT;
    Context& c = g_ctx[g_device];
    std::lock_guard<std::mutex> lock(c.mu);
    int st = ensure_context(c, g_device);
    if (st != LIZARDB200_OK) return st;
    return launch_decode_dict(c, dSrc, (const u64*)dSrcOff, dSrcLen, dDst, (const u64*)dDstOff, dDstCap, dDict, (const u64*)dDictOff,
                              dDictLen, nullptr, dResult, nUnits, (cudaStream_t)stream);
}
int LizardB200_compress_device(const void* dSrc, const uint64_t* dSrcOff, const uint32_t* dSrcLen,
                               void* dDst, const uint64_t* dDstOff, const uint32_t* dDstCap,
                               int* dResult, unsigned nUnits, int level, void* stream)
{
    Context& c = g_ctx[g_device];
    std::lock_guard<std::mutex> lock(c.mu);
    int st = ensure_context(c, g_device);
    if (st != LIZARDB200_OK) return st;
    return launch_encode(c, dSrc, (const u64*)dSrcOff, dSrcLen, dDst, (const u64*)dDstOff, dDstCap, dResult, nUnits, level, (cudaStream_t)stream);
}

int LizardB200_compress_dict_device(const void* dSrc, const uint64_t* dSrcOff, const uint32_t* dSrcLen,
                                    void* dDst, const uint64_t* dDstOff, const uint32_t* dDstCap,
                                    const void* dDict, const uint64_t* dDictOff, const uint32_t* dDictLen,
                                    int* dResult, unsigned nUnits, int level, void* stream)
{
    if (nUnits > 0 && (!dDictOff || !dDictLen)) return LIZARDB200_ERR_ARGUMENT;
    Context& c = g_ctx[g_device];
    std::lock_guard<std::mutex> lock(c.mu);
    int st = ensure_context(c, g_device);
    if (st != LIZARDB200_OK) return st;
    return launch_encode_dict(c, dSrc, (const u64*)dSrcOff, dSrcLen, dDst, (const u64*)dDstOff, dDstCap, dDict, (const u64*)dDictOff,
                              dDictLen, dResult, nUnits, level, (cudaStream_t)stream);
}

int LizardB200_gather_device(const void* dSrc, const uint64_t* dSrcOff, const int* dLen,
                             void* dDst, const uint64_t* dDstOff, unsigned nUnits, void* stream)
{
    if (nUnits == 0) return LIZARDB200_OK;
    if (!dSrc || !dSrcOff || !dLen || !dDst || !dDstOff) return LIZARDB200_ERR_ARGUMENT;
    Context& c = g_ctx[g_device];
    std::lock_guard<std::mutex> lock(c.mu);
    int st = ensure_context(c, g_device);
    if (st != LIZARDB200_OK) return st;
    const unsigned grid = nUnits < (unsigned)c.sm_count * 8u ? nUnits : (unsigned)c.sm_count * 8u;
    lizard_gather_segments_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const u8*)dSrc, (const u64*)dSrcOff, dLen,
                                                                            (u8*)dDst, (const u64*)dDstOff, nUnits);
    g_launches++;
    CU_OK(cudaGetLastError());
    return LIZARDB200_OK;
}

int LizardB200_decompress_batch(const void* const* src, const int* cSize, void* const* dst, const int* dstCap,
                                int* result, int n)
{
    return run_host_batch<false>(src, cSize, dst, dstCap, result, n, 0);
}
int LizardB200_decompress_partial_batch(const void* const* src, const int* cSize, void* const* dst, const int* dstCap,
                                        const int* targetOutputSize, int* result, int n)
{
    if (n > 0 && !targetOutputSize) return LIZARDB200_ERR_ARGUMENT;
    return run_host_batch<false>(src, cSize, dst, dstCap, result, n, 0, targetOutputSize);
}
int LizardB200_decompress_dict_batch(const void* const* src, const int* cSize, void* const* dst, const int* dstCap,
                                     const void* const* dict, const int* dictSize, int* result, int n)
{
    if (n > 0 && (!dict || !dictSize)) return LIZARDB200_ERR_ARGUMENT;
    return run_host_batch<false>(src, cSize, dst, dstCap, result, n, 0, nullptr, dict, dictSize);
}
int LizardB200_compress_batch(const void* const* src, const int* srcSize, void* const* dst, const int* dstCap,
                              int* result, int n, int level)
{
    return run_host_batch<true>(src, srcSize, dst, dstCap, result, n, level);
}

int LizardB200_compress_dict_batch(const void* const* src, const int* srcSize, void* const* dst, const int* dstCap,
                                   const void* const* dict, const int* dictSize, int* result, int n, int level)
{
    return run_host_compress_dict(src, srcSize, dst, dstCap, dict, dictSize, result, n, level);
}


// Contiguous host buffers (what a frame writer / file splitter has).  Copies go straight from / to the
// caller's memory (fast when it is pinned); tables are built on the host.
int LizardB200_compress_blocks(const void* src, size_t srcSize, int blockSize,
                               void* dst, size_t dstStride, int dstCapacityEach, int* result, int level)
{
    if (blockSize <= 0 || dstCapacityEach < 0 || (srcSize && (!src || !dst || !result))) return LIZARDB200_ERR_ARGUMENT;
    const size_t n = (srcSize + (size_t)blockSize - 1) / (size_t)blockSize;
    if (n == 0) return LIZARDB200_OK;
    if ((size_t)dstCapacityEach > dstStride) return LIZARDB200_ERR_ARGUMENT;
    Context& c = g_ctx[g_device];
    std::lock_guard<std::mutex> lock(c.mu);
    int st = ensure_context(c, g_device);
    if (st != LIZARDB200_OK) return st;
    if (!enc_level_ok(level)) { g_last_error = "compression level not implemented on the GPU"; return LIZARDB200_ERR_LEVEL; }
    const size_t tab_bytes = n * (8 + 4 + 8 + 4 + 4);
    CU_OK(c.pin_tab.reserve(tab_bytes));
    CU_OK(c.d_tab.reserve(tab_bytes));
    CU_OK(c.d_in.reserve(srcSize + 64));
    CU_OK(c.d_out.reserve(n * dstStride + 64));
    u64* t_in_off = (u64*)c.pin_tab.p; u64* t_out_off = t_in_off + n;
    u32* t_in_len = (u32*)(t_out_off + n); u32* t_out_cap = t_in_len + n; int* t_res = (int*)(t_out_cap + n);
    for (size_t i = 0; i < n; ++i) {
        t_in_off[i] = i * (size_t)blockSize; t_out_off[i] = i * dstStride;
        const size_t left = srcSize - i * (size_t)blockSize;
        t_in_len[i] = (u32)(left < (size_t)blockSize ? left : (size_t)blockSize);
        t_out_cap[i] = (u32)dstCapacityEach;
    }
    cudaStream_t s = c.stream;
    u8* dtab = (u8*)c.d_tab.p;
    // the whole strided region is copied back: what the units do not write (the slack behind each compressed block) must
    // not be bytes of an earlier call
    CU_OK(cudaMemsetAsync(c.d_out.p, 0, n * dstStride, s));
    CU_OK(cudaMemcpyAsync(c.d_in.p, src, srcSize, cudaMemcpyHostToDevice, s));
    CU_OK(cudaMemcpyAsync(dtab, c.pin_tab.p, tab_bytes - n * 4, cudaMemcpyHostToDevice, s));
    const u64* d_in_off = (const u64*)dtab; const u64* d_out_off = d_in_off + n;
    const u32* d_in_len = (const u32*)(d_out_off + n); const u32* d_out_cap = d_in_len + n; int* d_res = (int*)(d_out_cap + n);
    st = launch_encode(c, c.d_in.p, d_in_off, d_in_len, c.d_out.p, d_out_off, d_out_cap, d_res, (u32)n, level, s, nullptr, nullptr,
                       (size_t)blockSize > kBlockSize);
    if (st != LIZARDB200_OK) return st;
    CU_OK(cudaMemcpyAsync(t_res, d_res, n * 4, cudaMemcpyDeviceToHost, s));
    CU_OK(cudaMemcpyAsync(dst, c.d_out.p, n * dstStride, cudaMemcpyDeviceToHost, s));
    CU_OK(cudaStreamSynchronize(s));
    memcpy(result, t_res, n * 4);
    return LIZARDB200_OK;
}

int LizardB200_decompress_blocks(const void* src, size_t srcStride, const int* compressedSize, size_t nUnits,
                                 void* dst, int blockSize, int* result)
{
    if (blockSize <= 0 || (nUnits && (!src || !dst || !result || !compressedSize))) return LIZARDB200_ERR_ARGUMENT;
    const size_t n = nUnits;
    if (n == 0) return LIZARDB200_OK;
    Context& c = g_ctx[g_device];
    std::lock_guard<std::mutex> lock(c.mu);
    int st = ensure_context(c, g_device);
    if (st != LIZARDB200_OK) return st;
    const size_t tab_bytes = n * (8 + 4 + 8 + 4 + 4);
    CU_OK(c.pin_tab.reserve(tab_bytes));
    CU_OK(c.d_tab.reserve(tab_bytes));
    CU_OK(c.d_in.reserve(n * srcStride + 64));
    CU_OK(c.d_out.reserve(n * (size_t)blockSize + 64));
    u64* t_in_off = (u64*)c.pin_tab.p; u64* t_out_off = t_in_off + n;
    u32* t_in_len = (u32*)(t_out_off + n); u32* t_out_cap = t_in_len + n; int* t_res = (int*)(t_out_cap + n);
    for (size_t i = 0; i < n; ++i) {
        if (compressedSize[i] < 0 || (size_t)compressedSize[i] > srcStride) return LIZARDB200_ERR_ARGUMENT;
        t_in_off[i] = i * srcStride; t_out_off[i] = i * (size_t)blockSize;
        t_in_len[i] = (u32)compressedSize[i]; t_out_cap[i] = (u32)blockSize;
    }
    cudaStream_t s = c.stream;
    u8* dtab = (u8*)c.d_tab.p;
    CU_OK(cudaMemsetAsync(c.d_out.p, 0, n * (size_t)blockSize, s));      // short or failed units leave gaps: zeros, not stale data
    CU_OK(cudaMemcpyAsync(c.d_in.p, src, n * srcStride, cudaMemcpyHostToDevice, s));
    CU_OK(cudaMemcpyAsync(dtab, c.pin_tab.p, tab_bytes - n * 4, cudaMemcpyHostToDevice, s));
    const u64* d_in_off = (const u64*)dtab; const u64* d_out_off = d_in_off + n;
    const u32* d_in_len = (const u32*)(d_out_off + n); const u32* d_out_cap = d_in_len + n; int* d_res = (int*)(d_out_cap + n);
    st = launch_decode(c, c.d_in.p, d_in_off, d_in_len, c.d_out.p, d_out_off, d_out_cap, d_res, (u32)n, s);
    if (st != LIZARDB200_OK) return st;
    CU_OK(cudaMemcpyAsync(t_res, d_res, n * 4, cudaMemcpyDeviceToHost, s));
    CU_OK(cudaMemcpyAsync(dst, c.d_out.p, n * (size_t)blockSize, cudaMemcpyDeviceToHost, s));
    CU_OK(cudaStreamSynchronize(s));
    memcpy(result, t_res, n * 4);
    return LIZARDB200_OK;
}

int Lizard_decompress_safe(const char* src, char* dst, int compressedSize, int maxDecompressedSize)
{
    // lib/lizard_decompress.c:139: inputSize < 1 -> 0 before anything is read
    if (compressedSize < 1) return 0;
    if (maxDecompressedSize < 0) return -1;
    const void* s = src; void* d = dst; int r = -1;
    int st = LizardB200_decompress_batch(&s, &compressedSize, &d, &maxDecompressedSize, &r, 1);
    return st == LIZARDB200_OK ? r : st;
}

int Lizard_compress(const char* src, char* dst, int srcSize, int maxDstSize, int level)
{
    if (srcSize < 0 || maxDstSize < 0) return 0;
    // lib/lizard_compress.c:303-308 Lizard_verifyCompressionLevel
    if (level > (int)kMaxLevel) level = kMaxLevel;
    if (level < (int)kMinLevel) level = kDefaultLevel;
    const void* s = src; void* d = dst; int r = 0;
    int st = LizardB200_compress_batch(&s, &srcSize, &d, &maxDstSize, &r, 1, level);
    return st == LIZARDB200_OK ? r : 0;
}
int Lizard_compress_extState(void* state, const char* src, char* dst, int srcSize, int maxDstSize, int level)
{
    if (((size_t)state & (sizeof(void*) - 1)) != 0) return 0;   // lib/lizard_compress.c:586
    return Lizard_compress(src, dst, srcSize, maxDstSize, level);
}

// ---- the rest of lib/dll/liblizard.def: what callers of the block API link against -------------------------------------
// Stream OBJECTS are functional (the reference's frame layer creates one per context and hands it to
// Lizard_compress_extState, lib/lizard_frame.c:379-401, 436-451); the device keeps the real state, so the object records the
// level and what Lizard_loadDict was given.  Dictionary and streamed DECODING run on the GPU (Lizard_decompress_safe_usingDict,
// _continue).  On the compress side, a stream's FIRST Lizard_compress_continue runs on the GPU: after Lizard_loadDict it is the
// dictionary path (hashChain and priceFast levels), on a fresh or reset stream it is Lizard_compress (lib/lizard_compress.c:557).  Any later
// _continue would need the tables the previous call left behind, and Lizard_saveDict moves them: both fail with the reference's
// failure value 0, never with a CPU code path.
struct Lizard_stream_s {
    size_t allocatedMemory; int compressionLevel;
    int state;                        // kStreamFresh, kStreamDict (Lizard_loadDict ran) or kStreamSpent
    const char* dict; int dictSize;   // as given to Lizard_loadDict
};
enum { kStreamFresh = 0, kStreamDict = 1, kStreamSpent = 2 };
struct Lizard_streamDecode_s {                                   // lib/lizard_common.h:195-200
    const u8* externalDict; size_t extDictSize;
    const u8* prefixEnd; size_t prefixSize;
};
static const char* const kNoStreaming = "streaming compression across calls (linked blocks, Lizard_saveDict) is not implemented on the GPU path";

Lizard_stream_t* Lizard_createStream(int level)            // lib/lizard_compress.c:392-397
{
    if (level > (int)kMaxLevel) level = kMaxLevel;
    if (level < (int)kMinLevel) level = kDefaultLevel;
    Lizard_stream_t* p = (Lizard_stream_t*)malloc(sizeof(Lizard_stream_t));
    if (p) { p->allocatedMemory = sizeof(Lizard_stream_t); p->compressionLevel = level; p->state = kStreamFresh; p->dict = nullptr; p->dictSize = 0; }
    return p;
}
int Lizard_freeStream(Lizard_stream_t* p) { free(p); return 0; }              // :417-423
Lizard_stream_t* Lizard_resetStream(Lizard_stream_t* p, int level)            // :401-414
{
    if (!p) return Lizard_createStream(level);
    if (level > (int)kMaxLevel) level = kMaxLevel;
    if (level < (int)kMinLevel) level = kDefaultLevel;
    p->compressionLevel = level;
    p->state = kStreamFresh; p->dict = nullptr; p->dictSize = 0;
    return p;
}
int Lizard_loadDict(Lizard_stream_t* p, const char* dictionary, int dictSize)   // :426-437
{
    if (dictSize > (int)kDictSize) { dictionary += dictSize - (int)kDictSize; dictSize = (int)kDictSize; }
    p->state = dictSize >= 0 ? kStreamDict : kStreamSpent;
    p->dict = dictionary; p->dictSize = dictSize;
    return dictSize;
}
int Lizard_saveDict(Lizard_stream_t* p, char*, int) { p->state = kStreamSpent; g_last_error = kNoStreaming; return 0; }
int Lizard_compress_continue(Lizard_stream_t* p, const char* src, char* dst, int srcSize, int maxDstSize)   // :550-580
{
    const int state = p->state;
    p->state = kStreamSpent;
    if (state == kStreamFresh) return Lizard_compress(src, dst, srcSize, maxDstSize, p->compressionLevel);
    if (state != kStreamDict) { g_last_error = kNoStreaming; return 0; }
    if (srcSize < 0 || maxDstSize < 0) return 0;
    const void* s = src; void* d = dst; const void* dict = p->dict; int r = 0;
    const int st = LizardB200_compress_dict_batch(&s, &srcSize, &d, &maxDstSize, &dict, &p->dictSize, &r, 1, p->compressionLevel);
    return st == LIZARDB200_OK ? r : 0;
}

Lizard_streamDecode_t* Lizard_createStreamDecode(void) { return (Lizard_streamDecode_t*)calloc(1, sizeof(Lizard_streamDecode_t)); }
int Lizard_freeStreamDecode(Lizard_streamDecode_t* p) { free(p); return 0; }
int Lizard_setStreamDecode(Lizard_streamDecode_t* p, const char* dict, int dictSize)   // lib/lizard_decompress.c:303-310
{
    p->prefixSize = (size_t)dictSize;
    p->prefixEnd = (const u8*)dict + dictSize;
    p->externalDict = nullptr;
    p->extDictSize = 0;
    return 1;
}

namespace {
// One unit against the window [ext, ext + extSize) followed by [pre, pre + preSize) in front of dst (the window of
// Lizard_decompress_safe_continue, lib/lizard_decompress.c:322-344): the bytes its matches can reach are gathered into one
// buffer and decoded as an external dictionary whose reach is the whole window.
int decompress_window(const char* src, char* dst, int compressedSize, int maxOut, const u8* ext, size_t extSize,
                      const u8* pre, size_t preSize)
{
    if (compressedSize < 1) return 0;
    if (maxOut < 0) return -1;
    const int lv = (u8)src[0];
    const size_t total = extSize + preSize;
    const size_t win = (lv >= (int)kMinLevel && lv <= (int)kMaxLevel) ? dict_window(lv) : 0;
    const size_t keep = total < win ? total : win;
    std::vector<u8> buf(keep + 1);
    const size_t from_pre = keep < preSize ? keep : preSize, from_ext = keep - from_pre;
    if (from_ext) memcpy(buf.data(), ext + extSize - from_ext, from_ext);
    if (from_pre) memcpy(buf.data() + from_ext, pre + preSize - from_pre, from_pre);
    // the reference checks offsets against the whole window unless the external part alone is 2^24 bytes or more; from a
    // window of 2^24 bytes on no offset can fail the check either
    const u32 reach = total >= ((size_t)1 << 24) ? kDictUnchecked : (u32)total;
    const void* s = src; void* d = dst; const void* dict = buf.data(); const int dsize = (int)keep; int r = -1;
    int st = run_host_batch<false>(&s, &compressedSize, &d, &maxOut, &r, 1, 0, nullptr, &dict, &dsize, &reach);
    return st == LIZARDB200_OK ? r : st;
}
}  // namespace

int Lizard_decompress_safe_continue(Lizard_streamDecode_t* p, const char* src, char* dst, int compressedSize, int maxOutputSize)
{
    int r;
    if (p->prefixEnd == (const u8*)dst) {
        r = decompress_window(src, dst, compressedSize, maxOutputSize, p->externalDict, p->extDictSize,
                              p->prefixEnd - p->prefixSize, p->prefixSize);
        if (r <= 0) return r;
        p->prefixSize += (size_t)r;
        p->prefixEnd += r;
    } else {
        p->extDictSize = p->prefixSize;
        p->externalDict = p->prefixEnd - p->extDictSize;
        r = decompress_window(src, dst, compressedSize, maxOutputSize, p->externalDict, p->extDictSize, nullptr, 0);
        if (r <= 0) return r;
        p->prefixSize = (size_t)r;
        p->prefixEnd = (const u8*)dst + r;
    }
    return r;
}
int Lizard_decompress_safe_partial(const char* src, char* dst, int compressedSize, int targetOutputSize, int maxDecompressedSize)
{
    // same argument handling as Lizard_decompress_safe (lib/lizard_decompress.c:139, 272-275)
    if (compressedSize < 1) return 0;
    if (maxDecompressedSize < 0) return -1;
    const void* s = src; void* d = dst; int r = -1;
    int st = LizardB200_decompress_partial_batch(&s, &compressedSize, &d, &maxDecompressedSize, &targetOutputSize, &r, 1);
    return st == LIZARDB200_OK ? r : st;
}
int Lizard_decompress_safe_usingDict(const char* src, char* dst, int compressedSize, int maxDecompressedSize,
                                     const char* dictStart, int dictSize)
{
    // lib/lizard_decompress.c:351-360: without a dictionary this is Lizard_decompress_safe
    if (dictSize == 0) return Lizard_decompress_safe(src, dst, compressedSize, maxDecompressedSize);
    if (dictSize < 0) return -1;
    if (compressedSize < 1) return 0;
    if (maxDecompressedSize < 0) return -1;
    const void* s = src; void* d = dst; const void* dict = dictStart; int r = -1;
    int st = LizardB200_decompress_dict_batch(&s, &compressedSize, &d, &maxDecompressedSize, &dict, &dictSize, &r, 1);
    return st == LIZARDB200_OK ? r : st;
}

}  // extern "C"

#include "frame.inl"
