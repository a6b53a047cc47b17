// common.cuh -- shared definitions for the sm_90a kernels of libh3dgs.so.
// Constants are the published algorithm's (see oracle/oracle.c and DESIGN.md
// "recalled constants"; the hierarchy-rasterizer source is absent from the reference checkout).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include "../../include/h3dgs.h"

namespace h3dgs {

constexpr float kNearPlane = 0.2f;
constexpr float kFovClamp = 1.3f;
constexpr float kDilation = 0.3f;
constexpr float kLambdaFloor = 0.1f;
constexpr int kTile = H3DGS_TILE;
constexpr int kTilePixels = kTile * kTile;
constexpr float kAlphaCap = 0.99f;
constexpr float kAlphaSkip = 1.0f / 255.0f;
constexpr float kTStop = 0.0001f;
constexpr float kWEps = 0.0000001f;
constexpr uint32_t kKidsMask = 0xFFFFFu;
constexpr int kClampShift = 20;
// per-tile sorted record copy: kids saturate at 16 bits (65535, the largest count the blend kernels see), the upper
// half holds the reach mask of the tile's sixteen 4x4-pixel blocks (binning.cu::block_mask16)
constexpr uint32_t kSortedKidsMask = 0xFFFFu;
constexpr int kBlockShift = 16;

// Per-Gaussian projected record: 3 x float4 = 48 B, 16-B aligned, so a batch of
// records is one contiguous cp.async.bulk (TMA) transfer.
//   a = {x, y, conic.x, conic.y}
//   b = {conic.z, opacity, t, kbits}     kbits: bits 0..19 num_node_kids (k <= 1 stored as 1, saturated at 2^20 - 1),
//                                        20..22 SH clamp flags; the per-tile
//                                        SORTED copy instead holds kids in bits 0..15 (saturated at 65535) and, in bits 16..31, the mask
//                                        of the tile's sixteen 4x4-pixel blocks this entry can reach (binning.cu)
//   c = {r, g, b, invdepth}
struct __align__(16) Record { float4 a, b, c; };
static_assert(sizeof(Record) == 48, "record must be 48 bytes");

__host__ __device__ inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// ---- state buffer layouts (byte offsets inside the three alloc'd buffers) ----
struct GeomLayout {
    size_t depths, tiles_touched, offsets, rank_mask, records, scan_temp, total;
    size_t scan_temp_bytes;
};
struct BinLayout {
    size_t keys_unsorted, keys_sorted, vals_unsorted, vals_sorted, sort_temp, sorted_records, total;
    size_t sort_temp_bytes;
};
struct ImgLayout {
    size_t final_T, n_contrib, ranges, tile_max_contrib, tile_count, scan_info, total;
};
// written by tile_scan_kernel; read back by the host in exact mode (the one num_rendered round trip).
// overflow: capacity mode only -- the frame does not fit (bin_capacity, sort_capacity); all ranges are
// emptied and key emission is skipped, so every later stage is a no-op for this frame.
struct ScanInfo { uint32_t D, max_count, overflow, prefilter_bad; };   // prefilter_bad: K1 culled a point although prefiltered was set
// largest per-tile list the shared-memory sort handles; bigger lists fall back to the global CUB sort
constexpr int kTileSortCap = 8192;

GeomLayout geom_layout(int P);
BinLayout bin_layout(int64_t D);
ImgLayout img_layout(int W, int H);

// per-stage event timing (api.cu); no-ops unless h3dgs_profile_enable(1)
void prof_begin(int stage, cudaStream_t s);
void prof_end(int stage, cudaStream_t s);
struct ProfScope {
    int stage; cudaStream_t s;
    ProfScope(int st, cudaStream_t ss) : stage(st), s(ss) { prof_begin(stage, s); }
    ~ProfScope() { prof_end(stage, s); }
};

// 64-B pinned host scratch per device for the small D2H read-backs (num_rendered, cut size): a
// pageable destination makes cudaMemcpyAsync stage through the driver (api.cu)
int pinned_scratch(void** out);

// error plumbing (api.cu)
void set_error(const char* fmt, ...);
extern int64_t g_launches;

#define H3_CUDA(call)                                                                      \
    do {                                                                                   \
        cudaError_t e__ = (call);                                                          \
        if (e__ != cudaSuccess) {                                                          \
            h3dgs::set_error("%s failed at %s:%d: %s", #call, __FILE__, __LINE__,          \
                             cudaGetErrorString(e__));                                     \
            return H3DGS_ECUDA;                                                            \
        }                                                                                  \
    } while (0)

// after a kernel launch: count it, catch launch errors; in debug mode also sync
#define H3_LAUNCHED(name, debug, stream)                                                   \
    do {                                                                                   \
        h3dgs::g_launches++;                                                               \
        cudaError_t e__ = cudaGetLastError();                                              \
        if (e__ == cudaSuccess && (debug)) e__ = cudaStreamSynchronize(stream);            \
        if (e__ != cudaSuccess) {                                                          \
            h3dgs::set_error("kernel %s failed: %s", name, cudaGetErrorString(e__));       \
            return H3DGS_ECUDA;                                                            \
        }                                                                                  \
    } while (0)

// ---- stage entry points (one per .cu file) ----
int launch_preprocess(const h3dgs_raster_args& a, int32_t* radii, float* depths, uint32_t* tiles_touched,
                      uint8_t* rank_mask, Record* records, uint32_t* tile_count, ScanInfo* info, cudaStream_t s);
int launch_tile_scan(const h3dgs_raster_args& a, const uint32_t* tile_count, uint32_t* ranges, ScanInfo* info,
                     uint32_t cap_entries, uint32_t cap_list, cudaStream_t s);
int launch_tile_binning(const h3dgs_raster_args& a, const int32_t* radii, const float* depths, const Record* records,
                        int64_t D, uint32_t max_count, uint8_t* bin, const BinLayout& bl, const uint32_t* ranges,
                        const ScanInfo* info, uint32_t* tile_count, cudaStream_t s);
int launch_preprocess_color(const h3dgs_raster_args& a, const int32_t* radii, const uint32_t* tiles_touched,
                            Record* records, cudaStream_t s);
int launch_sh_backward(const h3dgs_raster_args& a, const int32_t* radii, const uint8_t* rank_mask, const Record* records,
                       const float* accum, float* dL_dmeans3D, float* dL_dsh, cudaStream_t s);
int launch_scan(const uint32_t* in, uint32_t* out, int n, void* temp, size_t temp_bytes, cudaStream_t s, bool debug);
size_t scan_temp_bytes(int n);
size_t sort_temp_bytes(int64_t n);
int launch_binning(const h3dgs_raster_args& a, const int32_t* radii, const float* depths, const uint32_t* offsets,
                   const Record* records, int64_t D, uint8_t* bin, const BinLayout& bl, uint32_t* ranges,
                   cudaStream_t s);
int launch_render_forward(const h3dgs_raster_args& a, const uint32_t* ranges, const Record* sorted_records,
                          float* out_color, float* out_invdepth, float* final_T, uint32_t* n_contrib,
                          uint32_t* tile_max_contrib, cudaStream_t s);   // peer mode: pixels go to a.peer_image[*]
int launch_render_backward(const h3dgs_raster_args& a, const uint32_t* ranges, const Record* sorted_records,
                           const uint32_t* point_list, const float* final_T, const uint32_t* n_contrib,
                           const uint32_t* tile_max_contrib, const float* dL_dcolor, const float* dL_dinvdepth,
                           float* accum /*[P][10] zeroed*/, cudaStream_t s);
int launch_preprocess_backward(const h3dgs_raster_args& a, const int32_t* radii, const uint8_t* rank_mask, const Record* records,
                               const float* accum, float* dL_dmeans3D, float* dL_dmeans2D, float* dL_dsh,
                               float* dL_dcolors, float* dL_dopacities, float* dL_dscales, float* dL_drots,
                               float* dL_dcov3D, cudaStream_t s);

#ifdef __CUDACC__
// Pixel layout of the blend kernels: CTA = 128 threads = 4 warps; warp q owns the 8x8 quadrant
// (q & 1, q >> 1) of the 16x16 tile; lane l owns column (l & 7) and the two rows 2*(l >> 3), +1.
__device__ __forceinline__ void quad_pixel(int tile_x, int tile_y, int warp, int lane, int& px, int& py0) {
    px = tile_x * kTile + 8 * (warp & 1) + (lane & 7);
    py0 = tile_y * kTile + 8 * (warp >> 1) + 2 * (lane >> 3);
}

// Group walk (render_*_kernel<..., GROUPS = true>): the same quadrant per warp, but lanes 8 g .. 8 g + 7 own the
// 4x4-pixel block g = (g & 1, g >> 1) of it -- lane k of the group: column (k & 3), rows 2 (k >> 2), +1 -- and each
// 8-lane group walks only the entries whose block bit is set (common.cuh kBlockShift, binning.cu::block_mask16).
__device__ __forceinline__ void group_pixel(int tile_x, int tile_y, int warp, int lane, int& px, int& py0) {
    const int g = lane >> 3, k = lane & 7;
    px = tile_x * kTile + 8 * (warp & 1) + 4 * (g & 1) + (k & 3);
    py0 = tile_y * kTile + 8 * (warp >> 1) + 4 * (g >> 1) + 2 * (k >> 2);
}
// Each kernel defaults to the walk that is faster for it on the H100 (DESIGN.md §3.1): the backward walks per group (on
// config #3 it runs 27 % fewer loop iterations than the one-list-per-warp walk, at 2.3x the gradient reductions), the
// forward walks one list per warp.  H3DGS_GROUPWALK=1 forces the group walk in both kernels, H3DGS_GROUPWALK=0 one list per warp in both; the two walks
// compute the same results bit for bit.
inline bool use_group_walk(bool dflt) {
    const char* e = getenv("H3DGS_GROUPWALK");
    return (e && e[0]) ? e[0] != '0' : dflt;
}

#endif

// peer mode (h3dgs_raster_args.peer_count > 1): device pointers into the memory of every rank, by value in the kernel parameters
struct PeerPtrs { void* p[H3DGS_MAX_PEERS]; int n; };
inline PeerPtrs peer_ptrs(void* const* src, int n) {
    PeerPtrs r; r.n = n > 1 ? n : 0;
    for (int k = 0; k < H3DGS_MAX_PEERS; k++) r.p[k] = (k < r.n) ? src[k] : nullptr;
    return r;
}
// block-cyclic ownership of rendered rows in peer mode: blocks of 2^shift rows dealt round-robin to the ranks
struct RowCycle { int shift, world, rank; };
inline RowCycle row_cycle(const h3dgs_raster_args& a) {
    RowCycle c; c.world = a.peer_count > 1 ? a.peer_count : 0; c.rank = a.shard_index; c.shift = a.grad_cyclic_log2;
    return c;
}
// number of rows (padded to whole blocks) rank `c.rank` owns out of P
inline int cyclic_local_rows(const RowCycle& c, int P) {
    const int blocks = (P + (1 << c.shift) - 1) >> c.shift;
    return ((blocks + c.world - 1 - c.rank) / c.world) << c.shift;
}
#ifdef __CUDACC__
// local (dense) index -> rendered row of the owning rank
__device__ __forceinline__ int cyclic_row(const RowCycle& c, int local) {
    return ((((local >> c.shift) * c.world + c.rank)) << c.shift) + (local & ((1 << c.shift) - 1));
}
__device__ __forceinline__ bool cyclic_owned(const RowCycle& c, int row) { return ((row >> c.shift) % c.world) == c.rank; }
#endif

#ifdef __CUDACC__
// Peer mode, backward phase 2 (K9): every rank's phase 1 has left its PARTIAL [P][10] sums in its own accumulator and
// pushed the rows other ranks own into the owners' staging areas (preprocess_backward.cu::peer_push_kernel).  The owner
// of row i adds its own partial row and the staged rows of the ranks whose tile rows the Gaussian touches (rank_mask,
// written by K1), in rank order: the reduce-scatter of the per-Gaussian sums -- sparse (a Gaussian touches 1-2 tile
// rows on average), independent of arrival order, all loads local.  (A first version PULLED the rows with loads over
// NVLink inside K9: 8-byte remote reads serialise on the link latency; remote stores are posted.)
struct StagePtrs { const float* own; const float* stage; int n, rank; size_t slot_floats; };   // stage: [n][P][10] on this rank
// pairs [2 * first, 2 * first + 2 * NPAIR) of accumulator row i, summed over the ranks of `mask`
template <int NPAIR>
__device__ __forceinline__ void gather_accum_pairs(const StagePtrs& sp, uint32_t mask, int i, int first, float (&out)[2 * NPAIR]) {
#pragma unroll
    for (int k = 0; k < 2 * NPAIR; k++) out[k] = 0.f;
#pragma unroll
    for (int r = 0; r < H3DGS_MAX_PEERS; r++) {
        if (r < sp.n && ((mask >> r) & 1u)) {
            const float* row = (r == sp.rank ? sp.own : sp.stage + (size_t)r * sp.slot_floats) + (size_t)i * 10 + 2 * first;
#pragma unroll
            for (int k = 0; k < NPAIR; k++) {
                const float2 v = __ldcg(reinterpret_cast<const float2*>(row + 2 * k));      // L2: written by a peer through NVLink
                out[2 * k] += v.x; out[2 * k + 1] += v.y;
            }
        }
    }
}
#endif
inline StagePtrs stage_ptrs(const h3dgs_raster_args& a, const float* accum) {
    StagePtrs sp; sp.own = accum; sp.n = a.peer_count > 1 ? a.peer_count : 0; sp.rank = a.shard_index;
    sp.stage = sp.n ? static_cast<const float*>(a.peer_stage[a.shard_index]) : nullptr;
    sp.slot_floats = (size_t)a.P * 10;
    return sp;
}
int launch_peer_push(const h3dgs_raster_args& a, const uint8_t* rank_mask, const float* accum, cudaStream_t s);

// Loop statistics of the blend kernels, HOST EMULATION BUILD ONLY (tests/emul; the emulator is single-threaded):
// 0 bwd warp iterations | 1 bwd iterations left at the no-taker vote | 2 bwd pixel-entries taken | 3 bwd group-iterations
// with an entry | 4 of those without any taker | 8 fwd warp iterations | 9 fwd pixel-entries taken | 10 fwd group-iterations
#ifdef H3_SIMT_EMU
extern long long g_emu_stats[16];
#define H3_STAT(i, n) (h3dgs::g_emu_stats[i] += (n))
#else
#define H3_STAT(i, n) ((void)0)
#endif

// accum row layout (floats): 0,1 dmean2D.xy | 2,3,4 dconic | 5 dopacity | 6,7,8 dcolor | 9 dinvdepth
constexpr int kAccum = 10;

}  // namespace h3dgs

#ifdef __CUDACC__
#include "pair_math.cuh"      // packed FP32x2 arithmetic of the blend kernels
#endif
