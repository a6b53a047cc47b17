// render_forward.cu -- K6: per-tile front-to-back alpha blend (replaces FORWARD::render).
// Semantics per oracle/oracle.c::oracle_render_forward.
//
// Design: one CTA (128 threads, two pixels each) per 16x16 tile.  The tile's depth-sorted records were
// materialised contiguously by binning.cu, so a batch of 256 records is ONE 12 KB
// cp.async.bulk (TMA) transfer into shared memory, double-buffered behind an
// mbarrier; no thread spends registers or LSU issue slots on staging.  Every pixel
// thread then reads records as shared-memory broadcasts.  Early termination: a
// CTA-wide vote (__syncthreads_count) per batch, which doubles as the "stage free"
// signal for the producer thread.
#include "common.cuh"
#include "tma.cuh"

namespace h3dgs {

constexpr int kFwdBatch = 256;
constexpr int kFwdMinBlocks = 1;
constexpr int kFwdStages = 2;

// Two vertically adjacent pixels per thread: CTA = 128 threads = 4 warps, warp q owns one 8x8-pixel
// quadrant of the tile (quad_pixel).
// The entry's record, its dx terms, the survivor loop and (in backward) the 8-lane reduction are
// shared by the two pixels; only the per-pixel arithmetic of the pair (pair_math.cuh) is done twice.
constexpr int kFwdThreads = 128;

// warp q's quadrant is (q & 1, q >> 1); lane l owns its column (l & 7) and the two rows 2*(l >> 3), +1
__device__ __forceinline__ void quad_pixel(int tile_x, int tile_y, int warp, int lane, int& px, int& py0) {
    px = tile_x * kTile + 8 * (warp & 1) + (lane & 7);
    py0 = tile_y * kTile + 8 * (warp >> 1) + 2 * (lane >> 3);
}

template <bool HIER, bool DEPTH>
__global__ void __launch_bounds__(kFwdThreads, kFwdMinBlocks)
render_forward_kernel(int W, int H, int gx, int shard_count, int shard_index, const uint2* __restrict__ ranges,
                      const Record* __restrict__ sorted, const float* __restrict__ bg, float* __restrict__ out_color,
                      float* __restrict__ out_invdepth, float* __restrict__ final_T, uint32_t* __restrict__ n_contrib,
                      uint32_t* __restrict__ tile_max_contrib, const PeerPtrs peers)
{
    __shared__ __align__(128) Record s_rec[kFwdStages][kFwdBatch];
    __shared__ __align__(8) uint64_t s_full[kFwdStages];
    __shared__ uint32_t s_max;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tile_x = blockIdx.x % gx;
    const int tile_y = (blockIdx.x / gx) * shard_count + shard_index;
    const int tile = tile_y * gx + tile_x;
    const uint2 range = ranges[tile];
    const int n = (int)(range.y - range.x);
    const int nb = (n + kFwdBatch - 1) / kFwdBatch;
    const Record* src = sorted + range.x;

    if (tid == 0) {
        for (int s = 0; s < kFwdStages; s++) mbar_init(&s_full[s], 1);
        s_max = 0;
        fence_mbar_init();
    }
    __syncthreads();
    int issued = 0;
    if (tid == 0) {
        for (int s = 0; s < kFwdStages && s < nb; s++) {
            const uint32_t bytes = (uint32_t)min(kFwdBatch, n - s * kFwdBatch) * (uint32_t)sizeof(Record);
            mbar_arrive_expect_tx(&s_full[s], bytes);
            tma_load_1d(&s_rec[s][0], src + (size_t)s * kFwdBatch, bytes, &s_full[s]);
        }
    }
    issued = min(kFwdStages, nb);

    int px, py0;
    quad_pixel(tile_x, tile_y, warp, lane, px, py0);
    const int py1 = py0 + 1;
    const bool in0 = px < W && py0 < H, in1 = px < W && py1 < H;
    const float fpx = (float)px;
    const f2 nfpy = pk(-(float)py0, -(float)py1);
    bool done0 = !in0, done1 = !in1;
    // packed per-pixel state {pixel 0, pixel 1} (common.cuh "packed FP32 pairs")
    f2 T = bc(1.0f);
    float Ca0 = 0.f, Ca1 = 0.f, Ca2 = 0.f, Cb0 = 0.f, Cb1 = 0.f, Cb2 = 0.f, inv0 = 0.f, inv1 = 0.f;
    uint32_t last0 = 0, last1 = 0;
    const int qsel = kBlockShift + 4 * warp;                // this warp's four block bits in the entries' reach mask

    int waited = 0;
    for (int b = 0; b < nb; b++) {
        const int st = b % kFwdStages;
        mbar_wait(&s_full[st], (uint32_t)((b / kFwdStages) & 1));
        waited = b + 1;
        const int cnt = min(kFwdBatch, n - b * kFwdBatch);
        const Record* rec = &s_rec[st][0];
        const uint32_t base = (uint32_t)(b * kFwdBatch);
        // one entry at the thread's two pixels (straight-line: a per-thread `continue`/`break` here leaves the warp split
        // into fragments that each re-walk the list -- measured: 18x the instructions)
        auto blend_entry = [&](int j) {
            const float4 a = rec[j].a;
            const float4 bb = rec[j].b;
            const float4 c = rec[j].c;
            const uint32_t kb = __float_as_uint(bb.w);
            f2 d, G, al, unused;
            const f2 pw = pair_power(a, bb, a.x - fpx, nfpy, d);
            pair_gauss(pw, bb.y, G, al);
            pair_hier_alpha<HIER, false>(al, bb.z, kb & kSortedKidsMask, al, unused);
            bool v0, v1;
            const f2 w = pair_blend(pw, al, T, done0, done1, v0, v1);
            upk(fma2(bc(c.x), w, pk(Ca0, Cb0)), Ca0, Cb0);
            upk(fma2(bc(c.y), w, pk(Ca1, Cb1)), Ca1, Cb1);
            upk(fma2(bc(c.z), w, pk(Ca2, Cb2)), Ca2, Cb2);
            if (DEPTH) upk(fma2(bc(c.w), w, pk(inv0, inv1)), inv0, inv1);
            if (lane == 0) H3_STAT(8, 1);
            H3_STAT(9, (v0 ? 1 : 0) + (v1 ? 1 : 0));
            const uint32_t idx = base + (uint32_t)j + 1u;
            last0 = v0 ? idx : last0; last1 = v1 ? idx : last1;
        };
        // One list per warp: per round of 32 entries each lane tests ONE entry against this warp's quadrant and a ballot
        // compacts the survivors, so culled entries cost nothing per pixel.  The survivor loop is warp-uniform (same
        // mask in every lane).  A warp leaves the batch only when all of its 64 pixels are done.
        for (int j0 = 0; j0 < cnt; j0 += 32) {
            if (__all_sync(0xffffffffu, done0 && done1)) break;
            const int jl = j0 + lane;
            const uint32_t nib = jl < cnt ? (__float_as_uint(rec[jl].b.w) >> qsel) & 0xFu : 0u;
            uint32_t m = __ballot_sync(0xffffffffu, nib != 0u);
            while (m != 0u) {
                const int j = j0 + __ffs(m) - 1;
                m &= m - 1;
                blend_entry(j);
            }
        }
        const int ndone = __syncthreads_count(done0 && done1);
        if (ndone == kFwdThreads) break;
        if (b + kFwdStages < nb) {
            if (tid == 0) {
                const int nb2 = b + kFwdStages;
                const uint32_t bytes = (uint32_t)min(kFwdBatch, n - nb2 * kFwdBatch) * (uint32_t)sizeof(Record);
                mbar_arrive_expect_tx(&s_full[st], bytes);
                tma_load_1d(&s_rec[st][0], src + (size_t)nb2 * kFwdBatch, bytes, &s_full[st]);
            }
            issued = b + kFwdStages + 1;
        }
    }
    // a CTA must not retire while a bulk copy into its shared memory is in flight
    if (tid == 0)
        for (int b = waited; b < issued; b++) mbar_wait(&s_full[b % kFwdStages], (uint32_t)((b / kFwdStages) & 1));

    const float bg0 = bg[0], bg1 = bg[1], bg2 = bg[2];
    auto store = [&](bool inside, int py, float T, float c0, float c1, float c2, float invd, uint32_t last) {
        if (!inside) return;
        const size_t pix = (size_t)py * W + px;
        final_T[pix] = T;
        n_contrib[pix] = last;
        if (peers.n > 1) {
            // peer mode: the finished pixel goes into the [3,H,W] image of every rank whose pointer is given (plain stores; remote ones
            // travel over NVLink while other tiles are still blending) -- the all-gather of rendered tiles, fused
            const size_t plane = (size_t)H * W;
            const float v0 = c0 + T * bg0, v1 = c1 + T * bg1, v2 = c2 + T * bg2;
#pragma unroll
            for (int r = 0; r < H3DGS_MAX_PEERS; r++)        // compile-time indices: the pointers stay in the parameter bank
                if (r < peers.n && peers.p[r]) {
                    float* o = static_cast<float*>(peers.p[r]);
                    o[pix] = v0; o[plane + pix] = v1; o[2 * plane + pix] = v2;
                }
            if (DEPTH) out_invdepth[(((size_t)(blockIdx.x / gx)) * kTile + (size_t)(py & (kTile - 1))) * W + px] = invd;
        } else if (shard_count > 1) {
            // packed shard layout [local tile row][channel][16][W]: one contiguous slab per
            // rank, so the image exchange is a single all-gather (h3dgs/dist.py)
            const size_t local_row = blockIdx.x / gx;
            const size_t o = ((local_row * 3) * kTile + (size_t)(py & (kTile - 1))) * W + px;
            const size_t cs = (size_t)kTile * W;
            out_color[o] = c0 + T * bg0; out_color[o + cs] = c1 + T * bg1; out_color[o + 2 * cs] = c2 + T * bg2;
            if (DEPTH) out_invdepth[(local_row * kTile + (size_t)(py & (kTile - 1))) * W + px] = invd;
        } else {
            const size_t plane = (size_t)H * W;
            out_color[pix] = c0 + T * bg0; out_color[plane + pix] = c1 + T * bg1; out_color[2 * plane + pix] = c2 + T * bg2;
            if (DEPTH) out_invdepth[pix] = invd;
        }
    };
    store(in0, py0, lo(T), Ca0, Ca1, Ca2, inv0, last0);
    store(in1, py1, hi(T), Cb0, Cb1, Cb2, inv1, last1);
    const uint32_t wmax = __reduce_max_sync(0xffffffffu, max(last0, last1));
    if (lane == 0) atomicMax(&s_max, wmax);
    __syncthreads();
    if (tid == 0) tile_max_contrib[tile] = s_max;
}

int launch_render_forward(const h3dgs_raster_args& a, const uint32_t* ranges, const Record* sorted_records,
                          float* out_color, float* out_invdepth, float* final_T, uint32_t* n_contrib,
                          uint32_t* tile_max_contrib, cudaStream_t s)
{
    const int W = a.image_width, H = a.image_height;
    const int gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
    const int sc = a.shard_count > 0 ? a.shard_count : 1, si = a.shard_count > 0 ? a.shard_index : 0;
    const int rows = (gy + sc - 1 - si) / sc;
    if (rows <= 0 || gx <= 0) return H3DGS_OK;
    const bool hier = a.interpolation_weights != nullptr;
    const bool depth = a.do_depth != 0;
    const dim3 grid(gx * rows), block(kFwdThreads);
    ProfScope prof(H3DGS_STAGE_RENDER_FWD, s);
    const PeerPtrs peers = peer_ptrs(a.peer_image, a.peer_count);
#define LAUNCH(HI, DE)                                                                                         \
    render_forward_kernel<HI, DE><<<grid, block, 0, s>>>(W, H, gx, sc, si, (const uint2*)ranges, sorted_records, \
                                                         a.bg, out_color, out_invdepth, final_T, n_contrib,      \
                                                         tile_max_contrib, peers)
    if (hier) { if (depth) LAUNCH(true, true); else LAUNCH(true, false); }
    else      { if (depth) LAUNCH(false, true); else LAUNCH(false, false); }
#undef LAUNCH
    H3_LAUNCHED("render_forward", a.debug, s);
    return H3DGS_OK;
}

}  // namespace h3dgs
