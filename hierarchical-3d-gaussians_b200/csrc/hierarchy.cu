// hierarchy.cu -- the LOD cut: expand_to_size + get_interpolation_weights
// (replaces gaussian_hierarchy._C, call sites train_post.py:91-113,
// render_hierarchy.py:58-80).  Semantics per oracle/oracle.c::oracle_expand_to_size /
// oracle_interpolation_weights (UNPINNED: the gaussian-hierarchy source is absent).
//
// The cut is a flat map over all N nodes (a node is emitted when it is finer than the
// target while its parent is not, or when it is too coarse but holds leaf Gaussians),
// with an order-preserving compaction -- one kernel, one pass (lod_cut_fused_kernel).
// HBM-bound: 28 B node + 32 B box (+ the parent's box, an L2 hit in BFS order) per node.
#include <float.h>
#include "common.cuh"
#include "tma.cuh"

namespace h3dgs {

struct Node { int depth, parent, start, count_leafs, count_merged, start_children, count_children; };

__device__ __forceinline__ float node_size(const float4* __restrict__ boxes, int id, float vx, float vy, float vz) {
    const float4 mn = __ldg(boxes + 2 * (size_t)id), mx = __ldg(boxes + 2 * (size_t)id + 1);
    const bool inside = vx >= mn.x && vx <= mx.x && vy >= mn.y && vy <= mx.y && vz >= mn.z && vz <= mx.z;
    if (inside) return FLT_MAX;
    const float cx = fmaxf(mn.x, fminf(mx.x, vx)) - vx;
    const float cy = fmaxf(mn.y, fminf(mx.y, vy)) - vy;
    const float cz = fmaxf(mn.z, fminf(mx.z, vz)) - vz;
    const float dist = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(cx, cx), __fmul_rn(cy, cy)), __fmul_rn(cz, cz)));
    return mn.w / dist;
}

// transition weight of node `id` under `parent` (oracle_interpolation_weights)
__device__ __forceinline__ float transition_weight(const float4* __restrict__ boxes, int id, int parent, float target,
                                                   float vx, float vy, float vz)
{
    if (parent == -1) return 1.0f;
    const float psize = node_size(boxes, parent, vx, vy, vz);
    if (psize > 2.0f * target) return 1.0f;
    const float size = node_size(boxes, id, vx, vy, vz);
    const float start = fmaxf(0.5f * psize, size);
    const float diff = psize - start;
    if (diff <= 0) return 1.0f;
    const float tdiff = fmaxf(0.0f, target - start);
    return fmaxf(1.0f - (tdiff / diff), 0.0f);
}

__global__ void __launch_bounds__(256)
interpolation_weights_kernel(int n, const int* __restrict__ node_indices, float target, const int* __restrict__ nodes,
                             const float4* __restrict__ boxes, float vx, float vy, float vz, float* __restrict__ ts,
                             int* __restrict__ kids)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int id = node_indices[i];
    const int parent = nodes[7 * (size_t)id + 1];
    ts[i] = transition_weight(boxes, id, parent, target, vx, vy, vz);
    kids[i] = parent == -1 ? 1 : nodes[7 * (size_t)parent + 6];
}

// ------------------------------------------------------------------------------------------------------------
// Single-pass cut: mark + order-preserving compaction + emission (+ weights) in ONE kernel, every node and box read
// once.  CTAs take tiles of kCutTile consecutive nodes in launch order (dynamic tile id); the position of a tile's
// output is the sum of the counts of all earlier tiles, obtained with a decoupled look-back over a per-tile status
// word (aggregate available -> inclusive prefix available), so no second pass over the counts is needed.
//
// The kernel is a latency-bound stream (7-int node rows and the dependent fetch of the parent's box), so the tile's
// two contiguous slabs -- 28 KB of nodes, 32 KB of boxes -- are brought into shared memory by two bulk copies (TMA)
// issued by one thread: no registers or LSU issue slots are spent on the stream, three CTAs per SM keep 180 KB in
// flight (of the H100's 228 KB of shared memory per SM), and the threads read their rows from shared memory (stride 7 words: conflict-free).  A thread owns four
// CONSECUTIVE nodes (siblings share the parent's box), keeps their two sizes for the weight, fetches what the
// emission needs from the parent's node while the scan and the look-back run, and one block scan serves the tile.
// Algorithmic traffic: 28 B node + 32 B box per node (the parent's box and node are L2 hits in BFS order) in,
// 20 B per emitted row out.
// ------------------------------------------------------------------------------------------------------------
constexpr int kCutThreads = 256, kCutItems = 4, kCutTile = kCutThreads * kCutItems;
constexpr unsigned long long kTileAgg = 1ull << 62, kTilePrefix = 2ull << 62, kTileValue = (1ull << 62) - 1;
constexpr size_t kCutSmem = (size_t)kCutTile * 7 * sizeof(int) + (size_t)kCutTile * 2 * sizeof(float4);

__device__ __forceinline__ float box_size(const float4 mn, const float4 mx, float vx, float vy, float vz) {
    const bool inside = vx >= mn.x && vx <= mx.x && vy >= mn.y && vy <= mx.y && vz >= mn.z && vz <= mx.z;
    if (inside) return FLT_MAX;
    const float cx = fmaxf(mn.x, fminf(mx.x, vx)) - vx;
    const float cy = fmaxf(mn.y, fminf(mx.y, vy)) - vy;
    const float cz = fmaxf(mn.z, fminf(mx.z, vz)) - vz;
    const float dist = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(cx, cx), __fmul_rn(cy, cy)), __fmul_rn(cz, cz)));
    return mn.w / dist;
}

__global__ void __launch_bounds__(kCutThreads, 3)
lod_cut_fused_kernel(int N, const int* __restrict__ nodes, const float4* __restrict__ boxes, float target,
                     const float* __restrict__ target_dev, const float* __restrict__ viewpoint,
                     unsigned long long* __restrict__ tile_state /* [tiles] zeroed */, unsigned int* __restrict__ tile_counter /* zeroed */,
                     int* __restrict__ render_indices, int* __restrict__ parent_indices, int* __restrict__ nodes_of_render,
                     float* __restrict__ ts, int* __restrict__ kids, int* __restrict__ total)
{
    extern __shared__ float4 s_cut[];                         // boxes [kCutTile][2] | nodes [kCutTile][7]
    __shared__ uint64_t s_bar[2];
    __shared__ int s_warp[kCutThreads / 32];
    __shared__ int s_tile, s_base;
    float4* s_box = s_cut;
    int* s_node = reinterpret_cast<int*>(s_cut + 2 * kCutTile);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool aligned = ((((uintptr_t)nodes) | ((uintptr_t)boxes)) & 15) == 0;
    if (tid == 0) {
        const int t = (int)atomicAdd(tile_counter, 1u);
        s_tile = t;
        const int cnt = min(kCutTile, N - t * kCutTile);
        if (aligned && (cnt & 3) == 0) {                      // 28 * cnt bytes must be a multiple of 16
            mbar_init(&s_bar[0], 1); mbar_init(&s_bar[1], 1);
            fence_mbar_init();
            mbar_arrive_expect_tx(&s_bar[0], (uint32_t)cnt * 32u);
            tma_load_1d(s_box, boxes + 2 * (size_t)t * kCutTile, (uint32_t)cnt * 32u, &s_bar[0]);
            mbar_arrive_expect_tx(&s_bar[1], (uint32_t)cnt * 28u);
            tma_load_1d(s_node, nodes + 7 * (size_t)t * kCutTile, (uint32_t)cnt * 28u, &s_bar[1]);
        }
    }
    __syncthreads();
    const int tile = s_tile;
    const int tile_nodes = min(kCutTile, N - tile * kCutTile);
    if (target_dev) target = *target_dev;
    const float vx = viewpoint[0], vy = viewpoint[1], vz = viewpoint[2];
    if (aligned && (tile_nodes & 3) == 0) {
        mbar_wait(&s_bar[0], 0u);
        mbar_wait(&s_bar[1], 0u);
    } else {                                                  // ragged last tile / unaligned views: plain loads
        for (int k = tid; k < tile_nodes * 2; k += kCutThreads) s_box[k] = boxes[2 * (size_t)tile * kCutTile + k];
        for (int k = tid; k < tile_nodes * 7; k += kCutThreads) s_node[k] = nodes[7 * (size_t)tile * kCutTile + k];
        __syncthreads();
    }

    int cnt[kCutItems], pg[kCutItems], kk[kCutItems];
    float size[kCutItems], psize[kCutItems];
    int sum = 0;
#pragma unroll
    for (int k = 0; k < kCutItems; k++) {
        const int j = tid * kCutItems + k;
        int count = 0;
        size[k] = 0.f; psize[k] = 0.f; pg[k] = -1; kk[k] = 1;
        if (j < tile_nodes) {
            const int* nd = s_node + 7 * j;
            const int depth = nd[0], parent = nd[1], cl = nd[3], cm = nd[4];
            size[k] = box_size(s_box[2 * j], s_box[2 * j + 1], vx, vy, vz);
            const bool coarse = size[k] >= target;
            // the parent's box decides the nodes that are fine enough, and the weight of every emitted node
            if (parent != -1 && (!coarse || cl > 0)) {
                psize[k] = box_size(__ldg(boxes + 2 * (size_t)parent), __ldg(boxes + 2 * (size_t)parent + 1), vx, vy, vz);
                if (coarse) count = cl;
                else if (psize[k] >= target) { count = cl; if (depth != 0) count += cm; }
                if (count > 0) {
                    pg[k] = __ldg(nodes + 7 * (size_t)parent + 2);
                    if (kids) kk[k] = __ldg(nodes + 7 * (size_t)parent + 6);
                }
            } else if (coarse) count = cl;                    // the root
        }
        cnt[k] = count;
        sum += count;
    }
    // ---- one block-wide exclusive scan of the thread sums ----
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    int wbase = 0, carry = 0;
#pragma unroll
    for (int w = 0; w < kCutThreads / 32; w++) { const int v = s_warp[w]; if (w < warp) wbase += v; carry += v; }
    int off = wbase + incl - sum;                             // position of this thread's first row inside the tile
    // ---- decoupled look-back: exclusive prefix of this tile over all earlier tiles ----
    // (by warp 0, 32 status words per round trip; a look-back by the whole CTA trades the barrier stall for as much
    // long-scoreboard stall)
    if (warp == 0) {
        const unsigned long long agg = (unsigned long long)carry;
        if (lane == 0) {
            __threadfence();
            *((volatile unsigned long long*)(tile_state + tile)) = (tile == 0 ? kTilePrefix : kTileAgg) | agg;
        }
        long long prefix = 0;
        int idx = tile - 1;
        while (idx >= 0) {
            const int j = idx - lane;
            unsigned long long st = kTilePrefix;              // lanes past the beginning: "prefix 0"
            if (j >= 0) { do { st = *((volatile unsigned long long*)(tile_state + j)); } while ((st >> 62) == 0ull); }
            const unsigned full = __ballot_sync(0xffffffffu, (st >> 62) == 2ull);
            const int first = full ? __ffs(full) - 1 : 32;    // nearest predecessor whose inclusive prefix is known
            long long v = (lane <= first) ? (long long)(st & kTileValue) : 0ll;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            prefix += v;
            if (full) break;
            idx -= 32;
        }
        if (lane == 0) {
#ifdef H3_SIMT_EMU      /* the emulator runs the CTAs one after the other: a test switch keeps most tiles at "aggregate only" so that the */
            const bool upgrade = !(getenv("H3DGS_EMU_CUT_AGG_ONLY") && (tile % 300) != 0);     /* multi-window look-back is exercised */
#else
            const bool upgrade = true;
#endif
            if (tile != 0 && upgrade) {
                __threadfence();
                *((volatile unsigned long long*)(tile_state + tile)) = kTilePrefix | ((unsigned long long)prefix + agg);
            }
            s_base = (int)prefix;
            if (tile == (N + kCutTile - 1) / kCutTile - 1) *total = (int)(prefix + (long long)agg);
        }
    }
    __syncthreads();
    off += s_base;
    // ---- emission (about half of the nodes) ----
#pragma unroll
    for (int k = 0; k < kCutItems; k++) {
        if (cnt[k] == 0) continue;
        const int j = tid * kCutItems + k;
        const int n = tile * kCutTile + j;
        const int start = s_node[7 * j + 2];
        float tw = 1.0f;                                      // oracle_interpolation_weights
        if (ts && s_node[7 * j + 1] != -1 && !(psize[k] > 2.0f * target)) {
            const float st = fmaxf(0.5f * psize[k], size[k]);
            const float diff = psize[k] - st;
            if (diff > 0) tw = fmaxf(1.0f - (fmaxf(0.0f, target - st) / diff), 0.0f);
        }
        for (int q = 0; q < cnt[k]; q++) {
            render_indices[off + q] = start + q;
            parent_indices[off + q] = pg[k];
            nodes_of_render[off + q] = n;
            if (ts) ts[off + q] = tw;
            if (kids) kids[off + q] = kk[k];
        }
        off += cnt[k];
    }
}

}  // namespace h3dgs

using namespace h3dgs;

extern "C" size_t h3dgs_expand_scratch_bytes(int32_t N) {
    const size_t tiles = ((size_t)(N > 0 ? N : 1) + kCutTile - 1) / kCutTile;
    return align_up(tiles * 8 + 8) + 256;          // tile status words + tile counter | the count of h3dgs_expand_to_size
}

// every path reads `boxes` as float4 (the bulk copy, the plain-load fallback, interpolation_weights_kernel); only
// `nodes` may be a view at any 4-byte offset
static bool boxes_misaligned(const float* boxes, const char* who) {
    if ((((uintptr_t)boxes) & 15) == 0) return false;
    set_error("%s: boxes must be 16-byte aligned (got %p)", who, (const void*)boxes);
    return true;
}

// one launch of the single-pass cut; scratch holds the tile status words and the tile counter
static int launch_cut(int N, const int32_t* nodes, const float* boxes, float target_size, const float* target_size_dev,
                      const float* viewpoint, int32_t* render_indices, int32_t* parent_indices, int32_t* nodes_for_render_indices,
                      float* ts, int32_t* num_kids, int32_t* total, void* scratch, cudaStream_t s)
{
    const int tiles = (N + kCutTile - 1) / kCutTile;
    unsigned long long* state = (unsigned long long*)scratch;
    unsigned int* counter = (unsigned int*)(state + tiles);
    H3_CUDA(cudaMemsetAsync(scratch, 0, (size_t)tiles * 8 + 8, s));
    static bool smem_opt_in[64] = {};                          // per device, once (and never inside a stream capture: the
    int dev = 0;                                               // first cut of a GraphedStep is its eager probe pass)
    H3_CUDA(cudaGetDevice(&dev));
    if (!smem_opt_in[dev & 63]) {
        H3_CUDA(cudaFuncSetAttribute(lod_cut_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kCutSmem));
        smem_opt_in[dev & 63] = true;
    }
    lod_cut_fused_kernel<<<tiles, kCutThreads, kCutSmem, s>>>(N, nodes, (const float4*)boxes, target_size, target_size_dev, viewpoint, state,
                                                       counter, render_indices, parent_indices, nodes_for_render_indices, ts,
                                                       num_kids, total);
    H3_LAUNCHED("lod_cut_fused", 0, s);
    return H3DGS_OK;
}

extern "C" int h3dgs_expand_to_size(int32_t N, const int32_t* nodes, const float* boxes, float target_size,
                                    const float* viewpoint, float, float, float, int32_t* render_indices,
                                    int32_t* parent_indices, int32_t* nodes_for_render_indices, void* scratch,
                                    void* stream)
{
    if (N <= 0) return 0;
    if (boxes_misaligned(boxes, "expand_to_size")) return H3DGS_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    const int tiles = (N + kCutTile - 1) / kCutTile;
    int32_t* total = (int32_t*)((uint8_t*)scratch + align_up((size_t)tiles * 8 + 8));
    { ProfScope prof(H3DGS_STAGE_LOD_CUT, s);
    if (int rc = launch_cut(N, nodes, boxes, target_size, nullptr, viewpoint, render_indices, parent_indices,
                            nodes_for_render_indices, nullptr, nullptr, total, scratch, s)) return rc; }
    void* pin = nullptr;
    if (int rc = pinned_scratch(&pin)) return rc;
    H3_CUDA(cudaMemcpyAsync(pin, total, sizeof(int), cudaMemcpyDeviceToHost, s));
    H3_CUDA(cudaStreamSynchronize(s));
    return *static_cast<const int*>(pin);
}

extern "C" int h3dgs_lod_cut(int32_t N, const int32_t* nodes, const float* boxes, float target_size,
                             const float* target_size_dev, const float* viewpoint, int32_t* render_indices, int32_t* parent_indices,
                             int32_t* nodes_for_render_indices, float* ts, int32_t* num_kids, int32_t* count,
                             void* scratch, void* stream)
{
    if (N <= 0) { set_error("lod_cut: empty hierarchy"); return H3DGS_EINVAL; }
    if (!nodes || !boxes || !viewpoint || !render_indices || !parent_indices || !nodes_for_render_indices || !ts ||
        !num_kids || !count || !scratch) { set_error("lod_cut: NULL argument"); return H3DGS_EINVAL; }
    if (boxes_misaligned(boxes, "lod_cut")) return H3DGS_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope prof(H3DGS_STAGE_LOD_CUT, s);
    // rows after the cut: index -1 = "skip" for the rasterizer (the head is overwritten by the cut)
    H3_CUDA(cudaMemsetAsync(render_indices, 0xFF, (size_t)N * sizeof(int32_t), s));
    return launch_cut(N, nodes, boxes, target_size, target_size_dev, viewpoint, render_indices, parent_indices,
                      nodes_for_render_indices, ts, num_kids, count, scratch, s);
}

extern "C" int h3dgs_get_interpolation_weights(int32_t n, const int32_t* node_indices, float target_size,
                                               const int32_t* nodes, const float* boxes, float vx, float vy, float vz,
                                               float, float, float, float* ts, int32_t* num_kids, void* stream)
{
    if (n <= 0) return H3DGS_OK;
    if (boxes_misaligned(boxes, "get_interpolation_weights")) return H3DGS_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope prof(H3DGS_STAGE_LOD_WEIGHTS, s);
    interpolation_weights_kernel<<<(n + 255) / 256, 256, 0, s>>>(n, node_indices, target_size, nodes,
                                                                 (const float4*)boxes, vx, vy, vz, ts, num_kids);
    H3_LAUNCHED("interpolation_weights", 0, s);
    return H3DGS_OK;
}
