// render_backward.cu -- K7: per-tile gradient replay (replaces BACKWARD::render).
// Semantics per oracle/oracle.c::oracle_render_backward.
//
// One CTA (128 threads, two pixels each) per tile, records streamed back-to-front with the same TMA
// double buffer as the forward; the arithmetic of a thread's two pixels is pair_math.cuh's; per-entry partials are reduced
// over the group's 8 lanes (group walk) or the warp (one list per warp) with a transpose-reduce (span_reduce), and the
// lanes holding the 9 (10 with depth) totals issue one or two predicated red.global.add per entry --
// 16x to 64x fewer atomics than the classic one-atomic-per-pixel formulation.
#include "common.cuh"
#include "tma.cuh"

namespace h3dgs {

// H3_BLEND_OCC8 (build switch, A/B on hardware): 224-entry batches (26.8 KB of shared memory per CTA) and a 64-register
// cap, so that 8 instead of 7 CTAs share an SM
#ifdef H3_BLEND_OCC8
constexpr int kBwdBatch = 224;
constexpr int kBwdMinBlocks = 8;
#else
constexpr int kBwdBatch = 256;
constexpr int kBwdMinBlocks = 1;
#endif
constexpr int kBwdStages = 2;

// Reduce the per-lane partials v[0..8] (v[0..9] with DEPTH) over every aligned span of SPAN lanes (8: a group of the
// group walk, 32: the warp) with a transpose-reduce.  Eight of them, u = v[0..3], v[5..8], go down the span's three top
// lane bits: at every level each lane keeps half of its values and ships the other half (4 + 2 + 1 shuffles), so the
// lanes whose top bits read q = 4 b_top + 2 b_mid + b_low end up with the total of u[q] (span_slot); a 32-lane span adds
// the lower two bits by plain butterflies.  v[4] rides along as a plain butterfly in x; with DEPTH it is paired with v[9]
// at the top level, so x holds the total of v[9] on the lanes whose top bit is set.  Per span: 10 shuffles (8 lanes) or
// 14 (32 lanes) and 14 selects (16 with DEPTH) for 9 or 10 values, instead of 10 x 3 or 10 x 5 shuffles.
__device__ __forceinline__ float xchg_add(float keep, float send, int mask) {
    return keep + __shfl_xor_sync(0xffffffffu, send, mask);
}
template <int SPAN, bool DEPTH>
__device__ __forceinline__ float span_reduce(const float (&v)[10], int lane, float& x) {
    constexpr int top = SPAN / 2, mid = SPAN / 4, low = SPAN / 8;
    const bool bt = lane & top, bm = lane & mid, bl = lane & low;
    float a[4], b[2];
#pragma unroll
    for (int i = 0; i < 4; i++) a[i] = xchg_add(bt ? v[5 + i] : v[i], bt ? v[i] : v[5 + i], top);
    x = DEPTH ? xchg_add(bt ? v[9] : v[4], bt ? v[4] : v[9], top) : xchg_add(v[4], v[4], top);
#pragma unroll
    for (int i = 0; i < 2; i++) b[i] = xchg_add(bm ? a[2 + i] : a[i], bm ? a[i] : a[2 + i], mid);
    x = xchg_add(x, x, mid);
    float r = xchg_add(bl ? b[1] : b[0], bl ? b[0] : b[1], low);
    x = xchg_add(x, x, low);
#pragma unroll
    for (int m = low / 2; m >= 1; m /= 2) { r = xchg_add(r, r, m); x = xchg_add(x, x, m); }
    return r;
}
// accum column of span_reduce's r on lane k of its span: u[q] with q = k / (SPAN / 8)
template <int SPAN>
__device__ __forceinline__ int span_slot(int k) { const int q = k / (SPAN / 8); return q < 4 ? q : q + 1; }

constexpr int kBwdThreads = 128;      // two vertically adjacent pixels per thread (see render_forward.cu)

// Tile-sharded frames (NCCL or peer mode): the sums of a rank's own tiles go into ITS accumulator; the exchange follows
// (peer mode: preprocess_backward.cu::peer_push_kernel stores the finished partial rows into the owners' staging areas).
// A first version added every (tile, Gaussian) row straight into the owner's memory with system-scope red.add: 4-byte
// reductions over NVLink made the replay several times slower.
template <bool HIER, bool DEPTH, bool GROUPS>
__global__ void __launch_bounds__(kBwdThreads, kBwdMinBlocks)
render_backward_kernel(int W, int H, int gx, int shard_count, int shard_index, const uint2* __restrict__ ranges,
                       const Record* __restrict__ sorted, const uint32_t* __restrict__ point_list,
                       const float* __restrict__ bg, const float* __restrict__ final_T,
                       const uint32_t* __restrict__ n_contrib, const uint32_t* __restrict__ tile_max_contrib,
                       const float* __restrict__ dL_dcolor, const float* __restrict__ dL_dinvdepth,
                       float* __restrict__ accum)
{
    __shared__ __align__(128) Record s_rec[kBwdStages][kBwdBatch];
    __shared__ uint32_t s_id[kBwdStages][kBwdBatch];
    __shared__ __align__(8) uint64_t s_full[kBwdStages];
    __shared__ __align__(16) uint8_t s_list[GROUPS ? kBwdThreads / 32 : 1][4][GROUPS ? kBwdBatch : 4];   // group walk: per warp, four lists of entry positions

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tile_x = blockIdx.x % gx;
    const int tile_y = (blockIdx.x / gx) * shard_count + shard_index;
    const int tile = tile_y * gx + tile_x;
    const uint2 range = ranges[tile];
    const int n = min((int)(range.y - range.x), (int)tile_max_contrib[tile]);   // nothing beyond the last contributor
    const int nb = (n + kBwdBatch - 1) / kBwdBatch;
    if (nb == 0) return;
    const Record* src = sorted + range.x;
    const uint32_t* ids = point_list + range.x;

    // Gaussian ids of a batch are staged with plain loads (their global address is only
    // 4-B aligned, below the 16-B granularity of bulk copies).  iteration it = 0..nb-1
    // handles batch b = nb-1-it (back to front).
    auto stage_ids = [&](int it) {
        const int b = nb - 1 - it, st = it % kBwdStages;
        for (int k = tid; k < kBwdBatch; k += kBwdThreads) {
            const int e = b * kBwdBatch + k;
            if (e < n) s_id[st][k] = ids[e];
        }
    };
    for (int it = 0; it < kBwdStages && it < nb; it++) stage_ids(it);
    if (GROUPS)                           // the warp's four lists: 4 kBwdBatch bytes = kBwdBatch words
        for (int k = lane; k < kBwdBatch; k += 32) reinterpret_cast<uint32_t*>(&s_list[warp][0][0])[k] = 0u;
    if (tid == 0) {
        for (int s = 0; s < kBwdStages; s++) mbar_init(&s_full[s], 1);
        fence_mbar_init();
    }
    __syncthreads();
    auto issue = [&](int it) {
        const int b = nb - 1 - it, st = it % kBwdStages;
        const uint32_t bytes = (uint32_t)min(kBwdBatch, n - b * kBwdBatch) * (uint32_t)sizeof(Record);
        mbar_arrive_expect_tx(&s_full[st], bytes);
        tma_load_1d(&s_rec[st][0], src + (size_t)b * kBwdBatch, bytes, &s_full[st]);
    };
    if (tid == 0)
        for (int it = 0; it < kBwdStages && it < nb; it++) issue(it);

    int px, py0;
    if (GROUPS) group_pixel(tile_x, tile_y, warp, lane, px, py0);
    else quad_pixel(tile_x, tile_y, warp, lane, px, py0);
    // accum columns this lane adds (-1: none): group walk, r of span_reduce<8> and x on lane 0 (v[4]) and lane 4 (v[9]);
    // one list per warp, see the reduction below
    const int k8 = lane & 7;
    const int slot = GROUPS ? span_slot<8>(k8)
                            : (lane & 3) == 0 ? span_slot<32>(lane) : lane == 1 ? 4 : (DEPTH && lane == 17) ? 9 : -1;
    const int xslot = k8 == 0 ? 4 : (DEPTH && k8 == 4) ? 9 : -1;
    const int grp = lane >> 3;
    const int py1 = py0 + 1;
    const bool in0 = px < W && py0 < H, in1 = px < W && py1 < H;
    const float fpx = (float)px;
    const f2 nfpy = pk(-(float)py0, -(float)py1);
    const size_t pix0 = (size_t)py0 * W + px, pix1 = (size_t)py1 * W + px, plane = (size_t)H * W;
    const float Tf0 = in0 ? final_T[pix0] : 0.f, Tf1 = in1 ? final_T[pix1] : 0.f;
    const f2 Tf = pk(Tf0, Tf1);
    PairState ps = {Tf, bc(0.f)};
    const int last0 = in0 ? (int)n_contrib[pix0] : 0, last1 = in1 ? (int)n_contrib[pix1] : 0;
    float ga0 = 0.f, ga1 = 0.f, ga2 = 0.f, gad = 0.f, gb0 = 0.f, gb1 = 0.f, gb2 = 0.f, gbd = 0.f;
    if (in0) { ga0 = dL_dcolor[pix0]; ga1 = dL_dcolor[plane + pix0]; ga2 = dL_dcolor[2 * plane + pix0]; if (DEPTH) gad = dL_dinvdepth[pix0]; }
    if (in1) { gb0 = dL_dcolor[pix1]; gb1 = dL_dcolor[plane + pix1]; gb2 = dL_dcolor[2 * plane + pix1]; if (DEPTH) gbd = dL_dinvdepth[pix1]; }
    const f2 g0 = pk(ga0, gb0), g1 = pk(ga1, gb1), g2 = pk(ga2, gb2), gd = pk(gad, gbd);
    const f2 neg_bgd = pk(-(bg[0] * ga0 + bg[1] * ga1 + bg[2] * ga2), -(bg[0] * gb0 + bg[1] * gb1 + bg[2] * gb2));
    const int wlast = (int)__reduce_max_sync(0xffffffffu, (unsigned)max(last0, last1));   // nothing in this quadrant beyond it
    const int qsel = kBlockShift + 4 * warp;                // this warp's four block bits in the entries' reach mask
    // group walk: nothing of a group's 16 pixels lies beyond its own last contributor
    int gl0, gl1, gl2, gl3;
    {
        int gm = max(last0, last1);
        gm = max(gm, __shfl_xor_sync(0xffffffffu, gm, 4)); gm = max(gm, __shfl_xor_sync(0xffffffffu, gm, 2));
        gm = max(gm, __shfl_xor_sync(0xffffffffu, gm, 1));
        gl0 = __shfl_sync(0xffffffffu, gm, 0); gl1 = __shfl_sync(0xffffffffu, gm, 8);
        gl2 = __shfl_sync(0xffffffffu, gm, 16); gl3 = __shfl_sync(0xffffffffu, gm, 24);
    }

    for (int it = 0; it < nb; it++) {
        const int st = it % kBwdStages, b = nb - 1 - it;
        mbar_wait(&s_full[st], (uint32_t)((it / kBwdStages) & 1));
        const int cnt = min(kBwdBatch, n - b * kBwdBatch);
        const Record* rec = &s_rec[st][0];
        // one entry at the thread's two pixels; has = false: this lane's group has no entry in this iteration
        auto replay_entry = [&](int j, bool has) {
            const int e = b * kBwdBatch + j;              // 0-based list position; contributor number e+1
            const float4 a = rec[j].a;
            const float4 bb = rec[j].b;
            const uint32_t gid = s_id[st][j];             // loaded with the record: same uniform address arithmetic
            const uint32_t kb = __float_as_uint(bb.w);
            const float dx = a.x - fpx;
            // alpha of the two pixels with exactly the forward's arithmetic and decisions
            f2 d, G, al, dadb = bc(1.0f);                // dadb is only read with HIER
            const f2 pw = pair_power(a, bb, dx, nfpy, d);
            pair_gauss(pw, bb.y, G, al);
            float pw0, pw1, al0, al1;
            upk(pw, pw0, pw1); upk(al, al0, al1);
            // the hierarchy weight only lowers alpha (1 - (1-a)^(1/k) <= a), so an entry that no pixel of
            // the warp takes at its base alpha is skipped before that arithmetic
            bool v0 = has && e < last0 && pw0 <= 0.0f && al0 >= kAlphaSkip;
            bool v1 = has && e < last1 && pw1 <= 0.0f && al1 >= kAlphaSkip;
            if (lane == 0) H3_STAT(0, 1);
            if ((lane & 7) == 0 && has) H3_STAT(3, 1);
            if (!__any_sync(0xffffffffu, v0 || v1)) { if (lane == 0) H3_STAT(1, 1); return; }            // warp-uniform
            if (HIER) {
                pair_hier_alpha<HIER, true>(al, bb.z, kb & kSortedKidsMask, al, dadb);
                upk(al, al0, al1);
                v0 = v0 && al0 >= kAlphaSkip;
                v1 = v1 && al1 >= kAlphaSkip;
            }
            H3_STAT(2, (v0 ? 1 : 0) + (v1 ? 1 : 0));
#ifdef H3_SIMT_EMU
            { const uint32_t tk = __ballot_sync(0xffffffffu, v0 || v1);
              if (GROUPS && (lane & 7) == 0 && has && ((tk >> (8 * grp)) & 0xFFu) == 0u) H3_STAT(4, 1); }
#endif
            G = sel2(v0, v1, G, bc(0.f));
            al = sel2(v0, v1, al, bc(0.f));
            const float4 c = rec[j].c;
            f2 cg = fma2(bc(c.z), g2, fma2(bc(c.y), g1, mul2(bc(c.x), g0)));
            if (DEPTH) cg = fma2(bc(c.w), gd, cg);
            float v[10];
            pair_grad<HIER, DEPTH>(a, bb, dx, d, G, al, dadb, cg, Tf, neg_bgd, g0, g1, g2, gd, ps, v);
            float* row = accum + (size_t)gid * kAccum;
            float x;
            if (GROUPS) {
                // every group reduces its own entry over its 8 lanes; groups without a taker stay silent
                const bool taker = ((__ballot_sync(0xffffffffu, v0 || v1) >> (8 * grp)) & 0xFFu) != 0u;
                const float r = span_reduce<8, DEPTH>(v, lane, x);
                if (taker) atomicAdd(row + slot, r);
                if (taker && xslot >= 0) atomicAdd(row + xslot, x);
            } else {
                // lanes 4 q hold the totals of u[q], lane 1 the total of v[4], lane 17 (DEPTH) the one of v[9]: one atomic
                const float r = span_reduce<32, DEPTH>(v, lane, x);
                if (slot >= 0) atomicAdd(row + slot, (lane & 3) == 0 ? r : x);
            }
        };
        if (GROUPS) {
            // Group walk (see render_forward.cu): per batch the warp compacts four lists of entry positions -- an entry is
            // listed for a group when its block bit is set and it lies before the group's last contributor -- and the
            // groups replay their lists back to front in lockstep.
            uint8_t* lst = &s_list[warp][0][0];
            const uint32_t lt = (1u << lane) - 1u;
            int c0 = 0, c1 = 0, c2 = 0, c3 = 0;
            for (int j0 = 0; j0 < cnt; j0 += 32) {
                const int jl = j0 + lane, e = b * kBwdBatch + jl;
                uint32_t nib = jl < cnt ? (__float_as_uint(rec[jl].b.w) >> qsel) & 0xFu : 0u;
                nib &= (e < gl0 ? 1u : 0u) | (e < gl1 ? 2u : 0u) | (e < gl2 ? 4u : 0u) | (e < gl3 ? 8u : 0u);
                const uint32_t m0 = __ballot_sync(0xffffffffu, nib & 1u), m1 = __ballot_sync(0xffffffffu, nib & 2u);
                const uint32_t m2 = __ballot_sync(0xffffffffu, nib & 4u), m3 = __ballot_sync(0xffffffffu, nib & 8u);
                if (nib & 1u) lst[c0 + __popc(m0 & lt)] = (uint8_t)jl;
                if (nib & 2u) lst[kBwdBatch + c1 + __popc(m1 & lt)] = (uint8_t)jl;
                if (nib & 4u) lst[2 * kBwdBatch + c2 + __popc(m2 & lt)] = (uint8_t)jl;
                if (nib & 8u) lst[3 * kBwdBatch + c3 + __popc(m3 & lt)] = (uint8_t)jl;
                c0 += __popc(m0); c1 += __popc(m1); c2 += __popc(m2); c3 += __popc(m3);
            }
            __syncwarp();
            const int mylen = grp == 0 ? c0 : grp == 1 ? c1 : grp == 2 ? c2 : c3;
            const int maxlen = max(max(c0, c1), max(c2, c3));
            const uint8_t* my = lst + grp * kBwdBatch;
            // positions past a group's own list are stale entries of an earlier list (zeroed at the start), so they name
            // records of the batch and the load needs no branch; has = false keeps them out of the sums and the state
            for (int i = maxlen - 1; i >= 0; i--) replay_entry((int)my[i], i < mylen);
            __syncwarp();                     // the lists are rebuilt for the next batch
        } else {
            // back to front; per round of 32 entries a ballot compacts the entries that can reach this warp's quadrant at all
            for (int j0 = (cnt - 1) & ~31; j0 >= 0; j0 -= 32) {
                const int jl = j0 + lane;
                const uint32_t nib = (jl < cnt && (b * kBwdBatch + jl) < wlast) ? (__float_as_uint(rec[jl].b.w) >> qsel) & 0xFu : 0u;
                uint32_t m = __ballot_sync(0xffffffffu, nib != 0u);
                while (m != 0u) {
                    const int top = 31 - __clz(m);
                    m &= ~(1u << top);
                    replay_entry(j0 + top, true);
                }
            }
        }
        __syncthreads();                      // every thread is done with stage st (records and ids)
        if (it + kBwdStages < nb) {
            if (tid == 0) issue(it + kBwdStages);
            stage_ids(it + kBwdStages);       // read two iterations later, after the next __syncthreads
        }
    }
}

int launch_render_backward(const h3dgs_raster_args& a, const uint32_t* ranges, const Record* sorted_records,
                           const uint32_t* point_list, const float* final_T, const uint32_t* n_contrib,
                           const uint32_t* tile_max_contrib, const float* dL_dcolor, const float* dL_dinvdepth,
                           float* accum, cudaStream_t s)
{
    const int W = a.image_width, H = a.image_height;
    const int gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
    const int sc = a.shard_count > 0 ? a.shard_count : 1, si = a.shard_count > 0 ? a.shard_index : 0;
    const int rows = (gy + sc - 1 - si) / sc;
    if (rows <= 0 || gx <= 0) return H3DGS_OK;
    const bool hier = a.interpolation_weights != nullptr;
    const bool depth = a.do_depth != 0 && dL_dinvdepth != nullptr;
    const dim3 grid(gx * rows), block(kBwdThreads);
    ProfScope prof(H3DGS_STAGE_RENDER_BWD, s);
    const bool groups = use_group_walk(true);
#define LAUNCH(HI, DE, GR)                                                                                          \
    render_backward_kernel<HI, DE, GR><<<grid, block, 0, s>>>(W, H, gx, sc, si, (const uint2*)ranges, sorted_records, \
                                                              point_list, a.bg, final_T, n_contrib, tile_max_contrib, \
                                                              dL_dcolor, dL_dinvdepth, accum)
#define LAUNCH2(HI, DE) do { if (groups) LAUNCH(HI, DE, true); else LAUNCH(HI, DE, false); } while (0)
    if (hier) { if (depth) LAUNCH2(true, true); else LAUNCH2(true, false); }
    else      { if (depth) LAUNCH2(false, true); else LAUNCH2(false, false); }
#undef LAUNCH2
#undef LAUNCH
    H3_LAUNCHED("render_backward", a.debug, s);
    return H3DGS_OK;
}

}  // namespace h3dgs
