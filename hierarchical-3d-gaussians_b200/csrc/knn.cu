// knn.cu -- simple_knn._C.distCUDA2 (scene/gaussian_model.py:21, 190-194): for every point, the mean of the squared
// distances to its three nearest OTHER points, exactly.  GaussianModel.create_from_pcd turns it into the initial scale of
// every Gaussian of an SfM cloud (10^5 .. a few 10^6 points of very uneven density, plus, for the coarse stage, a skybox
// shell at 10x the scene radius).
//
// Pipeline (all on `stream`, no host synchronisation, all scratch from the caller):
//   1. bbox_kernel      bounding box over the finite coordinates (order-preserving uint atomicMax) and the finite count
//   2. morton_kernel    30-bit Morton key per point (an axis of zero extent maps to 0; non-finite points: 1 << 30, last)
//   3. 4 LSD passes     stable key/index radix sort, 8-bit digits: histogram -> one-block scan -> stable scatter
//   4. gather_kernel    points in sorted order as float4 {x, y, z, original index}
//   5. boxes_kernel     count-based AABBs: 32 sorted points per leaf box, 32 leaf boxes per upper box.  Count-based
//                       boxes stay tight around a dense scene however far a skybox stretches the global box.
//   6. search_kernel    one warp per 32 consecutive sorted points: seeded with the warp's own leaf, then its own upper
//                       box, then every other upper box -- each box pruned against the warp's largest current b2 (warp
//                       box vs box) and each leaf again per lane (point vs box) before its 32 points are scanned.
// The pruning bounds are computed with the same monotone fp32 operations as the distances, so a bound never exceeds a
// distance it stands for: the search is exact whatever order the boxes are visited in, and the result depends only on
// the set of points.  This file is compiled with -fmad=false: the arithmetic is pinned (h3dgs.h).
#include <float.h>
#include <math.h>
#include "common.cuh"
#include "float_key.cuh"

namespace h3dgs {
namespace {

constexpr int kLeaf = 32, kUpper = 32;             // points per leaf box, leaf boxes per upper box
constexpr int kSortThreads = 256, kSortSub = 16;   // sort tile: 16 sub-tiles of 256 keys per block
constexpr int kSortTile = kSortThreads * kSortSub;
constexpr int kRadixBits = 8, kRadix = 1 << kRadixBits, kSortPasses = 4;   // keys are 31 bits
constexpr int kScanThreads = 1024;
constexpr uint32_t kNonFiniteKey = 1u << 30;
constexpr unsigned kFull = 0xffffffffu;

// bbox[0..2] ~key(min), [3..5] key(max) (order-preserving uint encoding: both reduced with atomicMax, from 0),
// [6] finite count
struct KnnLayout { size_t bbox, keys_a, keys_b, vals_a, vals_b, counts, pts, leaves, uppers, total; };

inline int sort_blocks(int P) { return (P + kSortTile - 1) / kSortTile; }

KnnLayout knn_layout(int64_t P) {
    KnnLayout l; size_t o = 0;
    const size_t n = (size_t)P, nl = (n + kLeaf - 1) / kLeaf, nu = (nl + kUpper - 1) / kUpper;
    const size_t nb = (n + kSortTile - 1) / kSortTile;
    l.bbox = o;   o += align_up(8 * sizeof(uint32_t));
    l.keys_a = o; o += align_up(n * sizeof(uint32_t));
    l.keys_b = o; o += align_up(n * sizeof(uint32_t));
    l.vals_a = o; o += align_up(n * sizeof(uint32_t));
    l.vals_b = o; o += align_up(n * sizeof(uint32_t));
    l.counts = o; o += align_up((size_t)kRadix * nb * sizeof(uint32_t));
    l.pts = o;    o += align_up(n * sizeof(float4));
    l.leaves = o; o += align_up(nl * 2 * sizeof(float4));
    l.uppers = o; o += align_up(nu * 2 * sizeof(float4));
    l.total = o;
    return l;
}

__device__ __forceinline__ bool finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }


// the pinned distance: dx = q.x - p.x, d = (dx*dx + dy*dy) + dz*dz, every operation rounded
__device__ __forceinline__ float dist2(float4 q, float px, float py, float pz) {
    const float dx = q.x - px, dy = q.y - py, dz = q.z - pz;
    return (dx * dx + dy * dy) + dz * dz;
}
// lower bound of dist2 over the box [lo, hi] seen from [plo, phi] (a point: plo = phi).  Each gap is one rounded
// subtraction of a box face from a query coordinate beyond it, which rounding keeps <= |dx|; squares and sums are monotone.
__device__ __forceinline__ float box_gap2(float4 lo, float4 hi, float plx, float ply, float plz, float phx, float phy, float phz) {
    const float gx = fmaxf(fmaxf(lo.x - phx, plx - hi.x), 0.f);
    const float gy = fmaxf(fmaxf(lo.y - phy, ply - hi.y), 0.f);
    const float gz = fmaxf(fmaxf(lo.z - phz, plz - hi.z), 0.f);
    return (gx * gx + gy * gy) + gz * gz;
}

__global__ void __launch_bounds__(256) bbox_kernel(int P, const float* __restrict__ pts, uint32_t* __restrict__ bbox) {
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    uint32_t nfin = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
        const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
        if (finite3(x, y, z)) {
            lo[0] = fminf(lo[0], x); lo[1] = fminf(lo[1], y); lo[2] = fminf(lo[2], z);
            hi[0] = fmaxf(hi[0], x); hi[1] = fmaxf(hi[1], y); hi[2] = fmaxf(hi[2], z);
            nfin++;
        }
    }
    for (int a = 0; a < 3; a++) { lo[a] = warp_min(lo[a]); hi[a] = warp_max(hi[a]); }
    for (int o = 16; o; o >>= 1) nfin += __shfl_xor_sync(kFull, nfin, o);
    if ((threadIdx.x & 31) == 0 && nfin) {
        for (int a = 0; a < 3; a++) { atomicMax(bbox + a, ~f2key(lo[a])); atomicMax(bbox + 3 + a, f2key(hi[a])); }
        atomicAdd(bbox + 6, nfin);
    }
}

__device__ __forceinline__ uint32_t spread10(uint32_t v) {       // bit k -> bit 3k
    v = (v | (v << 16)) & 0x030000FFu;
    v = (v | (v << 8)) & 0x0300F00Fu;
    v = (v | (v << 4)) & 0x030C30C3u;
    v = (v | (v << 2)) & 0x09249249u;
    return v;
}
__device__ __forceinline__ uint32_t cell10(float x, float lo, float hi) {
    const float ext = hi - lo;
    if (!(ext > 0.f) || !isfinite(ext)) return 0u;
    const float t = fminf(fmaxf((x - lo) / ext * 1024.f, 0.f), 1023.f);
    return (uint32_t)t;
}

__global__ void __launch_bounds__(256) morton_kernel(int P, const float* __restrict__ pts, const uint32_t* __restrict__ bbox,
                                                     uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
    uint32_t k = kNonFiniteKey;
    if (finite3(x, y, z)) {
        k = (spread10(cell10(x, key2f(~bbox[0]), key2f(bbox[3]))) << 2) | (spread10(cell10(y, key2f(~bbox[1]), key2f(bbox[4]))) << 1) |
            spread10(cell10(z, key2f(~bbox[2]), key2f(bbox[5])));
    }
    keys[i] = k;
    vals[i] = (uint32_t)i;
}

// counts[d * nb + b] = number of keys of sort tile b whose digit is d
__global__ void __launch_bounds__(kSortThreads) radix_hist_kernel(int P, int shift, const uint32_t* __restrict__ keys,
                                                                  uint32_t* __restrict__ counts) {
    __shared__ uint32_t hist[kRadix];
    hist[threadIdx.x] = 0;
    __syncthreads();
    const int begin = blockIdx.x * kSortTile, end = min(begin + kSortTile, P);
    for (int e = begin + threadIdx.x; e < end; e += kSortThreads) atomicAdd(&hist[(keys[e] >> shift) & (kRadix - 1)], 1u);
    __syncthreads();
    counts[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = hist[threadIdx.x];
}

// exclusive scan of counts[0 .. n) in place, one block
__global__ void __launch_bounds__(kScanThreads) radix_scan_kernel(int n, uint32_t* __restrict__ counts) {
    __shared__ uint32_t part[kScanThreads / 32];
    const int chunk = (n + kScanThreads - 1) / kScanThreads;
    const int b = threadIdx.x * chunk, e = min(b + chunk, n);
    uint32_t s = 0;
    for (int k = b; k < e; k++) s += counts[k];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = s;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(kFull, inc, o); if (lane >= o) inc += v; }
    if (lane == 31) part[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = part[lane], wi = w;
        for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(kFull, wi, o); if (lane >= o) wi += v; }
        part[lane] = wi - w;
    }
    __syncthreads();
    uint32_t run = part[warp] + inc - s;
    for (int k = b; k < e; k++) { const uint32_t c = counts[k]; counts[k] = run; run += c; }
}

// stable scatter of sort tile b: sub-tiles in order, inside one by (warp, lane); equal digits of a warp found with 8 ballots
__global__ void __launch_bounds__(kSortThreads) radix_scatter_kernel(int P, int shift, const uint32_t* __restrict__ counts,
                                                                     const uint32_t* __restrict__ kin, const uint32_t* __restrict__ vin,
                                                                     uint32_t* __restrict__ kout, uint32_t* __restrict__ vout) {
    constexpr int kWarps = kSortThreads / 32;
    __shared__ uint32_t base[kRadix];
    __shared__ uint32_t wcount[kWarps][kRadix];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    base[t] = counts[(size_t)t * gridDim.x + blockIdx.x];
    for (int r = 0; r < kSortSub; r++) {
        for (int w = 0; w < kWarps; w++) wcount[w][t] = 0;
        __syncthreads();
        const int e = blockIdx.x * kSortTile + r * kSortThreads + t;
        const bool valid = e < P;
        uint32_t k = 0, v = 0;
        if (valid) { k = kin[e]; v = vin[e]; }
        const uint32_t d = (k >> shift) & (kRadix - 1);
        uint32_t peers = __ballot_sync(kFull, valid);
#pragma unroll
        for (int bit = 0; bit < kRadixBits; bit++) {
            const bool on = (d >> bit) & 1u;
            const uint32_t m = __ballot_sync(kFull, on);
            peers &= on ? m : ~m;
        }
        const uint32_t below = peers & ((1u << lane) - 1u);
        if (valid && below == 0u) wcount[warp][d] = __popc(peers);
        __syncthreads();
        if (valid) {
            uint32_t pos = base[d] + __popc(below);
            for (int w = 0; w < warp; w++) pos += wcount[w][d];
            kout[pos] = k; vout[pos] = v;
        }
        __syncthreads();
        uint32_t add = 0;
        for (int w = 0; w < kWarps; w++) add += wcount[w][t];
        base[t] += add;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) gather_kernel(int P, const float* __restrict__ pts, const uint32_t* __restrict__ vals,
                                                     float4* __restrict__ out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= P) return;
    const uint32_t i = vals[k];
    out[k] = make_float4(pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2], __uint_as_float(i));
}

// block u: upper box u; warp w of it: leaf box kUpper * u + w.  Only the finite prefix [0, Pf) of the sorted points.
__global__ void __launch_bounds__(kLeaf * kUpper) boxes_kernel(const float4* __restrict__ pts, const uint32_t* __restrict__ bbox,
                                                               float4* __restrict__ leaves, float4* __restrict__ uppers) {
    __shared__ float4 s_lo[kUpper], s_hi[kUpper];
    const int Pf = (int)bbox[6];
    if (blockIdx.x * (kLeaf * kUpper) >= Pf) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int k = blockIdx.x * (kLeaf * kUpper) + threadIdx.x;
    float lx = FLT_MAX, ly = FLT_MAX, lz = FLT_MAX, hx = -FLT_MAX, hy = -FLT_MAX, hz = -FLT_MAX;
    if (k < Pf) { const float4 p = pts[k]; lx = hx = p.x; ly = hy = p.y; lz = hz = p.z; }
    lx = warp_min(lx); ly = warp_min(ly); lz = warp_min(lz);
    hx = warp_max(hx); hy = warp_max(hy); hz = warp_max(hz);
    const int leaf = blockIdx.x * kUpper + warp;
    if (lane == 0) {
        s_lo[warp] = make_float4(lx, ly, lz, 0.f); s_hi[warp] = make_float4(hx, hy, hz, 0.f);
        if (leaf * kLeaf < Pf) { leaves[2 * leaf] = s_lo[warp]; leaves[2 * leaf + 1] = s_hi[warp]; }
    }
    __syncthreads();
    if (warp == 0) {
        const float4 lo = s_lo[lane], hi = s_hi[lane];
        lx = warp_min(lo.x); ly = warp_min(lo.y); lz = warp_min(lo.z);
        hx = warp_max(hi.x); hy = warp_max(hi.y); hz = warp_max(hi.z);
        if (lane == 0) {
            uppers[2 * blockIdx.x] = make_float4(lx, ly, lz, 0.f);
            uppers[2 * blockIdx.x + 1] = make_float4(hx, hy, hz, 0.f);
        }
    }
}

struct Best { float b0, b1, b2; };
__device__ __forceinline__ void insert(Best& b, float d) {
    if (d < b.b2) {
        if (d < b.b1) { b.b2 = b.b1; if (d < b.b0) { b.b1 = b.b0; b.b0 = d; } else { b.b1 = d; } }
        else { b.b2 = d; }
    }
}

struct Query {
    float px, py, pz;                        // this lane's point
    float lx, ly, lz, hx, hy, hz;            // the warp's box
    int i;                                   // sorted position (the self exclusion)
    bool active;
};

__device__ __forceinline__ float warp_bound(const Best& b, bool active) {
    return __uint_as_float(__reduce_max_sync(kFull, active ? __float_as_uint(b.b2) : 0u));    // b2 >= 0: uint order
}

__device__ __forceinline__ void scan_leaf(const float4* __restrict__ pts, int Pf, int leaf, const Query& q, Best& b) {
    const int begin = leaf * kLeaf, end = min(begin + kLeaf, Pf);
    for (int j = begin; j < end; j++) {
        const float d = dist2(__ldg(pts + j), q.px, q.py, q.pz);
        if (j != q.i) insert(b, d);
    }
}

// the leaves of upper box u, except `skip`: first against the warp's box and bound, then per lane
__device__ __forceinline__ void visit_upper(const float4* __restrict__ pts, const float4* __restrict__ leaves, int Pf, int nl,
                                            int u, int skip, const Query& q, Best& b, float& bound) {
    const int lane = threadIdx.x & 31;
    const int leaf = u * kUpper + lane;
    bool want = false;
    if (leaf < nl && leaf != skip) {
        const float4 lo = __ldg(leaves + 2 * leaf), hi = __ldg(leaves + 2 * leaf + 1);
        want = box_gap2(lo, hi, q.lx, q.ly, q.lz, q.hx, q.hy, q.hz) < bound;
    }
    uint32_t m = __ballot_sync(kFull, want);
    while (m) {
        const int L = u * kUpper + __ffs(m) - 1;
        m &= m - 1;
        const float4 lo = __ldg(leaves + 2 * L), hi = __ldg(leaves + 2 * L + 1);
        const bool need = q.active && box_gap2(lo, hi, q.px, q.py, q.pz, q.px, q.py, q.pz) < b.b2;
        if (__any_sync(kFull, need)) {
            scan_leaf(pts, Pf, L, q, b);
            bound = warp_bound(b, q.active);
        }
    }
}

__global__ void __launch_bounds__(128) search_kernel(int P, const float4* __restrict__ pts, const uint32_t* __restrict__ bbox,
                                                     const float4* __restrict__ leaves, const float4* __restrict__ uppers,
                                                     float* __restrict__ out) {
    const int Pf = (int)bbox[6];
    const int lane = threadIdx.x & 31;
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int i = w * kLeaf + lane;
    if (w * kLeaf >= Pf) {                                   // non-finite points only: unspecified, here NaN
        if (i < P) out[__float_as_uint(pts[i].w)] = __int_as_float(0x7fc00000);
        return;
    }
    const int nl = (Pf + kLeaf - 1) / kLeaf, nu = (nl + kUpper - 1) / kUpper;
    Query q;
    q.i = i;
    q.active = i < Pf;
    const float4 p = __ldg(pts + min(i, Pf - 1));
    q.px = p.x; q.py = p.y; q.pz = p.z;
    q.lx = warp_min(p.x); q.ly = warp_min(p.y); q.lz = warp_min(p.z);
    q.hx = warp_max(p.x); q.hy = warp_max(p.y); q.hz = warp_max(p.z);
    Best b{FLT_MAX, FLT_MAX, FLT_MAX};
    scan_leaf(pts, Pf, w, q, b);                             // the warp's own leaf: w
    float bound = warp_bound(b, q.active);
    const int own = w / kUpper;
    visit_upper(pts, leaves, Pf, nl, own, w, q, b, bound);
    for (int c = 0; c < nu; c += 32) {
        const int u = c + lane;
        bool want = false;
        if (u < nu && u != own) {
            const float4 lo = __ldg(uppers + 2 * u), hi = __ldg(uppers + 2 * u + 1);
            want = box_gap2(lo, hi, q.lx, q.ly, q.lz, q.hx, q.hy, q.hz) < bound;
        }
        uint32_t m = __ballot_sync(kFull, want);
        while (m) {
            const int U = c + __ffs(m) - 1;
            m &= m - 1;
            const float4 lo = __ldg(uppers + 2 * U), hi = __ldg(uppers + 2 * U + 1);
            if (box_gap2(lo, hi, q.lx, q.ly, q.lz, q.hx, q.hy, q.hz) < bound)      // the bound may have shrunk
                visit_upper(pts, leaves, Pf, nl, U, -1, q, b, bound);
        }
    }
    if (i < P) out[__float_as_uint(pts[i].w)] = q.active ? ((b.b0 + b.b1) + b.b2) / 3.0f : __int_as_float(0x7fc00000);
}

}  // namespace
}  // namespace h3dgs

using namespace h3dgs;

extern "C" size_t h3dgs_knn_scratch_bytes(int64_t P) { return P > 0 ? knn_layout(P).total : 0; }

extern "C" int h3dgs_dist_knn3(int32_t P, const float* points, float* mean_dist2, void* scratch, void* stream) {
    if (P < 0 || (P > 0 && (!points || !mean_dist2 || !scratch))) {
        set_error("dist_knn3: bad arguments"); return H3DGS_EINVAL;
    }
    if (P == 0) return H3DGS_OK;
    cudaStream_t s = (cudaStream_t)stream;
    const KnnLayout l = knn_layout(P);
    uint8_t* base = static_cast<uint8_t*>(scratch);
    uint32_t* bbox = reinterpret_cast<uint32_t*>(base + l.bbox);
    uint32_t* keys[2] = {reinterpret_cast<uint32_t*>(base + l.keys_a), reinterpret_cast<uint32_t*>(base + l.keys_b)};
    uint32_t* vals[2] = {reinterpret_cast<uint32_t*>(base + l.vals_a), reinterpret_cast<uint32_t*>(base + l.vals_b)};
    uint32_t* counts = reinterpret_cast<uint32_t*>(base + l.counts);
    float4* pts = reinterpret_cast<float4*>(base + l.pts);
    float4* leaves = reinterpret_cast<float4*>(base + l.leaves);
    float4* uppers = reinterpret_cast<float4*>(base + l.uppers);

    H3_CUDA(cudaMemsetAsync(bbox, 0, 8 * sizeof(uint32_t), s));        // the identity of every word's reduction
    const int blocks256 = (P + 255) / 256;
    bbox_kernel<<<min(blocks256, 1024), 256, 0, s>>>(P, points, bbox);
    H3_LAUNCHED("knn_bbox", 0, s);
    morton_kernel<<<blocks256, 256, 0, s>>>(P, points, bbox, keys[0], vals[0]);
    H3_LAUNCHED("knn_morton", 0, s);
    const int nb = sort_blocks(P);
    for (int pass = 0; pass < kSortPasses; pass++) {
        const int src = pass & 1, shift = pass * kRadixBits;
        radix_hist_kernel<<<nb, kSortThreads, 0, s>>>(P, shift, keys[src], counts);
        H3_LAUNCHED("knn_radix_hist", 0, s);
        radix_scan_kernel<<<1, kScanThreads, 0, s>>>(kRadix * nb, counts);
        H3_LAUNCHED("knn_radix_scan", 0, s);
        radix_scatter_kernel<<<nb, kSortThreads, 0, s>>>(P, shift, counts, keys[src], vals[src], keys[src ^ 1], vals[src ^ 1]);
        H3_LAUNCHED("knn_radix_scatter", 0, s);
    }
    static_assert(kSortPasses % 2 == 0, "the sorted keys end in buffer a");
    gather_kernel<<<blocks256, 256, 0, s>>>(P, points, vals[0], pts);
    H3_LAUNCHED("knn_gather", 0, s);
    boxes_kernel<<<(P + kLeaf * kUpper - 1) / (kLeaf * kUpper), kLeaf * kUpper, 0, s>>>(pts, bbox, leaves, uppers);
    H3_LAUNCHED("knn_boxes", 0, s);
    search_kernel<<<(P + 127) / 128, 128, 0, s>>>(P, pts, bbox, leaves, uppers, mean_dist2);
    H3_LAUNCHED("knn_search", 0, s);
    return H3DGS_OK;
}
