// hier_merge.cu -- the hierarchy merger (the GaussianHierarchyMerger stage of scripts/full_train.py:241-264): K chunk
// hierarchies -> one hierarchy, each chunk keeping the leaf Gaussians its cell owns, the pieces joined by an LBVH top
// tree built with the creator's code (hier_tree.cuh).  The contract (ownership, pieces, top tree, output layout) is
// include/h3dgs.h h3dgs_merge_hierarchies; it is this project's own rule, not a restatement of upstream's.
//
// Inputs are the chunks' arrays concatenated, with per-chunk node and row offsets; indices inside a node table stay
// chunk-local.  Pipeline (all on `stream`; an offline tool, so it synchronises between the phases):
//   1. node_check_kernel   the node table checks, row claims (a count per row), the parent links for the cycle check
//      row_kernel          rows claimed twice, the leaf Gaussians' input checks, ownership (fp32, no FMA)
//      jump_kernel         pointer jumping on the parent links; cycle_kernel: a node whose jump does not end at a
//                          root (parent -1) is on or below a cycle
//                          -> read back the error flags
//   2. purity_kernel       bottom-up: every leaf Gaussian marks its node's ancestors "holds a leaf", an unowned one
//                          also "impure"; each walk stops at a marked node and after the chunk's node count
//      pure_up_kernel + jump_kernel    the highest pure ancestor of every pure node (pointer jumping)
//      flag_kernel         item roots, one-Gaussian items, kept non-root nodes and the kept nodes' rows; three cub
//                          scans number them -> read back R, the kept count and the output row count; allocate the
//                          work block
//   3. item_kernel         the item list; every leaf Gaussian's item as a sort key, cub radix sort, segment starts
//      moment_kernel       one warp per item: W, mu, Sigma, SH over its leaf Gaussians, lanes strided over the
//                          segment and a butterfly in a fixed order (deterministic, no fp64 atomics)
//      the top tree        bbox_kernel, then build_tree (hier_tree.cuh) with the items as its leaves
//   4. slot_kernel, map_kernel    where every kept input node lands; count_kernel + cub scan: the row blocks
//                          -> allocate the outputs
//   5. node_out_kernel     nodes, boxes, the top tree's merged rows, the source of every copied row
//      row_copy_kernel     the copied rows
// Deterministic: the atomics are order-independent (claim counts, error flags, the bounding box's max reduction).
// Compiled with -fmad=false: the ownership arithmetic and the Morton quantisation are pinned fp32.
#include <vector>
#include "hier_tree.cuh"

namespace h3dgs {
namespace {

constexpr int kMaxInt = 0x7fffffff;

// hdr words (int32): [0] a bad node table entry [1] a bad leaf Gaussian [2] a row claimed twice [3] a parent cycle
//                    [4] R [5] kept non-root nodes [6] rows of the kept input nodes [7] subtree items
constexpr int kMergeHdr = 16;

struct MergeLayout {
    size_t hdr, node_off, row_off, cells, impure, hasleaf, up, claim, row_node, row_flag, item_flag, item_scan,
        kept_flag, kept_scan, node_rows, node_rows_scan, out_of_node, keys_a, keys_b, vals_a, vals_b, temp, total, temp_bytes;
};

MergeLayout merge_layout(int K, int64_t N, int64_t M) {
    MergeLayout l; size_t o = 0;
    size_t t1 = 0, t2 = 0, t3 = 0;
    cub::DeviceScan::InclusiveSum(nullptr, t1, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(N + M));
    cub::DeviceScan::InclusiveSum(nullptr, t2, (const int32_t*)nullptr, (int32_t*)nullptr, (int)N);
    cub::DeviceRadixSort::SortPairs(nullptr, t3, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int)M, 0, 32);
    l.temp_bytes = t1 > t2 ? t1 : t2;
    if (t3 > l.temp_bytes) l.temp_bytes = t3;
    l.hdr = o;         o += align_up(kMergeHdr * sizeof(int32_t));
    l.node_off = o;    o += align_up((K + 1) * sizeof(int32_t));
    l.row_off = o;     o += align_up((K + 1) * sizeof(int32_t));
    l.cells = o;       o += align_up(4 * K * sizeof(float));
    l.impure = o;      o += align_up(N);
    l.hasleaf = o;     o += align_up(N);
    l.up = o;          o += align_up(N * sizeof(int32_t));
    l.claim = o;       o += align_up(M * sizeof(int32_t));
    l.row_node = o;    o += align_up(M * sizeof(int32_t));
    l.row_flag = o;    o += align_up(M);
    l.item_flag = o;   o += align_up((N + M) * sizeof(int32_t));
    l.item_scan = o;   o += align_up((N + M) * sizeof(int32_t));
    l.kept_flag = o;   o += align_up(N * sizeof(int32_t));
    l.kept_scan = o;   o += align_up(N * sizeof(int32_t));
    l.node_rows = o;   o += align_up(N * sizeof(int32_t));
    l.node_rows_scan = o; o += align_up(N * sizeof(int32_t));
    l.out_of_node = o; o += align_up(N * sizeof(int32_t));
    l.keys_a = o;      o += align_up(M * sizeof(uint32_t));
    l.keys_b = o;      o += align_up(M * sizeof(uint32_t));
    l.vals_a = o;      o += align_up(M * sizeof(uint32_t));
    l.vals_b = o;      o += align_up(M * sizeof(uint32_t));
    l.temp = o;        o += align_up(l.temp_bytes);
    l.total = o;
    return l;
}

// the work block (allocated once R and the kept count are known)
struct WorkLayout {
    size_t item_ref, item_depth, item_pos, item_mom, item_sh, item_box, seg, slot, kept_list, counts, starts, tree,
        txyz, tshs, topac, tls, trot, tnodes, tboxes, tsrc, temp, total, temp_bytes;
    BuildLayout b;
};

WorkLayout work_layout(int R, int NO, int kept) {
    WorkLayout l; size_t o = 0;
    const size_t r = (size_t)R, T = 2 * r - 1;
    l.b = build_layout(R);
    size_t t = 0;
    cub::DeviceScan::InclusiveSum(nullptr, t, (const int64_t*)nullptr, (int64_t*)nullptr, NO);
    l.temp_bytes = t;
    l.item_ref = o;   o += align_up(r * sizeof(int32_t));
    l.item_depth = o; o += align_up(r * sizeof(int32_t));
    l.item_pos = o;   o += align_up(r * 3 * sizeof(float));
    l.item_mom = o;   o += align_up(r * kMoments * sizeof(double));
    l.item_sh = o;    o += align_up(r * kSH * sizeof(double));
    l.item_box = o;   o += align_up(r * 8 * sizeof(float));
    l.seg = o;        o += align_up((r + 1) * sizeof(int32_t));
    l.slot = o;       o += align_up(r * sizeof(int32_t));
    l.kept_list = o;  o += align_up((size_t)(kept > 0 ? kept : 1) * sizeof(int32_t));
    l.counts = o;     o += align_up((size_t)NO * sizeof(int64_t));
    l.starts = o;     o += align_up((size_t)NO * sizeof(int64_t));
    l.tree = o;       o += align_up(l.b.total);
    l.txyz = o;       o += align_up(T * 3 * sizeof(float));
    l.tshs = o;       o += align_up(T * kSH * sizeof(float));
    l.topac = o;      o += align_up(T * sizeof(float));
    l.tls = o;        o += align_up(T * 3 * sizeof(float));
    l.trot = o;       o += align_up(T * 4 * sizeof(float));
    l.tnodes = o;     o += align_up(T * 7 * sizeof(int32_t));
    l.tboxes = o;     o += align_up(T * 8 * sizeof(float));
    l.tsrc = o;       o += align_up(T * sizeof(int32_t));
    l.temp = o;       o += align_up(l.temp_bytes);
    l.total = o;
    return l;
}

struct Chunks {
    const int32_t* node_off;     // [K + 1]
    const int32_t* row_off;      // [K + 1]
    const float* cells;          // [K][cx, cy, ex, ey]
    int K;
};
// the chunk holding global index g of an offset table (the last c with off[c] <= g)
__device__ __forceinline__ int chunk_of(const int32_t* off, int K, int g) {
    int lo = 0, hi = K - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= g) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// a one-Gaussian item's reference: -2 - row, so that it collides neither with an input node (>= 0) nor with the -1 by
// which source_node marks a top interior node
__device__ __forceinline__ int single_ref(int row) { return -2 - row; }
__device__ __forceinline__ int single_row(int ref) { return -2 - ref; }

struct Src {
    const float *xyz, *shs, *opacities, *log_scales, *rotations, *boxes;
    const int32_t* nodes;
};

__global__ void __launch_bounds__(256) node_check_kernel(int N, Chunks ch, Src in, int32_t* __restrict__ hdr,
                                                         int32_t* __restrict__ claim, int32_t* __restrict__ row_node,
                                                         uint8_t* __restrict__ row_flag, int32_t* __restrict__ up) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N) return;
    const int c = chunk_of(ch.node_off, ch.K, g);
    const int n0 = ch.node_off[c], r0 = ch.row_off[c];
    const int Nc = ch.node_off[c + 1] - n0, Mc = ch.row_off[c + 1] - r0;
    const int i = g - n0;
    const int32_t* nd = in.nodes + 7 * (size_t)g;
    const int parent = nd[1], start = nd[2], cl = nd[3], cm = nd[4], sc = nd[5], cc = nd[6];
    bool ok = cl >= 0 && cm >= 0 && cc >= 0 && parent >= -1 && parent < Nc && parent != i;
    const int64_t rows = (int64_t)cl + cm;
    const bool rows_ok = ok && (rows == 0 || (start >= 0 && start + rows <= Mc));
    ok = rows_ok;
    if (ok && cc > 0) {
        ok = sc >= 0 && (int64_t)sc + cc <= Nc;
        for (int k = 0; ok && k < cc; k++) ok = in.nodes[7 * ((size_t)n0 + sc + k) + 1] == i;
    }
    if (ok && parent >= 0) {
        const int32_t* pd = in.nodes + 7 * ((size_t)n0 + parent);
        ok = pd[6] > 0 && pd[5] <= i && (int64_t)i < (int64_t)pd[5] + pd[6];
    }
    if (!ok) atomicMax(hdr + 0, 1);
    up[g] = ok && parent >= 0 ? n0 + parent : g;
    if (!rows_ok) return;
    for (int q = 0; q < (int)rows; q++) {
        const int r = r0 + start + q;
        atomicAdd(claim + r, 1);
        row_node[r] = g;
        row_flag[r] = q < cl ? 1 : 0;
    }
}

// k1 = squared distance of (x, y) to the cell, k2 = max(|dx| / ex, |dy| / ey): every operation rounded in fp32
__device__ __forceinline__ int owner_of(float x, float y, const float* __restrict__ cells, int K) {
    int best = 0;
    float b1 = 0.f, b2 = 0.f;
    for (int j = 0; j < K; j++) {
        const float cx = cells[4 * j], cy = cells[4 * j + 1], ex = cells[4 * j + 2], ey = cells[4 * j + 3];
        const float ax = fabsf(x - cx), ay = fabsf(y - cy);
        const float ox = fmaxf(ax - 0.5f * ex, 0.f), oy = fmaxf(ay - 0.5f * ey, 0.f);
        const float k1 = ox * ox + oy * oy;
        const float k2 = fmaxf(ax / ex, ay / ey);
        if (j == 0 || k1 < b1 || (k1 == b1 && k2 < b2)) { best = j; b1 = k1; b2 = k2; }
    }
    return best;
}

__global__ void __launch_bounds__(256) row_kernel(int M, Chunks ch, Src in, const int32_t* __restrict__ claim,
                                                  uint8_t* __restrict__ row_flag, int32_t* __restrict__ hdr) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= M) return;
    const int n = claim[r];
    if (n > 1) atomicMax(hdr + 2, 1);
    if (n != 1 || !(row_flag[r] & 1)) return;
    bool ok = true;
    for (int a = 0; a < 3; a++) {
        const float x = in.xyz[3 * (size_t)r + a], ls = in.log_scales[3 * (size_t)r + a];
        ok = ok && isfinite(x) && isfinite(ls) && ls <= kMaxLogScale;
    }
    for (int a = 0; a < 4; a++) ok = ok && isfinite(in.rotations[4 * (size_t)r + a]);
    const float o = in.opacities[r];
    if (!ok || !(o >= 0.f) || !isfinite(o)) { atomicMax(hdr + 1, 1); return; }
    const int c = chunk_of(ch.row_off, ch.K, r);
    if (owner_of(in.xyz[3 * (size_t)r], in.xyz[3 * (size_t)r + 1], ch.cells, ch.K) == c) row_flag[r] |= 2;
}

// one round of pointer jumping, in place (every value stays an ancestor, so the fixed point is the same)
__global__ void __launch_bounds__(256) jump_kernel(int N, int32_t* __restrict__ up) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N) return;
    up[g] = up[up[g]];
}

// after enough rounds every node's jump ends at its root; one that ends elsewhere (on a cycle, of any length) never
// reaches a root
__global__ void __launch_bounds__(256) cycle_kernel(int N, const int32_t* __restrict__ nodes, const int32_t* __restrict__ up,
                                                    int32_t* __restrict__ hdr) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N) return;
    if (nodes[7 * (size_t)up[g] + 1] != -1) atomicMax(hdr + 3, 1);
}

// marks n and its ancestors in flag, stopping at a marked node; at most `bound` steps
__device__ __forceinline__ void mark_up(volatile uint8_t* flag, const int32_t* __restrict__ nodes, int n0, int n, int bound) {
    for (int s = 0; s < bound && n >= 0; s++) {
        const int g = n0 + n;
        if (flag[g]) return;
        flag[g] = 1;
        n = nodes[7 * (size_t)g + 1];
    }
}

__global__ void __launch_bounds__(256) purity_kernel(int M, Chunks ch, const int32_t* __restrict__ nodes,
                                                     const int32_t* __restrict__ claim, const int32_t* __restrict__ row_node,
                                                     const uint8_t* __restrict__ row_flag, uint8_t* impure, uint8_t* hasleaf) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= M) return;
    if (claim[r] != 1 || !(row_flag[r] & 1)) return;
    const int g = row_node[r];
    const int c = chunk_of(ch.node_off, ch.K, g);
    const int n0 = ch.node_off[c], Nc = ch.node_off[c + 1] - n0;
    mark_up(hasleaf, nodes, n0, g - n0, Nc);
    if (!(row_flag[r] & 2)) mark_up(impure, nodes, n0, g - n0, Nc);
}

// up[g]: the pure parent of a pure node, else g
__global__ void __launch_bounds__(256) pure_up_kernel(int N, Chunks ch, const int32_t* __restrict__ nodes,
                                                      const uint8_t* __restrict__ impure, int32_t* __restrict__ up) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N) return;
    const int p = nodes[7 * (size_t)g + 1];
    const int pg = p >= 0 ? ch.node_off[chunk_of(ch.node_off, ch.K, g)] + p : -1;
    up[g] = !impure[g] && pg >= 0 && !impure[pg] ? pg : g;
}

// item slots: [0, N) the item roots, [N, N + M) the one-Gaussian items; kept_flag: the kept non-root nodes; node_rows:
// the rows every kept input node brings
__global__ void __launch_bounds__(256) flag_kernel(int N, int M, const int32_t* __restrict__ nodes, const int32_t* __restrict__ claim,
                                                   const int32_t* __restrict__ row_node, const uint8_t* __restrict__ row_flag,
                                                   const uint8_t* __restrict__ impure, const uint8_t* __restrict__ hasleaf,
                                                   const int32_t* __restrict__ up, int32_t* __restrict__ item_flag,
                                                   int32_t* __restrict__ kept_flag, int32_t* __restrict__ node_rows) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) {
        const bool pure = !impure[i];
        const bool root = pure && hasleaf[i] && up[i] == i, kept = pure && up[i] != i && hasleaf[up[i]];
        item_flag[i] = root;
        kept_flag[i] = kept;
        node_rows[i] = root || kept ? nodes[7 * (size_t)i + 3] + nodes[7 * (size_t)i + 4] : 0;
    } else if (i < N + M) {
        const int r = i - N;
        item_flag[i] = claim[r] == 1 && row_flag[r] == 3 && impure[row_node[r]];
    }
}

// the kept input nodes' rows are distinct claimed input rows, so their sum (< M) does not overflow
__global__ void __launch_bounds__(256) totals_kernel(int N, int M, const int32_t* __restrict__ item_scan,
                                                     const int32_t* __restrict__ kept_scan,
                                                     const int32_t* __restrict__ node_rows_scan, int32_t* __restrict__ hdr) {
    hdr[4] = item_scan[N + M - 1];
    hdr[5] = kept_scan[N - 1];
    hdr[6] = node_rows_scan[N - 1];
    hdr[7] = item_scan[N - 1];
}

// the item list (ref: the root node, or single_ref(row) for a one-Gaussian item; its depth) and every row's sort key (its item,
// R for a row in no item)
__global__ void __launch_bounds__(256) item_kernel(int N, int M, int R, Src in, const int32_t* __restrict__ claim,
                                                   const int32_t* __restrict__ row_node, const uint8_t* __restrict__ row_flag,
                                                   const uint8_t* __restrict__ impure, const int32_t* __restrict__ up,
                                                   const int32_t* __restrict__ item_flag, const int32_t* __restrict__ item_scan,
                                                   int32_t* __restrict__ item_ref, int32_t* __restrict__ item_depth,
                                                   uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N + M) return;
    if (item_flag[i]) {
        const int it = item_scan[i] - 1;
        item_ref[it] = i < N ? i : single_ref(i - N);
        item_depth[it] = i < N ? in.nodes[7 * (size_t)i] : 0;
    }
    if (i < N) return;
    const int r = i - N;
    uint32_t key = (uint32_t)R;
    if (claim[r] == 1 && row_flag[r] == 3) {
        const int g = row_node[r];
        key = (uint32_t)(impure[g] ? item_scan[i] - 1 : item_scan[up[g]] - 1);
    }
    keys[r] = key;
    vals[r] = (uint32_t)r;
}

__global__ void __launch_bounds__(256) seg_kernel(int M, int R, const uint32_t* __restrict__ keys, int32_t* __restrict__ seg) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= M) return;
    const uint32_t k = keys[p];
    if (k >= (uint32_t)R) return;
    if (p == 0 || keys[p - 1] != k) seg[k] = p;
    if (p == M - 1 || keys[p + 1] >= (uint32_t)R) seg[R] = p + 1;
}

__device__ __forceinline__ double warp_sum(double v) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

// one warp per item: its moments over the leaf Gaussians rows[seg[it] .. seg[it + 1]), in the creator's fp64 formulas
// (W = 0: the unweighted mean); its position (mu in fp32) and box (a whole subtree's input box, or the creator's leaf
// box of a one-Gaussian item)
__global__ void __launch_bounds__(128) moment_kernel(int R, Src in, const uint32_t* __restrict__ rows,
                                                     const int32_t* __restrict__ seg, const int32_t* __restrict__ item_ref,
                                                     double* __restrict__ item_mom, double* __restrict__ item_sh,
                                                     float* __restrict__ item_pos, float* __restrict__ item_box) {
    const int it = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (it >= R) return;
    const int b = seg[it], e = seg[it + 1];
    double W = 0.0, cnt = 0.0, wm[3] = {0.0, 0.0, 0.0}, um[3] = {0.0, 0.0, 0.0};
    for (int k = b + lane; k < e; k += 32) {
        const int r = (int)rows[k];
        double C[6];
        const double w = gauss_moments(in.log_scales + 3 * (size_t)r, in.rotations + 4 * (size_t)r, in.opacities[r], C);
        W += w; cnt += 1.0;
        for (int a = 0; a < 3; a++) { const double x = in.xyz[3 * (size_t)r + a]; wm[a] += w * x; um[a] += x; }
    }
    W = warp_sum(W); cnt = warp_sum(cnt);
    double mu[3];
    for (int a = 0; a < 3; a++) { wm[a] = warp_sum(wm[a]); um[a] = warp_sum(um[a]); mu[a] = W > 0.0 ? wm[a] / W : um[a] / cnt; }
    const double D = W > 0.0 ? W : cnt;
    double S[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    const int ia[6] = {0, 0, 0, 1, 1, 2}, ib[6] = {0, 1, 2, 1, 2, 2};
    for (int k = b + lane; k < e; k += 32) {
        const int r = (int)rows[k];
        double C[6];
        const double w = gauss_moments(in.log_scales + 3 * (size_t)r, in.rotations + 4 * (size_t)r, in.opacities[r], C);
        const double f = W > 0.0 ? w : 1.0;
        double d[3];
        for (int a = 0; a < 3; a++) d[a] = (double)in.xyz[3 * (size_t)r + a] - mu[a];
#pragma unroll
        for (int q = 0; q < 6; q++) S[q] += f * (C[q] + d[ia[q]] * d[ib[q]]);
    }
    double* m = item_mom + kMoments * (size_t)it;
    for (int q = 0; q < 6; q++) { S[q] = warp_sum(S[q]); if (lane == 0) m[4 + q] = S[q] / D; }
    if (lane == 0) {
        m[0] = W;
        for (int a = 0; a < 3; a++) { m[1 + a] = mu[a]; item_pos[3 * (size_t)it + a] = (float)mu[a]; }
    }
    for (int c0 = 0; c0 < kSH; c0 += 16) {
        double sh[16];
#pragma unroll
        for (int c = 0; c < 16; c++) sh[c] = 0.0;
        for (int k = b + lane; k < e; k += 32) {
            const int r = (int)rows[k];
            double f = 1.0;
            if (W > 0.0) { double C[6]; f = gauss_moments(in.log_scales + 3 * (size_t)r, in.rotations + 4 * (size_t)r, in.opacities[r], C); }
            const float* s = in.shs + kSH * (size_t)r + c0;
#pragma unroll
            for (int c = 0; c < 16; c++) sh[c] += f * (double)s[c];
        }
#pragma unroll
        for (int c = 0; c < 16; c++) { sh[c] = warp_sum(sh[c]); if (lane == 0) item_sh[kSH * (size_t)it + c0 + c] = sh[c] / D; }
    }
    if (lane != 0) return;
    const int ref = item_ref[it];
    float* box = item_box + 8 * (size_t)it;
    if (ref >= 0) {
        for (int q = 0; q < 8; q++) box[q] = in.boxes[8 * (size_t)ref + q];
    } else {
        const int r = single_row(ref);
        double C[6];
        gauss_moments(in.log_scales + 3 * (size_t)r, in.rotations + 4 * (size_t)r, in.opacities[r], C);
        gauss_box(in.xyz + 3 * (size_t)r, C, box);
    }
}

// the merger's leaves: item s with its moments, SH, box and depth
struct ItemLeaves {
    const double *mom, *sh;
    const float* box;
    const int32_t* depth;
    __device__ __forceinline__ void operator()(int p, int s, int32_t* nd, const Out& out, double* __restrict__ mom_out,
                                               double* __restrict__ shm) const {
        nd[0] = depth[s];
        out.source[p] = s;
        for (int q = 0; q < kMoments; q++) mom_out[kMoments * (size_t)p + q] = mom[kMoments * (size_t)s + q];
        for (int c = 0; c < kSH; c++) shm[kSH * (size_t)p + c] = sh[kSH * (size_t)s + c];
        for (int q = 0; q < 8; q++) out.boxes[8 * (size_t)p + q] = box[8 * (size_t)s + q];
    }
};

__global__ void __launch_bounds__(256) slot_kernel(int T, const int32_t* __restrict__ tnodes, const int32_t* __restrict__ tsrc,
                                                   int32_t* __restrict__ slot) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= T || tnodes[7 * (size_t)p + 6] != 0) return;
    slot[tsrc[p]] = p;
}

// where every kept input node lands: an item root at its top-tree slot, a kept non-root node after the top tree
__global__ void __launch_bounds__(256) map_kernel(int N, int T, const int32_t* __restrict__ item_flag,
                                                  const int32_t* __restrict__ item_scan, const int32_t* __restrict__ kept_flag,
                                                  const int32_t* __restrict__ kept_scan, const int32_t* __restrict__ slot,
                                                  int32_t* __restrict__ out_of_node, int32_t* __restrict__ kept_list) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N) return;
    if (item_flag[g]) out_of_node[g] = slot[item_scan[g] - 1];
    else if (kept_flag[g]) {
        const int k = kept_scan[g] - 1;
        out_of_node[g] = T + k;
        kept_list[k] = g;
    }
}

// the input node an output node copies (-1: a top interior node; single_ref(row) <= -2: a one-Gaussian item)
__device__ __forceinline__ int source_node(int o, int T, const int32_t* tnodes, const int32_t* tsrc, const int32_t* item_ref,
                                           const int32_t* kept_list) {
    if (o >= T) return kept_list[o - T];
    if (tnodes[7 * (size_t)o + 6] != 0) return -1;
    return item_ref[tsrc[o]];
}

__global__ void __launch_bounds__(256) count_kernel(int NO, int T, const int32_t* __restrict__ nodes,
                                                    const int32_t* __restrict__ tnodes, const int32_t* __restrict__ tsrc,
                                                    const int32_t* __restrict__ item_ref, const int32_t* __restrict__ kept_list,
                                                    int64_t* __restrict__ counts) {
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= NO) return;
    const int g = source_node(o, T, tnodes, tsrc, item_ref, kept_list);
    counts[o] = g < 0 ? 1 : (int64_t)nodes[7 * (size_t)g + 3] + nodes[7 * (size_t)g + 4];
}

struct Dst {
    float *xyz, *shs, *opacities, *log_scales, *rotations, *boxes;
    int32_t *nodes, *source_chunk, *source_row;
};

__global__ void __launch_bounds__(256) node_out_kernel(int NO, int T, int RO, Chunks ch, Src in, Out tree,
                                                       const int32_t* __restrict__ item_ref, const int32_t* __restrict__ kept_list,
                                                       const int32_t* __restrict__ out_of_node, const int64_t* __restrict__ ends,
                                                       const int64_t* __restrict__ counts, Dst out) {
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= NO) return;
    const int g = source_node(o, T, tree.nodes, tree.source, item_ref, kept_list);
    const int cnt = (int)counts[o];
    const int start = cnt > 0 ? (int)(ends[o] - cnt) : (int)(ends[o] < RO ? ends[o] : RO - 1);
    int32_t* nd = out.nodes + 7 * (size_t)o;
    float* box = out.boxes + 8 * (size_t)o;
    if (g == -1) {                                   // a top interior node and its merged row
        const int32_t* tn = tree.nodes + 7 * (size_t)o;
        nd[0] = tn[0]; nd[1] = tn[1]; nd[2] = start; nd[3] = 0; nd[4] = 1; nd[5] = tn[5]; nd[6] = 2;
        for (int q = 0; q < 8; q++) box[q] = tree.boxes[8 * (size_t)o + q];
        for (int a = 0; a < 3; a++) {
            out.xyz[3 * (size_t)start + a] = tree.xyz[3 * (size_t)o + a];
            out.log_scales[3 * (size_t)start + a] = tree.log_scales[3 * (size_t)o + a];
        }
        for (int a = 0; a < 4; a++) out.rotations[4 * (size_t)start + a] = tree.rotations[4 * (size_t)o + a];
        out.opacities[start] = tree.opacities[o];
        for (int c = 0; c < kSH; c++) out.shs[kSH * (size_t)start + c] = tree.shs[kSH * (size_t)o + c];
        out.source_chunk[start] = -1; out.source_row[start] = -1;
        return;
    }
    if (g < -1) {                                    // a one-Gaussian item (its box is the tree's leaf box)
        const int r = single_row(g);
        const int c = chunk_of(ch.row_off, ch.K, r);
        nd[0] = 0; nd[1] = tree.nodes[7 * (size_t)o + 1]; nd[2] = start; nd[3] = 1; nd[4] = 0; nd[5] = 0; nd[6] = 0;
        for (int q = 0; q < 8; q++) box[q] = tree.boxes[8 * (size_t)o + q];
        out.source_chunk[start] = c; out.source_row[start] = r - ch.row_off[c];
        return;
    }
    // a kept input node: an item root at its slot, or a kept non-root node
    const int c = chunk_of(ch.node_off, ch.K, g);
    const int n0 = ch.node_off[c];
    const int32_t* in_nd = in.nodes + 7 * (size_t)g;
    nd[0] = in_nd[0];
    nd[1] = o < T ? tree.nodes[7 * (size_t)o + 1] : out_of_node[n0 + in_nd[1]];
    nd[2] = start; nd[3] = in_nd[3]; nd[4] = in_nd[4];
    nd[5] = in_nd[6] > 0 ? out_of_node[n0 + in_nd[5]] : 0;
    nd[6] = in_nd[6];
    for (int q = 0; q < 8; q++) box[q] = in.boxes[8 * (size_t)g + q];
    for (int q = 0; q < cnt; q++) { out.source_chunk[start + q] = c; out.source_row[start + q] = in_nd[2] + q; }
}

__global__ void __launch_bounds__(256) row_copy_kernel(int RO, Chunks ch, Src in, Dst out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= RO) return;
    const int c = out.source_chunk[k];
    if (c < 0) return;
    const size_t r = (size_t)ch.row_off[c] + out.source_row[k];
    for (int a = 0; a < 3; a++) { out.xyz[3 * (size_t)k + a] = in.xyz[3 * r + a]; out.log_scales[3 * (size_t)k + a] = in.log_scales[3 * r + a]; }
    for (int a = 0; a < 4; a++) out.rotations[4 * (size_t)k + a] = in.rotations[4 * r + a];
    out.opacities[k] = in.opacities[r];
    for (int q = 0; q < kSH; q++) out.shs[kSH * (size_t)k + q] = in.shs[kSH * r + q];
}

int jump_rounds(int N) {
    int r = 1;
    while ((int64_t(1) << (r - 1)) < N) r++;
    return r;
}

bool offsets_ok(int K, const int64_t* off) {
    if (off[0] != 0) return false;
    for (int c = 0; c < K; c++)
        if (off[c + 1] < off[c]) return false;
    return true;
}

}  // namespace
}  // namespace h3dgs

using namespace h3dgs;

extern "C" size_t h3dgs_merge_hierarchies_scratch_bytes(int32_t K, int64_t total_nodes, int64_t total_rows) {
    if (K < 1 || total_nodes < 1 || total_rows < 1 || total_nodes + total_rows > kMaxInt) return 0;
    return merge_layout(K, total_nodes, total_rows).total;
}

extern "C" int h3dgs_merge_hierarchies(int32_t K, const int64_t* node_offsets, const int64_t* row_offsets, const float* cells,
                                       const float* xyz, const float* shs, const float* opacities, const float* log_scales,
                                       const float* rotations, const int32_t* nodes, const float* boxes,
                                       h3dgs_alloc_fn alloc, void* alloc_user, int64_t* counts, void* scratch, void* stream) {
    if (K < 1 || !node_offsets || !row_offsets || !cells || !xyz || !shs || !opacities || !log_scales || !rotations ||
        !nodes || !boxes || !alloc || !counts || !scratch) {
        set_error("merge_hierarchies: bad arguments (K = %d)", K); return H3DGS_EINVAL;
    }
    if (!offsets_ok(K, node_offsets) || !offsets_ok(K, row_offsets)) {
        set_error("merge_hierarchies: the node and row offsets must start at 0 and not decrease"); return H3DGS_EINVAL;
    }
    const int64_t N64 = node_offsets[K], M64 = row_offsets[K];
    if (N64 < 1 || M64 < 1 || N64 + M64 > kMaxInt) {
        set_error("merge_hierarchies: %lld nodes and %lld rows (both >= 1, together at most 2^31 - 1)", (long long)N64,
                  (long long)M64);
        return H3DGS_EINVAL;
    }
    for (int c = 0; c < K; c++) {
        const float* cl = cells + 4 * c;
        if (!isfinite(cl[0]) || !isfinite(cl[1]) || !isfinite(cl[2]) || !isfinite(cl[3]) || !(cl[2] > 0.f) || !(cl[3] > 0.f)) {
            set_error("merge_hierarchies: chunk %d: a cell needs a finite center and a finite, positive extent", c);
            return H3DGS_EINVAL;
        }
    }
    const int N = (int)N64, M = (int)M64;
    cudaStream_t s = (cudaStream_t)stream;
    const MergeLayout l = merge_layout(K, N, M);
    uint8_t* base = static_cast<uint8_t*>(scratch);
    int32_t* hdr = reinterpret_cast<int32_t*>(base + l.hdr);
    int32_t* node_off = reinterpret_cast<int32_t*>(base + l.node_off);
    int32_t* row_off = reinterpret_cast<int32_t*>(base + l.row_off);
    float* dcells = reinterpret_cast<float*>(base + l.cells);
    uint8_t* impure = base + l.impure;
    uint8_t* hasleaf = base + l.hasleaf;
    int32_t* up = reinterpret_cast<int32_t*>(base + l.up);
    int32_t* claim = reinterpret_cast<int32_t*>(base + l.claim);
    int32_t* row_node = reinterpret_cast<int32_t*>(base + l.row_node);
    uint8_t* row_flag = base + l.row_flag;
    int32_t* item_flag = reinterpret_cast<int32_t*>(base + l.item_flag);
    int32_t* item_scan = reinterpret_cast<int32_t*>(base + l.item_scan);
    int32_t* kept_flag = reinterpret_cast<int32_t*>(base + l.kept_flag);
    int32_t* kept_scan = reinterpret_cast<int32_t*>(base + l.kept_scan);
    int32_t* node_rows = reinterpret_cast<int32_t*>(base + l.node_rows);
    int32_t* node_rows_scan = reinterpret_cast<int32_t*>(base + l.node_rows_scan);
    int32_t* out_of_node = reinterpret_cast<int32_t*>(base + l.out_of_node);
    uint32_t* keys_a = reinterpret_cast<uint32_t*>(base + l.keys_a);
    uint32_t* keys_b = reinterpret_cast<uint32_t*>(base + l.keys_b);
    uint32_t* vals_a = reinterpret_cast<uint32_t*>(base + l.vals_a);
    uint32_t* vals_b = reinterpret_cast<uint32_t*>(base + l.vals_b);
    void* temp = base + l.temp;
    size_t temp_bytes;
    int32_t host[kMergeHdr];
    std::vector<int32_t> off32(2 * (size_t)(K + 1));
    for (int c = 0; c <= K; c++) { off32[c] = (int32_t)node_offsets[c]; off32[K + 1 + c] = (int32_t)row_offsets[c]; }

    // 1. node table, row claims, leaf checks, ownership, cycles
    H3_CUDA(cudaMemcpyAsync(node_off, off32.data(), (K + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    H3_CUDA(cudaMemcpyAsync(row_off, off32.data() + K + 1, (K + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    H3_CUDA(cudaMemcpyAsync(dcells, cells, 4 * K * sizeof(float), cudaMemcpyHostToDevice, s));
    H3_CUDA(cudaMemsetAsync(hdr, 0, kMergeHdr * sizeof(int32_t), s));
    H3_CUDA(cudaMemsetAsync(claim, 0, (size_t)M * sizeof(int32_t), s));
    H3_CUDA(cudaMemsetAsync(row_flag, 0, (size_t)M, s));
    H3_CUDA(cudaMemsetAsync(impure, 0, (size_t)N, s));
    H3_CUDA(cudaMemsetAsync(hasleaf, 0, (size_t)N, s));
    const Chunks ch{node_off, row_off, dcells, K};
    const Src in{xyz, shs, opacities, log_scales, rotations, boxes, nodes};
    node_check_kernel<<<blocks(N, 256), 256, 0, s>>>(N, ch, in, hdr, claim, row_node, row_flag, up);
    H3_LAUNCHED("merge_node_check", 0, s);
    row_kernel<<<blocks(M, 256), 256, 0, s>>>(M, ch, in, claim, row_flag, hdr);
    H3_LAUNCHED("merge_rows", 0, s);
    const int rounds = jump_rounds(N);
    for (int k = 0; k < rounds; k++) {
        jump_kernel<<<blocks(N, 256), 256, 0, s>>>(N, up);
        H3_LAUNCHED("merge_jump", 0, s);
    }
    cycle_kernel<<<blocks(N, 256), 256, 0, s>>>(N, nodes, up, hdr);
    H3_LAUNCHED("merge_cycle", 0, s);
    H3_CUDA(cudaMemcpyAsync(host, hdr, kMergeHdr * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    H3_CUDA(cudaStreamSynchronize(s));
    if (host[0] || host[2] || host[3]) {
        set_error("merge_hierarchies: an inconsistent node table (%s)", host[0] ? "an index out of range or a child whose parent "
                  "disagrees" : host[2] ? "a row claimed by two nodes" : "a parent chain longer than the node count");
        return H3DGS_EINVAL;
    }
    if (host[1]) {
        set_error("merge_hierarchies: a leaf Gaussian with a non-finite position, log-scale or rotation, a log-scale above "
                  "300, or a negative or non-finite opacity");
        return H3DGS_EINVAL;
    }

    // 2. purity, items, kept nodes
    purity_kernel<<<blocks(M, 256), 256, 0, s>>>(M, ch, nodes, claim, row_node, row_flag, impure, hasleaf);
    H3_LAUNCHED("merge_purity", 0, s);
    pure_up_kernel<<<blocks(N, 256), 256, 0, s>>>(N, ch, nodes, impure, up);
    H3_LAUNCHED("merge_pure_up", 0, s);
    for (int k = 0; k < rounds; k++) {
        jump_kernel<<<blocks(N, 256), 256, 0, s>>>(N, up);
        H3_LAUNCHED("merge_jump", 0, s);
    }
    flag_kernel<<<blocks(N + M, 256), 256, 0, s>>>(N, M, nodes, claim, row_node, row_flag, impure, hasleaf, up, item_flag, kept_flag,
                                                   node_rows);
    H3_LAUNCHED("merge_flags", 0, s);
    temp_bytes = l.temp_bytes;
    H3_CUDA(cub::DeviceScan::InclusiveSum(temp, temp_bytes, item_flag, item_scan, N + M, s));
    temp_bytes = l.temp_bytes;
    H3_CUDA(cub::DeviceScan::InclusiveSum(temp, temp_bytes, kept_flag, kept_scan, N, s));
    temp_bytes = l.temp_bytes;
    H3_CUDA(cub::DeviceScan::InclusiveSum(temp, temp_bytes, node_rows, node_rows_scan, N, s));
    totals_kernel<<<1, 1, 0, s>>>(N, M, item_scan, kept_scan, node_rows_scan, hdr);
    H3_LAUNCHED("merge_totals", 0, s);
    H3_CUDA(cudaMemcpyAsync(host, hdr, kMergeHdr * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    H3_CUDA(cudaStreamSynchronize(s));
    const int R = host[4], kept = host[5];
    if (R < 1) {
        set_error("merge_hierarchies: no chunk owns any leaf Gaussian"); return H3DGS_EINVAL;
    }
    const int64_t NO64 = 2 * (int64_t)R - 1 + kept;
    if (NO64 > kMaxInt) {
        set_error("merge_hierarchies: %lld output nodes (at most 2^31 - 1)", (long long)NO64); return H3DGS_EINVAL;
    }
    // rows: one merged row per top interior node, one per one-Gaussian item, and the kept input nodes' blocks
    const int64_t RO64 = (int64_t)(R - 1) + (R - host[7]) + host[6];
    if (RO64 > kMaxInt) {
        set_error("merge_hierarchies: %lld output rows (at most 2^31 - 1)", (long long)RO64); return H3DGS_EINVAL;
    }
    const int T = 2 * R - 1, NO = (int)NO64, RO = (int)RO64;
    const WorkLayout w = work_layout(R, NO, kept);
    uint8_t* wb = static_cast<uint8_t*>(alloc(alloc_user, 9, w.total));
    if (!wb) { set_error("merge_hierarchies: the work block (%zu bytes) was not allocated", w.total); return H3DGS_ENOMEM; }
    int32_t* item_ref = reinterpret_cast<int32_t*>(wb + w.item_ref);
    int32_t* item_depth = reinterpret_cast<int32_t*>(wb + w.item_depth);
    float* item_pos = reinterpret_cast<float*>(wb + w.item_pos);
    double* item_mom = reinterpret_cast<double*>(wb + w.item_mom);
    double* item_sh = reinterpret_cast<double*>(wb + w.item_sh);
    float* item_box = reinterpret_cast<float*>(wb + w.item_box);
    int32_t* seg = reinterpret_cast<int32_t*>(wb + w.seg);
    int32_t* slot = reinterpret_cast<int32_t*>(wb + w.slot);
    int32_t* kept_list = reinterpret_cast<int32_t*>(wb + w.kept_list);
    int64_t* cnts = reinterpret_cast<int64_t*>(wb + w.counts);
    int64_t* ends = reinterpret_cast<int64_t*>(wb + w.starts);
    uint8_t* tree_base = wb + w.tree;
    const Out tree{reinterpret_cast<float*>(wb + w.txyz), reinterpret_cast<float*>(wb + w.tshs),
                   reinterpret_cast<float*>(wb + w.topac), reinterpret_cast<float*>(wb + w.tls),
                   reinterpret_cast<float*>(wb + w.trot), reinterpret_cast<float*>(wb + w.tboxes),
                   reinterpret_cast<int32_t*>(wb + w.tnodes), reinterpret_cast<int32_t*>(wb + w.tsrc)};

    // 3. items, their moments, the top tree
    item_kernel<<<blocks(N + M, 256), 256, 0, s>>>(N, M, R, in, claim, row_node, row_flag, impure, up, item_flag, item_scan,
                                                   item_ref, item_depth, keys_a, vals_a);
    H3_LAUNCHED("merge_items", 0, s);
    int key_bits = 1;
    while (key_bits < 32 && (int64_t(1) << key_bits) <= R) key_bits++;
    temp_bytes = l.temp_bytes;
    H3_CUDA(cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys_a, keys_b, vals_a, vals_b, M, 0, key_bits, s));
    H3_LAUNCHED("merge_sort_rows", 0, s);
    seg_kernel<<<blocks(M, 256), 256, 0, s>>>(M, R, keys_b, seg);
    H3_LAUNCHED("merge_segments", 0, s);
    moment_kernel<<<blocks(R, 4), 128, 0, s>>>(R, in, vals_b, seg, item_ref, item_mom, item_sh, item_pos, item_box);
    H3_LAUNCHED("merge_moments", 0, s);
    int32_t* thdr = reinterpret_cast<int32_t*>(tree_base + w.b.hdr);
    H3_CUDA(cudaMemsetAsync(thdr, 0, kHdrWords * sizeof(int32_t), s));
    bbox_kernel<<<min(blocks(R, 256), 1024), 256, 0, s>>>(R, item_pos, reinterpret_cast<uint32_t*>(thdr));
    H3_LAUNCHED("merge_bbox", 0, s);
    int32_t box_words[8];
    H3_CUDA(cudaMemcpyAsync(box_words, thdr, 8 * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    H3_CUDA(cudaStreamSynchronize(s));
    const int rc = build_tree(R, item_pos, quant_of(box_words), w.b, tree_base, ItemLeaves{item_mom, item_sh, item_box, item_depth},
                              tree, s, "merge_hierarchies");
    if (rc != H3DGS_OK) return rc;

    // 4. the output nodes and their row blocks
    slot_kernel<<<blocks(T, 256), 256, 0, s>>>(T, tree.nodes, tree.source, slot);
    H3_LAUNCHED("merge_slots", 0, s);
    map_kernel<<<blocks(N, 256), 256, 0, s>>>(N, T, item_flag, item_scan, kept_flag, kept_scan, slot, out_of_node, kept_list);
    H3_LAUNCHED("merge_map", 0, s);
    count_kernel<<<blocks(NO, 256), 256, 0, s>>>(NO, T, nodes, tree.nodes, tree.source, item_ref, kept_list, cnts);
    H3_LAUNCHED("merge_counts", 0, s);
    temp_bytes = w.temp_bytes;
    H3_CUDA(cub::DeviceScan::InclusiveSum(wb + w.temp, temp_bytes, cnts, ends, NO, s));     // ends[NO - 1] == RO

    // 5. outputs
    const size_t fb = sizeof(float), ib = sizeof(int32_t);
    const size_t bytes[9] = {(size_t)RO * 3 * fb, (size_t)RO * kSH * fb, (size_t)RO * fb, (size_t)RO * 3 * fb,
                             (size_t)RO * 4 * fb, (size_t)NO * 7 * ib, (size_t)NO * 8 * fb, (size_t)RO * ib, (size_t)RO * ib};
    void* p[9];
    for (int k = 0; k < 9; k++) {
        p[k] = alloc(alloc_user, k, bytes[k]);
        if (!p[k]) { set_error("merge_hierarchies: output %d (%zu bytes) was not allocated", k, bytes[k]); return H3DGS_ENOMEM; }
    }
    const Dst out{(float*)p[0], (float*)p[1], (float*)p[2], (float*)p[3], (float*)p[4], (float*)p[6], (int32_t*)p[5],
                  (int32_t*)p[7], (int32_t*)p[8]};
    node_out_kernel<<<blocks(NO, 256), 256, 0, s>>>(NO, T, RO, ch, in, tree, item_ref, kept_list, out_of_node, ends, cnts, out);
    H3_LAUNCHED("merge_node_out", 0, s);
    row_copy_kernel<<<blocks(RO, 256), 256, 0, s>>>(RO, ch, in, out);
    H3_LAUNCHED("merge_row_copy", 0, s);
    counts[0] = NO; counts[1] = RO; counts[2] = R;
    return H3DGS_OK;
}
