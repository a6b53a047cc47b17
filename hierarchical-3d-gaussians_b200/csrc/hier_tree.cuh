// hier_tree.cuh -- the LBVH tree build shared by the hierarchy creator (hier_build.cu) and the merger (hier_merge.cu):
// P leaves, each given by a position (for the Morton key) and by what the `Leaves` functor writes into its leaf slot
// (moments, SH, box, depth, source), -> 2P - 1 nodes in BFS order with the merged rows and union boxes of the interior
// nodes.  The rule is include/h3dgs.h h3dgs_build_hierarchy; the merger builds its top tree through the same code.
//
// Pipeline (all on `stream`, scratch from the caller):
//   1. (the caller) the bounding box of the positions -> Quant, the quantisation scale in fp32 on the host
//   2. morton_kernel      63-bit Morton key per leaf (21 bits per axis, x highest), the leaf index as the value
//   3. cub radix sort     stable, 63 key bits
//   4. karras_kernel      one thread per internal node: the radix tree of the augmented keys (key, sorted position)
//                         (Karras 2012), child and parent links in "unified" ids: internal node i -> i, leaf j -> P - 1 + j
//   5. level_kernel       level of every node by walking its parent links; sort key (level << 32) | first sorted position
//   6. cub radix sort     -> BFS order (level, range start); rank_kernel inverts it and records where each level begins
//                         -> read back the level offsets
//   7. leaf_kernel        every node's links in BFS ids; the leaf slots from `Leaves`
//   8. merge_kernel       one launch per level, deepest first: moments of a node from its two children (fp64, carrying
//                         the weight W), eigendecomposition (cyclic Jacobi), the merged row and the union box
// Deterministic: no atomics here.  Files including this are compiled with -fmad=false: the Morton quantisation is
// pinned fp32 arithmetic.
#pragma once
#include <cub/cub.cuh>
#include <float.h>
#include <math.h>
#include "common.cuh"
#include "float_key.cuh"

namespace h3dgs {
namespace {

constexpr int kThreads = 128;
constexpr int kMaxLevels = 128;           // the augmented key has 63 + 32 bits: at most 96 levels
constexpr int kSH = 48;                   // 16 coefficients x 3 channels
constexpr int kMoments = 10;              // W, mu[3], Sigma[6] (xx xy xz yy yz zz)
constexpr double kEigFloor = 1e-24;       // eigenvalues of a merged covariance are floored here (sigma >= 1e-12)
constexpr unsigned kFull = 0xffffffffu;
constexpr float kMaxLogScale = 300.0f;    // above it, sigma^2 = exp(2 log_scale) and the moments would overflow fp64

// hdr (int32 words): [0..2] ~key(min xyz) [3..5] key(max xyz) [6] bad input [7] number of levels
//                    [8 .. 8 + kMaxLevels] first BFS position of every level (then N)
constexpr int kHdrWords = 8 + kMaxLevels + 1;

struct BuildLayout {
    size_t hdr, keys_a, keys_b, vals_a, vals_b, src, left, right, parent, first, rank, moments, sh, temp, total;
    size_t temp_bytes;
};

BuildLayout build_layout(int64_t P) {
    BuildLayout l; size_t o = 0;
    const size_t n = (size_t)P, N = 2 * n - 1, I = n - 1;
    size_t t1 = 0, t2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, t1, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int)n, 0, 63);
    cub::DeviceRadixSort::SortPairs(nullptr, t2, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int)N, 0, 40);
    l.temp_bytes = t1 > t2 ? t1 : t2;
    l.hdr = o;     o += align_up(kHdrWords * sizeof(int32_t));
    l.keys_a = o;  o += align_up(N * sizeof(uint64_t));
    l.keys_b = o;  o += align_up(N * sizeof(uint64_t));
    l.vals_a = o;  o += align_up(N * sizeof(uint32_t));
    l.vals_b = o;  o += align_up(N * sizeof(uint32_t));
    l.src = o;     o += align_up(n * sizeof(uint32_t));
    l.left = o;    o += align_up((I ? I : 1) * sizeof(int32_t));
    l.right = o;   o += align_up((I ? I : 1) * sizeof(int32_t));
    l.parent = o;  o += align_up(N * sizeof(int32_t));
    l.first = o;   o += align_up((I ? I : 1) * sizeof(int32_t));
    l.rank = o;    o += align_up(N * sizeof(int32_t));
    l.moments = o; o += align_up(N * kMoments * sizeof(double));
    l.sh = o;      o += align_up(N * kSH * sizeof(double));
    l.temp = o;    o += align_up(l.temp_bytes);
    l.total = o;
    return l;
}

// the bounding box of P positions into hdr[0..5] (hdr zeroed by the caller)
__global__ void __launch_bounds__(256) bbox_kernel(int P, const float* __restrict__ xyz, uint32_t* __restrict__ hdr) {
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x)
        for (int a = 0; a < 3; a++) {
            const float x = xyz[3 * (size_t)i + a];
            lo[a] = fminf(lo[a], x); hi[a] = fmaxf(hi[a], x);
        }
    for (int a = 0; a < 3; a++) { lo[a] = warp_min(lo[a]); hi[a] = warp_max(hi[a]); }
    if ((threadIdx.x & 31) == 0)
        for (int a = 0; a < 3; a++) { atomicMax(hdr + a, ~f2key(lo[a])); atomicMax(hdr + 3 + a, f2key(hi[a])); }
}

__device__ __forceinline__ uint64_t spread21(uint32_t v) {          // bit k -> bit 3k
    uint64_t x = v & 0x1fffffu;
    x = (x | (x << 32)) & 0x1f00000000ffffull;
    x = (x | (x << 16)) & 0x1f0000ff0000ffull;
    x = (x | (x << 8)) & 0x100f00f00f00f00full;
    x = (x | (x << 4)) & 0x10c30c30c30c30c3ull;
    x = (x | (x << 2)) & 0x1249249249249249ull;
    return x;
}
// q = min(2097151, (uint32)((x - lo) * s)), every operation rounded in fp32 (a NaN product, which only an infinite
// extent can make, maps to the last cell)
__device__ __forceinline__ uint32_t cell21(float x, float lo, float s) {
    const float t = (x - lo) * s;
    return t < 2097151.0f ? (uint32_t)t : 2097151u;
}

struct Quant { float lo[3], s[3]; };

// the quantisation of the box read back from hdr[0..5]
inline Quant quant_of(const int32_t* host) {
    Quant q;
    for (int a = 0; a < 3; a++) {
        const float lo = key2f(~(uint32_t)host[a]), hi = key2f((uint32_t)host[3 + a]);
        q.lo[a] = lo;
        q.s[a] = hi == lo ? 0.0f : 2097152.0f / (hi - lo);
    }
    return q;
}

__global__ void __launch_bounds__(256) morton_kernel(int P, const float* __restrict__ xyz, Quant q, uint64_t* __restrict__ keys,
                                                     uint32_t* __restrict__ vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float* p = xyz + 3 * (size_t)i;
    keys[i] = (spread21(cell21(p[0], q.lo[0], q.s[0])) << 2) | (spread21(cell21(p[1], q.lo[1], q.s[1])) << 1) |
              spread21(cell21(p[2], q.lo[2], q.s[2]));
    vals[i] = (uint32_t)i;
}

__device__ __forceinline__ int clz64(uint64_t x) {
    const uint32_t h = (uint32_t)(x >> 32);
    return h ? __clz((int)h) : 32 + __clz((int)(uint32_t)x);
}
// length of the common prefix of the augmented keys (key, position) at sorted positions i and j; -1 outside [0, P)
__device__ __forceinline__ int delta(const uint64_t* __restrict__ k, int P, int i, long long j) {     // j in 64 bits: the search steps past 2^31
    if (j < 0 || j >= P) return -1;
    const uint64_t x = k[i] ^ k[j];
    return x ? clz64(x) : 64 + __clz((int)((uint32_t)i ^ (uint32_t)j));
}

// Karras, "Maximizing parallelism in the construction of BVHs, octrees, and k-d trees" (HPG 2012), section 4
__global__ void __launch_bounds__(kThreads) karras_kernel(int P, const uint64_t* __restrict__ k, int32_t* __restrict__ left,
                                                          int32_t* __restrict__ right, int32_t* __restrict__ parent,
                                                          int32_t* __restrict__ first) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P - 1) return;
    const int d = delta(k, P, i, i + 1) > delta(k, P, i, i - 1) ? 1 : -1;
    const int dmin = delta(k, P, i, i - d);
    long long lmax = 2;
    while (delta(k, P, i, i + lmax * d) > dmin) lmax *= 2;
    int l = 0;                                                       // < P
    for (long long t = lmax / 2; t >= 1; t /= 2)
        if (delta(k, P, i, i + (l + t) * d) > dmin) l += (int)t;
    const int j = i + l * d;
    const int dnode = delta(k, P, i, j);
    int s = 0, t = l;
    do {
        t = (t + 1) >> 1;
        if (s + t < l && delta(k, P, i, i + (long long)(s + t) * d) > dnode) s += t;
    } while (t > 1);
    const int gamma = i + s * d + min(d, 0);
    const int lo = min(i, j), hi = max(i, j);
    const int a = lo == gamma ? P - 1 + gamma : gamma;
    const int b = hi == gamma + 1 ? P - 1 + gamma + 1 : gamma + 1;
    left[i] = a; right[i] = b; first[i] = lo;
    parent[a] = i; parent[b] = i;
    if (i == 0) parent[0] = -1;
}

__global__ void __launch_bounds__(kThreads) level_kernel(int N, int P, const int32_t* __restrict__ parent,
                                                         const int32_t* __restrict__ first, uint64_t* __restrict__ keys,
                                                         uint32_t* __restrict__ vals) {
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= N) return;
    uint32_t level = 0;
    for (int p = parent[u]; p >= 0; p = parent[p]) level++;
    const uint32_t f = u < P - 1 ? (uint32_t)first[u] : (uint32_t)(u - (P - 1));
    keys[u] = ((uint64_t)level << 32) | f;
    vals[u] = (uint32_t)u;
}

__global__ void __launch_bounds__(kThreads) rank_kernel(int N, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ order,
                                                        int32_t* __restrict__ rank, int32_t* __restrict__ hdr) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= N) return;
    rank[order[p]] = p;
    const int level = (int)(keys[p] >> 32);
    if (p == 0 || level != (int)(keys[p - 1] >> 32)) hdr[8 + level] = p;
    if (p == N - 1) { hdr[7] = level + 1; hdr[8 + level + 1] = N; }
}

struct Out {
    float *xyz, *shs, *opacities, *log_scales, *rotations, *boxes;
    int32_t *nodes, *source;
};

__device__ __forceinline__ void write_box(float* __restrict__ box, const float lo[3], const float hi[3]) {
    const float e = fmaxf(fmaxf(hi[0] - lo[0], hi[1] - lo[1]), hi[2] - lo[2]);
    reinterpret_cast<float4*>(box)[0] = make_float4(lo[0], lo[1], lo[2], e);
    reinterpret_cast<float4*>(box)[1] = make_float4(hi[0], hi[1], hi[2], 0.f);
}

// a Gaussian's covariance Sigma = R diag(sigma^2) R^T from the normalised quaternion (a zero quaternion counts as the
// identity), its weight o * (s0 s1 + s0 s2 + s1 s2), and its box mu +- 3 sqrt(diag Sigma) rounded to fp32
__device__ __forceinline__ double gauss_moments(const float* ls, const float* r, float o, double C[6]) {
    const double s0 = exp((double)ls[0]), s1 = exp((double)ls[1]), s2 = exp((double)ls[2]);
    double w = r[0], qx = r[1], qy = r[2], qz = r[3];
    const double n = sqrt(w * w + qx * qx + qy * qy + qz * qz);
    if (n > 0.0) { w /= n; qx /= n; qy /= n; qz /= n; } else { w = 1.0; }
    const double R[3][3] = {{1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - w * qz), 2 * (qx * qz + w * qy)},
                            {2 * (qx * qy + w * qz), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - w * qx)},
                            {2 * (qx * qz - w * qy), 2 * (qy * qz + w * qx), 1 - 2 * (qx * qx + qy * qy)}};
    const double v[3] = {s0 * s0, s1 * s1, s2 * s2};
    const int ia[6] = {0, 0, 0, 1, 1, 2}, ib[6] = {0, 1, 2, 1, 2, 2};
#pragma unroll
    for (int e = 0; e < 6; e++)
        C[e] = R[ia[e]][0] * v[0] * R[ib[e]][0] + R[ia[e]][1] * v[1] * R[ib[e]][1] + R[ia[e]][2] * v[2] * R[ib[e]][2];
    return (double)o * (s0 * s1 + s0 * s2 + s1 * s2);
}
__device__ __forceinline__ void gauss_box(const float* x, const double C[6], float* __restrict__ box) {
    float lo[3], hi[3];
    const double diag[3] = {C[0], C[3], C[5]};
    for (int a = 0; a < 3; a++) {
        const double ext = 3.0 * sqrt(diag[a]);
        lo[a] = (float)((double)x[a] - ext);
        hi[a] = (float)((double)x[a] + ext);
    }
    write_box(box, lo, hi);
}

// links of every node in BFS ids; the leaf slots from `leaves(p, s, nd, out, mom, shm)`: s the leaf's input index, nd
// its node (links written; depth is the functor's), its moments at mom + kMoments p and SH at shm + kSH p
template <class Leaves>
__global__ void __launch_bounds__(kThreads) leaf_kernel(int N, int P, const uint32_t* __restrict__ order, const int32_t* __restrict__ rank,
                                                        const int32_t* __restrict__ parent, const int32_t* __restrict__ left,
                                                        const uint32_t* __restrict__ src, Leaves leaves, Out out,
                                                        double* __restrict__ mom, double* __restrict__ shm) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= N) return;
    const int u = (int)order[p];
    const bool leaf = u >= P - 1;
    int32_t* nd = out.nodes + 7 * (size_t)p;
    nd[1] = parent[u] >= 0 ? rank[parent[u]] : -1;
    nd[2] = p;
    nd[3] = leaf ? 1 : 0;
    nd[4] = leaf ? 0 : 1;
    nd[5] = leaf ? 0 : rank[left[u]];
    nd[6] = leaf ? 0 : 2;
    if (!leaf) return;
    leaves(p, (int)src[u - (P - 1)], nd, out, mom, shm);
}

// eigenvalues lam and eigenvectors (columns of V) of the symmetric matrix c (xx xy xz yy yz zz): cyclic Jacobi
__device__ void eig_sym3(const double c[6], double lam[3], double V[3][3]) {
    double A[3][3] = {{c[0], c[1], c[2]}, {c[1], c[3], c[4]}, {c[2], c[4], c[5]}};
    for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++) V[a][b] = a == b ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 32; sweep++) {
        const double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2];
        const double dia = A[0][0] * A[0][0] + A[1][1] * A[1][1] + A[2][2] * A[2][2];
        if (!(off > 1e-36 * dia)) break;
#pragma unroll
        for (int pq = 0; pq < 3; pq++) {
            const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
            if (A[p][q] == 0.0) continue;
            const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
            const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
            const double cs = 1.0 / sqrt(t * t + 1.0), sn = t * cs;
            for (int k = 0; k < 3; k++) {
                const double akp = A[k][p], akq = A[k][q];
                A[k][p] = cs * akp - sn * akq; A[k][q] = sn * akp + cs * akq;
            }
            for (int k = 0; k < 3; k++) {
                const double apk = A[p][k], aqk = A[q][k];
                A[p][k] = cs * apk - sn * aqk; A[q][k] = sn * apk + cs * aqk;
            }
            for (int k = 0; k < 3; k++) {
                const double vkp = V[k][p], vkq = V[k][q];
                V[k][p] = cs * vkp - sn * vkq; V[k][q] = sn * vkp + cs * vkq;
            }
        }
    }
    for (int a = 0; a < 3; a++) lam[a] = A[a][a];
}

// unit quaternion (w >= 0) of the rotation matrix R (det +1)
__device__ void quat_of(const double R[3][3], double q[4]) {
    const double tr = R[0][0] + R[1][1] + R[2][2];
    if (tr > 0.0) {
        const double S = 2.0 * sqrt(tr + 1.0);
        q[0] = 0.25 * S; q[1] = (R[2][1] - R[1][2]) / S; q[2] = (R[0][2] - R[2][0]) / S; q[3] = (R[1][0] - R[0][1]) / S;
    } else if (R[0][0] > R[1][1] && R[0][0] > R[2][2]) {
        const double S = 2.0 * sqrt(1.0 + R[0][0] - R[1][1] - R[2][2]);
        q[0] = (R[2][1] - R[1][2]) / S; q[1] = 0.25 * S; q[2] = (R[0][1] + R[1][0]) / S; q[3] = (R[0][2] + R[2][0]) / S;
    } else if (R[1][1] > R[2][2]) {
        const double S = 2.0 * sqrt(1.0 + R[1][1] - R[0][0] - R[2][2]);
        q[0] = (R[0][2] - R[2][0]) / S; q[1] = (R[0][1] + R[1][0]) / S; q[2] = 0.25 * S; q[3] = (R[1][2] + R[2][1]) / S;
    } else {
        const double S = 2.0 * sqrt(1.0 + R[2][2] - R[0][0] - R[1][1]);
        q[0] = (R[1][0] - R[0][1]) / S; q[1] = (R[0][2] + R[2][0]) / S; q[2] = (R[1][2] + R[2][1]) / S; q[3] = 0.25 * S;
    }
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]) * (q[0] < 0.0 ? -1.0 : 1.0);
    for (int a = 0; a < 4; a++) q[a] /= n;
}

// BFS positions [begin, end) of one level: every interior node from its two children (next level, already done)
__global__ void __launch_bounds__(kThreads) merge_kernel(int begin, int end, Out out, double* __restrict__ mom, double* __restrict__ shm) {
    const int p = begin + blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= end) return;
    int32_t* nd = out.nodes + 7 * (size_t)p;
    if (nd[6] == 0) return;                                          // a leaf: leaf_kernel wrote it
    const int ca = nd[5], cb = ca + 1;
    nd[0] = 1 + max(out.nodes[7 * (size_t)ca], out.nodes[7 * (size_t)cb]);
    out.source[p] = -1;
    const double* ma = mom + kMoments * (size_t)ca;
    const double* mb = mom + kMoments * (size_t)cb;
    const double W = ma[0] + mb[0];
    const double fa = W > 0.0 ? ma[0] / W : 0.5, fb = W > 0.0 ? mb[0] / W : 0.5;   // W = 0: the unweighted mean
    double mu[3], da[3], db[3], C[6];
    for (int a = 0; a < 3; a++) {
        mu[a] = fa * ma[1 + a] + fb * mb[1 + a];
        da[a] = ma[1 + a] - mu[a];
        db[a] = mb[1 + a] - mu[a];
    }
    const int ia[6] = {0, 0, 0, 1, 1, 2}, ib[6] = {0, 1, 2, 1, 2, 2};
#pragma unroll
    for (int e = 0; e < 6; e++)
        C[e] = fa * (ma[4 + e] + da[ia[e]] * da[ib[e]]) + fb * (mb[4 + e] + db[ia[e]] * db[ib[e]]);
    double* m = mom + kMoments * (size_t)p;
    m[0] = W;
    for (int a = 0; a < 3; a++) { m[1 + a] = mu[a]; out.xyz[3 * (size_t)p + a] = (float)mu[a]; }
    for (int e = 0; e < 6; e++) m[4 + e] = C[e];
    const double* sa = shm + kSH * (size_t)ca;
    const double* sb = shm + kSH * (size_t)cb;
    for (int c = 0; c < kSH; c++) {
        const double v = fa * sa[c] + fb * sb[c];
        shm[kSH * (size_t)p + c] = v;
        out.shs[kSH * (size_t)p + c] = (float)v;
    }

    double lam[3], V[3][3];
    eig_sym3(C, lam, V);
    // descending eigenvalues, right-handed frame
#pragma unroll
    for (int a = 0; a < 2; a++)
#pragma unroll
        for (int b = 0; b < 2 - a; b++)
            if (lam[b] < lam[b + 1]) {
                const double tl = lam[b]; lam[b] = lam[b + 1]; lam[b + 1] = tl;
                for (int k = 0; k < 3; k++) { const double tv = V[k][b]; V[k][b] = V[k][b + 1]; V[k][b + 1] = tv; }
            }
    const double det = V[0][0] * (V[1][1] * V[2][2] - V[1][2] * V[2][1]) - V[0][1] * (V[1][0] * V[2][2] - V[1][2] * V[2][0]) +
                       V[0][2] * (V[1][0] * V[2][1] - V[1][1] * V[2][0]);
    if (det < 0.0)
        for (int k = 0; k < 3; k++) V[k][2] = -V[k][2];
    double sg[3];
    for (int a = 0; a < 3; a++) {
        const double l = fmax(lam[a], kEigFloor);
        sg[a] = sqrt(l);
        out.log_scales[3 * (size_t)p + a] = (float)(0.5 * log(l));
    }
    out.opacities[p] = (float)(W / (sg[0] * sg[1] + sg[0] * sg[2] + sg[1] * sg[2]));
    double q[4];
    quat_of(V, q);
    for (int a = 0; a < 4; a++) out.rotations[4 * (size_t)p + a] = (float)q[a];

    const float* ba = out.boxes + 8 * (size_t)ca;
    const float* bb = out.boxes + 8 * (size_t)cb;
    float lo[3], hi[3];
    for (int a = 0; a < 3; a++) { lo[a] = fminf(ba[a], bb[a]); hi[a] = fmaxf(ba[4 + a], bb[4 + a]); }
    write_box(out.boxes + 8 * (size_t)p, lo, hi);
}

inline int blocks(int n, int t) { return (int)(((int64_t)n + t - 1) / t); }    // n up to 2^31 - 1

// steps 2-8 for P >= 1 leaves at positions xyz, quantised by q, in the scratch `base` laid out by l (its hdr in use by
// the caller: words 0..6 are left as they are).  Synchronises `s` once, after the leaves.
template <class Leaves>
int build_tree(int P, const float* xyz, const Quant& q, const BuildLayout& l, uint8_t* base, Leaves leaves, Out out,
               cudaStream_t s, const char* who) {
    const int N = 2 * P - 1;
    int32_t* hdr = reinterpret_cast<int32_t*>(base + l.hdr);
    uint64_t* keys_a = reinterpret_cast<uint64_t*>(base + l.keys_a);
    uint64_t* keys_b = reinterpret_cast<uint64_t*>(base + l.keys_b);
    uint32_t* vals_a = reinterpret_cast<uint32_t*>(base + l.vals_a);
    uint32_t* vals_b = reinterpret_cast<uint32_t*>(base + l.vals_b);
    uint32_t* src = reinterpret_cast<uint32_t*>(base + l.src);
    int32_t* left = reinterpret_cast<int32_t*>(base + l.left);
    int32_t* right = reinterpret_cast<int32_t*>(base + l.right);
    int32_t* parent = reinterpret_cast<int32_t*>(base + l.parent);
    int32_t* first = reinterpret_cast<int32_t*>(base + l.first);
    int32_t* rank = reinterpret_cast<int32_t*>(base + l.rank);
    double* mom = reinterpret_cast<double*>(base + l.moments);
    double* shm = reinterpret_cast<double*>(base + l.sh);
    void* temp = base + l.temp;
    size_t temp_bytes = l.temp_bytes;
    int32_t host[kHdrWords];

    // 2.-3. Morton keys, stable sort
    morton_kernel<<<blocks(P, 256), 256, 0, s>>>(P, xyz, q, keys_a, vals_a);
    H3_LAUNCHED("hier_morton", 0, s);
    H3_CUDA(cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys_a, keys_b, vals_a, src, P, 0, 63, s));
    H3_LAUNCHED("hier_sort_keys", 0, s);

    // 4.-6. radix tree, levels, BFS order
    if (P > 1) {
        karras_kernel<<<blocks(P - 1, kThreads), kThreads, 0, s>>>(P, keys_b, left, right, parent, first);
        H3_LAUNCHED("hier_karras", 0, s);
    } else {
        H3_CUDA(cudaMemsetAsync(parent, 0xff, sizeof(int32_t), s));
    }
    level_kernel<<<blocks(N, kThreads), kThreads, 0, s>>>(N, P, parent, first, keys_a, vals_a);
    H3_LAUNCHED("hier_level", 0, s);
    temp_bytes = l.temp_bytes;
    H3_CUDA(cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys_a, keys_b, vals_a, vals_b, N, 0, 40, s));
    H3_LAUNCHED("hier_sort_nodes", 0, s);
    rank_kernel<<<blocks(N, kThreads), kThreads, 0, s>>>(N, keys_b, vals_b, rank, hdr);
    H3_LAUNCHED("hier_rank", 0, s);
    H3_CUDA(cudaMemcpyAsync(host, hdr, kHdrWords * sizeof(int32_t), cudaMemcpyDeviceToHost, s));

    // 7. links, leaves
    leaf_kernel<Leaves><<<blocks(N, kThreads), kThreads, 0, s>>>(N, P, vals_b, rank, parent, left, src, leaves, out, mom, shm);
    H3_LAUNCHED("hier_leaf", 0, s);
    H3_CUDA(cudaStreamSynchronize(s));
    const int levels = host[7];
    if (levels < 1 || levels > kMaxLevels) {
        set_error("%s: %d levels", who, levels); return H3DGS_ECUDA;
    }

    // 8. bottom-up merge, one level per launch (the deepest level holds leaves only)
    for (int lv = levels - 2; lv >= 0; lv--) {
        const int b = host[8 + lv], e = host[8 + lv + 1];
        merge_kernel<<<blocks(e - b, kThreads), kThreads, 0, s>>>(b, e, out, mom, shm);
        H3_LAUNCHED("hier_merge", 0, s);
    }
    return H3DGS_OK;
}

}  // namespace
}  // namespace h3dgs
