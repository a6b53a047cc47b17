// lod_budget.cu -- the finest LOD threshold whose cut fits a Gaussian budget, chosen on the device ahead of the cut.
//
// The cut (hierarchy.cu, lod_cut_fused_kernel) is a flat per-node predicate.  With s = the node's box_size and q = its
// parent's, a node emits at threshold t
//     root:      cl             if s >= t, else 0
//     otherwise: cl             if s >= t
//                cl + [d != 0] cm  if !(s >= t) and q >= t
//                0              otherwise
// so the cut's row count is R(t) = sum_k w_k [t <= key_k] over keys that are node sizes: a node whose middle interval is
// not empty (s < q, or s NaN, with q not NaN) puts -[d != 0] cm at s and cl + [d != 0] cm at q, any other node cl at s.
// The term at q = the parent's size belongs to the parent's key, so each node's weight is its own term plus a sum over
// its children (contiguous: start_children, count_children) -- no atomics.  Keys below the floor never count for a
// t >= floor and NaN keys never count at all; they get the largest sort key and weight 0.  Sorting the (key, weight)
// pairs by size, descending, and taking an inclusive sum gives, at the first pair of each run of equal sizes x,
// R(nextafterf(x, +inf)) = the exclusive sum there.  The answer t* is the smallest t in [floor, t_max], t_max =
// max(floor, largest finite size), with R(t) <= budget: floor itself when R(floor) <= budget, else nextafterf(x) of the
// smallest feasible x below t_max (R need not be monotone, so every run is a candidate: one atomicMax over run
// positions, whose result does not depend on the order of the atomics), else t_max with the "unmet" flag.
//
// With the view cull's row mask (lod_cull.cu), cl and cm become the node's masked leaf and merged rows (vl, vm): the
// masked cut has the same per-node predicate with those counts, so the argument above holds unchanged.
//
// Launches: a memset, the key kernel, cub's radix sort and inclusive scan, the selection kernel and a one-thread
// finisher; every size is fixed by N, floor and budget are read on the device, so the call is capturable.
#include <cub/cub.cuh>
#include "common.cuh"
#include "float_key.cuh"
#include "lod_size.cuh"

namespace h3dgs {

constexpr int kBudgetThreads = 256;
// small words at the head of the scratch: keys at or above the floor, 1 + position of the smallest feasible candidate
// (0: none), N - position of the first candidate (0: none), number of +inf keys
enum { kBudgetKept = 0, kBudgetBest, kBudgetFirst, kBudgetInf, kBudgetWords };

__global__ void __launch_bounds__(kBudgetThreads)
budget_keys_kernel(int N, const int* __restrict__ nodes, const float4* __restrict__ boxes, float floor_t,
                   const float* __restrict__ floor_dev, const float* __restrict__ viewpoint, uint32_t* __restrict__ keys,
                   int* __restrict__ weights, int* __restrict__ small, const uint8_t* __restrict__ mask /* NULL: every row */)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (floor_dev) floor_t = *floor_dev;
    const float vx = viewpoint[0], vy = viewpoint[1], vz = viewpoint[2];
    bool kept = false;
    if (i < N) {
        const int* nd = nodes + 7 * (size_t)i;
        const float s = box_size(__ldg(boxes + 2 * (size_t)i), __ldg(boxes + 2 * (size_t)i + 1), vx, vy, vz);
        uint32_t key = 0xFFFFFFFFu;
        int w = 0;
        if (s >= floor_t) {
            kept = true;
            const int parent = nd[1];
            w = mask ? masked_rows(mask, nd[2], nd[3]) : nd[3];
            if (parent != -1) {
                const float q = box_size(__ldg(boxes + 2 * (size_t)parent), __ldg(boxes + 2 * (size_t)parent + 1), vx, vy, vz);
                if (!(s >= q) && q == q)
                    w = nd[0] != 0 ? -(mask ? masked_rows(mask, nd[2] + nd[3], nd[4]) : nd[4]) : 0;
            }
            const int first = nd[5], nk = nd[6];
            for (int c = first; c < first + nk; c++) {           // the children's terms at this node's size
                const int* cd = nodes + 7 * (size_t)c;
                const float sc = box_size(__ldg(boxes + 2 * (size_t)c), __ldg(boxes + 2 * (size_t)c + 1), vx, vy, vz);
                if (!(sc >= s)) {
                    const int rows = cd[3] + (cd[0] != 0 ? cd[4] : 0);
                    w += mask ? masked_rows(mask, cd[2], rows) : rows;
                }
            }
            key = ~f2key(s == 0.0f ? 0.0f : s);                  // -0 and +0 are one size; ascending = sizes descending
        }
        keys[i] = key;
        weights[i] = w;
    }
    const int n = __syncthreads_count(kept);
    if (threadIdx.x == 0 && n) atomicAdd(small + kBudgetKept, n);
}

__device__ __forceinline__ float key_size(uint32_t k) { return key2f(~k); }

// one thread per sorted pair: the end of the +inf run, and every candidate -- the first pair of a run of a finite size
// below the largest finite size -- with its row count
__global__ void __launch_bounds__(kBudgetThreads)
budget_select_kernel(int N, const uint32_t* __restrict__ keys, const int* __restrict__ weights, const int* __restrict__ incl,
                     int budget, const int* __restrict__ budget_dev, int* __restrict__ small)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const int M = small[kBudgetKept];
    if (j >= M) return;
    if (budget_dev) budget = *budget_dev;
    const uint32_t k = keys[j];
    const float x = key_size(k);
    if (x > FLT_MAX) {
        if (j + 1 == M || keys[j + 1] != k) small[kBudgetInf] = j + 1;
        return;
    }
    if (j == 0) return;
    const uint32_t kp = keys[j - 1];
    if (kp == k || key_size(kp) > FLT_MAX) return;
    atomicMax(small + kBudgetFirst, N - j);
    if (incl[j] - weights[j] <= budget) atomicMax(small + kBudgetBest, j + 1);
}

__global__ void budget_finish_kernel(int N, const uint32_t* __restrict__ keys, const int* __restrict__ weights,
                                     const int* __restrict__ incl, float floor_t, const float* __restrict__ floor_dev,
                                     int budget, const int* __restrict__ budget_dev, const int* __restrict__ small,
                                     float* __restrict__ threshold, int* __restrict__ info)
{
    if (floor_dev) floor_t = *floor_dev;
    if (budget_dev) budget = *budget_dev;
    const int M = small[kBudgetKept], best = small[kBudgetBest] - 1, inf = small[kBudgetInf];
    const int total = M > 0 ? incl[M - 1] : 0;                   // R(floor)
    float t = floor_t;
    int rows = total, unmet = 0;
    if (total <= budget) {
    } else if (best >= 0) {
        t = nextafterf(key_size(keys[best]), FLT_MAX);
        rows = incl[best] - weights[best];
    } else {
        unmet = 1;
        if (inf < M) {                                           // t_max = the largest finite size, whose run ends
            t = key_size(keys[inf]);                             // where the first candidate's begins
            rows = incl[small[kBudgetFirst] ? N - small[kBudgetFirst] - 1 : M - 1];
        }
    }
    *threshold = t;
    info[0] = rows; info[1] = unmet; info[2] = M; info[3] = total;
}

struct BudgetLayout { size_t keys_in, keys_out, w_in, w_out, temp, temp_bytes, total; };

static BudgetLayout budget_layout(int N) {
    BudgetLayout l;
    size_t sort_bytes = 0, scan_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int*)nullptr,
                                    (int*)nullptr, N);
    cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (const int*)nullptr, (int*)nullptr, N);
    const size_t a = align_up((size_t)N * 4);
    l.keys_in = align_up(kBudgetWords * sizeof(int));
    l.keys_out = l.keys_in + a;
    l.w_in = l.keys_out + a;
    l.w_out = l.w_in + a;
    l.temp = l.w_out + a;
    l.temp_bytes = sort_bytes > scan_bytes ? sort_bytes : scan_bytes;
    l.total = l.temp + align_up(l.temp_bytes);
    return l;
}

}  // namespace h3dgs

using namespace h3dgs;

extern "C" size_t h3dgs_lod_budget_scratch_bytes(int32_t N) { return budget_layout(N > 0 ? N : 1).total; }

static int lod_budget(const char* who, int32_t N, const int32_t* nodes, const float* boxes, const float* viewpoint,
                      float floor_size, const float* floor_dev, int32_t budget, const int32_t* budget_dev,
                      float* threshold_out, int32_t* info_out, void* scratch, void* stream, const uint8_t* mask)
{
    if (N <= 0) { set_error("%s: empty hierarchy", who); return H3DGS_EINVAL; }
    if (!nodes || !boxes || !viewpoint || !threshold_out || !info_out || !scratch) {
        set_error("%s: NULL argument", who);
        return H3DGS_EINVAL;
    }
    if ((((uintptr_t)boxes) & 15) != 0) { set_error("%s: boxes must be 16-byte aligned (got %p)", who, (const void*)boxes); return H3DGS_EINVAL; }
    if ((((uintptr_t)scratch) & 255) != 0) { set_error("%s: scratch must be 256-byte aligned (got %p)", who, scratch); return H3DGS_EINVAL; }
    if (!budget_dev && budget < 0) { set_error("%s: negative budget %d", who, budget); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope prof(H3DGS_STAGE_LOD_BUDGET, s);
    const BudgetLayout l = budget_layout(N);
    uint8_t* base = (uint8_t*)scratch;
    int* small = (int*)base;
    uint32_t *keys_in = (uint32_t*)(base + l.keys_in), *keys_out = (uint32_t*)(base + l.keys_out);
    int *w_in = (int*)(base + l.w_in), *w_out = (int*)(base + l.w_out);
    size_t temp_bytes = l.temp_bytes;
    const int blocks = (N + kBudgetThreads - 1) / kBudgetThreads;
    H3_CUDA(cudaMemsetAsync(small, 0, kBudgetWords * sizeof(int), s));
    budget_keys_kernel<<<blocks, kBudgetThreads, 0, s>>>(N, nodes, (const float4*)boxes, floor_size, floor_dev, viewpoint,
                                                         keys_in, w_in, small, mask);
    H3_LAUNCHED("lod_budget_keys", 0, s);
    H3_CUDA(cub::DeviceRadixSort::SortPairs(base + l.temp, temp_bytes, keys_in, keys_out, w_in, w_out, N, 0, 32, s));
    H3_LAUNCHED("lod_budget_sort", 0, s);
    int* incl = w_in;                                            // the unsorted weights are spent
    temp_bytes = l.temp_bytes;
    H3_CUDA(cub::DeviceScan::InclusiveSum(base + l.temp, temp_bytes, w_out, incl, N, s));
    H3_LAUNCHED("lod_budget_scan", 0, s);
    budget_select_kernel<<<blocks, kBudgetThreads, 0, s>>>(N, keys_out, w_out, incl, budget, budget_dev, small);
    H3_LAUNCHED("lod_budget_select", 0, s);
    budget_finish_kernel<<<1, 1, 0, s>>>(N, keys_out, w_out, incl, floor_size, floor_dev, budget, budget_dev, small,
                                         threshold_out, info_out);
    H3_LAUNCHED("lod_budget_finish", 0, s);
    return H3DGS_OK;
}

extern "C" int h3dgs_lod_budget(int32_t N, const int32_t* nodes, const float* boxes, const float* viewpoint, float floor_size,
                                const float* floor_dev, int32_t budget, const int32_t* budget_dev, float* threshold_out,
                                int32_t* info_out, void* scratch, void* stream)
{
    return lod_budget("lod_budget", N, nodes, boxes, viewpoint, floor_size, floor_dev, budget, budget_dev, threshold_out,
                      info_out, scratch, stream, nullptr);
}

extern "C" int h3dgs_lod_budget_masked(int32_t N, const int32_t* nodes, const float* boxes, const float* viewpoint,
                                       const uint8_t* row_mask, float floor_size, const float* floor_dev, int32_t budget,
                                       const int32_t* budget_dev, float* threshold_out, int32_t* info_out, void* scratch,
                                       void* stream)
{
    return lod_budget("lod_budget_masked", N, nodes, boxes, viewpoint, floor_size, floor_dev, budget, budget_dev,
                      threshold_out, info_out, scratch, stream, row_mask);
}
