// binning.cu -- K2..K5 of the path: inclusive scan of tiles_touched, duplicateWithKeys,
// (tile | depth) radix sort, identifyTileRanges, plus the step that
// MATERIALISES the depth-sorted per-tile record lists contiguously so that the
// blend kernels stream them with cp.async.bulk (TMA) instead of gathering.
// Semantics per oracle/oracle.c::oracle_bin.  Compiled with -fmad=false like
// preprocess.cu (the rect is re-derived from the stored pixel centre and radius).
#include <cub/cub.cuh>
#include "common.cuh"
#include "reach_mask.cuh"

namespace h3dgs {

size_t scan_temp_bytes(int n) {
    size_t bytes = 0;
    cub::DeviceScan::InclusiveSum(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, n > 0 ? n : 1);
    return bytes;
}
size_t sort_temp_bytes(int64_t n) {
    size_t bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                    (const uint32_t*)nullptr, (uint32_t*)nullptr, n > 0 ? n : 1);
    return bytes;
}

int launch_scan(const uint32_t* in, uint32_t* out, int n, void* temp, size_t temp_bytes, cudaStream_t s, bool debug) {
    if (n == 0) return H3DGS_OK;
    ProfScope prof(H3DGS_STAGE_SCAN, s);
    H3_CUDA(cub::DeviceScan::InclusiveSum(temp, temp_bytes, in, out, n, s));
    H3_LAUNCHED("scan", debug, s);
    return H3DGS_OK;
}

// One thread per Gaussian; emission order inside a Gaussian is y-outer, x-inner, and
// across Gaussians it is index order (offsets from the scan) -- with the stable sort
// this fixes the order of equal-depth entries exactly as the oracle's.
__global__ void __launch_bounds__(256)
duplicate_with_keys_kernel(int P, int W, int H, int shard_count, int shard_index, const int* __restrict__ radii,
                           const float* __restrict__ depths, const uint32_t* __restrict__ offsets,
                           const Record* __restrict__ records, uint64_t* __restrict__ keys,
                           uint32_t* __restrict__ vals)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int rad = radii[i];
    if (rad <= 0) return;
    const float4 a = records[i].a;
    const float ix = a.x, iy = a.y;
    const int gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
    const TileRect rect = tile_rect(ix, iy, rad, gx, gy);
    const int rminx = rect.x, rminy = rect.y, rmaxx = rect.z, rmaxy = rect.w;
    uint32_t off = (i == 0) ? 0u : offsets[i - 1];
    const uint32_t dbits = __float_as_uint(depths[i]);
    for (int y = rminy; y < rmaxy; y++) {
        if (shard_count > 1 && (y % shard_count) != shard_index) continue;
        for (int x = rminx; x < rmaxx; x++) {
            uint64_t key = (uint64_t)(y * gx + x);
            key = (key << 32) | dbits;
            keys[off] = key;
            vals[off] = (uint32_t)i;
            off++;
        }
    }
}

__global__ void __launch_bounds__(256)
identify_tile_ranges_kernel(int64_t D, const uint64_t* __restrict__ keys, uint32_t* __restrict__ ranges)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= D) return;
    const uint32_t tile = (uint32_t)(keys[i] >> 32);
    if (i == 0) ranges[2 * tile] = 0;
    else {
        const uint32_t prev = (uint32_t)(keys[i - 1] >> 32);
        if (prev != tile) { ranges[2 * prev + 1] = (uint32_t)i; ranges[2 * tile] = (uint32_t)i; }
    }
    if (i == D - 1) ranges[2 * tile + 1] = (uint32_t)D;
}

// kbits of the per-tile SORTED record copy: bits 0..15 num_node_kids (saturated at 65535), bits 16..31 the block mask.
// (The unsorted record keeps K1's layout: kids in bits 0..19, SH clamp flags in 20..22.)
__device__ __forceinline__ uint32_t sorted_kbits(uint32_t kbits, uint32_t mask16) {
    return min(kbits & kKidsMask, kSortedKidsMask) | (mask16 << kBlockShift);
}

// sorted_records[j] = records[point_list[j]] : 48-B gathers out of an L2-resident array.
// One thread per entry.  While the record is in registers, derive which of the four 8x8-pixel
// quadrants (= warps of the blend CTAs) of ITS tile the entry can reach at all: alpha >= 1/255
// needs q(d) = d^T Q d <= 2 ln(255 o); the exact minimum of the convex q over the quadrant's rectangle of
// pixel centres (0 if the mean is inside, else attained on an edge) is compared with that bound.  The
// test is conservative (margin for fp32 rounding; the hierarchy weight only lowers alpha), so skipping
// a quadrant never changes a result; the 4-bit mask is stored in spare bits of kbits.
__global__ void __launch_bounds__(256)
gather_records_kernel(int64_t D, const uint32_t* __restrict__ point_list, const uint64_t* __restrict__ keys, int gx,
                      const Record* __restrict__ records, Record* __restrict__ sorted)
{
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= D) return;
    const uint32_t g = point_list[j];
    const float4* src = reinterpret_cast<const float4*>(records + g);
    const float4 a = __ldg(src), b = __ldg(src + 1), c = __ldg(src + 2);
    const uint32_t tile = (uint32_t)(keys[j] >> 32);
    const int tile_y = (int)(tile / (uint32_t)gx), tile_x = (int)(tile - (uint32_t)tile_y * (uint32_t)gx);
    const uint32_t kb = sorted_kbits(__float_as_uint(b.w), block_mask16(a, b, tile_x, tile_y));
    float4* dst = reinterpret_cast<float4*>(sorted + j);
    dst[0] = a;
    dst[1] = make_float4(b.x, b.y, b.z, __uint_as_float(kb));
    dst[2] = c;
}

// ------------------------------------------------------------------------------------------
// Per-tile path (default): K1 has left a per-tile histogram.  (1) one CTA scans it into
// ranges[T] and reports D and the longest list; (2) every Gaussian drops (depth bits, idx) into
// its tiles' segments (slot claimed with an atomic -- order inside a segment is arbitrary);
// (3) one CTA per tile sorts its segment -- in registers up to 1024 entries, in shared memory beyond -- by the 64-bit key (depth bits, idx)
// -- exactly the order of a stable sort on depth over emission-in-index-order -- and, while the
// index is in registers, gathers the 48-B record and its quadrant-reach mask.  HBM traffic:
// 8 D (emit) + 8 D (read) + 12 D (keys/list out) + 96 D (records) instead of ~7 x 24 D for the
// global radix sort plus the separate gather.
// ------------------------------------------------------------------------------------------
// One CTA, kScanItems consecutive tiles per thread per pass (8160 tiles at 1080p = one pass of 1024 x 8): a thread
// scans its items in registers, one block-wide scan of the thread sums follows.
constexpr int kScanItems = 8;
__global__ void __launch_bounds__(1024)
tile_scan_kernel(int T, const uint32_t* __restrict__ tile_count, uint2* __restrict__ ranges, ScanInfo* __restrict__ info,
                 uint32_t cap_entries, uint32_t cap_list)
{
    __shared__ uint32_t s_warp[32];
    __shared__ uint32_t s_carry, s_max;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { s_carry = 0; s_max = 0; }
    __syncthreads();
    uint32_t local_max = 0;
    for (int base = 0; base < T; base += 1024 * kScanItems) {
        const int t0 = base + tid * kScanItems;
        uint32_t cnt[kScanItems], sum = 0;
#pragma unroll
        for (int k = 0; k < kScanItems; k++) {
            cnt[k] = (t0 + k) < T ? tile_count[t0 + k] : 0u;
            local_max = max(local_max, cnt[k]);
            sum += cnt[k];
        }
        uint32_t incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            uint32_t w = s_warp[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += v; }
            s_warp[lane] = w;
        }
        __syncthreads();
        uint32_t start = s_carry + (warp ? s_warp[warp - 1] : 0u) + incl - sum;
#pragma unroll
        for (int k = 0; k < kScanItems; k++) {
            if ((t0 + k) < T) ranges[t0 + k] = cnt[k] ? make_uint2(start, start + cnt[k]) : make_uint2(0u, 0u);   // empty tiles: (0,0)
            start += cnt[k];
        }
        __syncthreads();
        if (tid == 1023) s_carry = start;
        __syncthreads();
    }
    local_max = __reduce_max_sync(0xffffffffu, local_max);
    if (lane == 0) atomicMax(&s_max, local_max);
    __syncthreads();
    // capacity mode (cap_entries > 0): a frame that does not fit is turned into an empty one
    const bool overflow = cap_entries != 0u && (s_carry > cap_entries || s_max > cap_list);
    if (tid == 0) { info->D = s_carry; info->max_count = s_max; info->overflow = overflow ? 1u : 0u; }      // prefilter_bad: K1's
    if (overflow)
        for (int t = tid; t < T; t += 1024) ranges[t] = make_uint2(0u, 0u);
}

__global__ void __launch_bounds__(256)
emit_to_tiles_kernel(int P, int W, int H, int shard_count, int shard_index, const int* __restrict__ radii,
                     const float* __restrict__ depths, const Record* __restrict__ records,
                     const uint2* __restrict__ ranges, const ScanInfo* __restrict__ info,
                     uint32_t* __restrict__ tile_count, uint2* __restrict__ pairs)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int rad = radii[i];
    if (rad <= 0) return;
    if (info->overflow) return;                  // capacity mode: the segments would not fit `pairs`
    const float4 a = records[i].a;
    const float ix = a.x, iy = a.y;
    const int gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
    const TileRect rect = tile_rect(ix, iy, rad, gx, gy);
    const int rminx = rect.x, rminy = rect.y, rmaxx = rect.z, rmaxy = rect.w;
    const uint32_t dbits = __float_as_uint(depths[i]);
    // The slot claims return a value, so each costs a full L2 round trip: walk the rect as a flat index
    // and keep four independent claims (then four range loads, then four stores) in flight per thread.
    const int w = rmaxx - rminx, area = w * (rmaxy - rminy);
    for (int t0 = 0; t0 < area; t0 += 4) {
        int tl[4]; uint32_t sl[4], st[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            tl[k] = -1;
            const int t = t0 + k;
            if (t < area) {
                const int y = rminy + t / w, x = rminx + t % w;
                if (shard_count <= 1 || (y % shard_count) == shard_index) tl[k] = y * gx + x;
            }
        }
#pragma unroll
        for (int k = 0; k < 4; k++) if (tl[k] >= 0) sl[k] = atomicSub(tile_count + tl[k], 1u) - 1u;   // histogram doubles as cursor
#pragma unroll
        for (int k = 0; k < 4; k++) if (tl[k] >= 0) st[k] = ranges[tl[k]].x;
#pragma unroll
        for (int k = 0; k < 4; k++)
            if (tl[k] >= 0) pairs[st[k] + sl[k]] = make_uint2((uint32_t)i, dbits);   // little-endian u64 = depth << 32 | idx
    }
}

// one CTA (128 threads) per tile: bitonic sort of (depth bits << 32 | idx), then gather.
//
// Lists of up to 128 x 8 entries are sorted IN REGISTERS: thread t holds the IPT consecutive elements
// t*IPT .. t*IPT + IPT-1 of a network over M = 128*IPT keys, so of the log2(M)(log2(M)+1)/2 stages (45 for
// M = 512) the strides below IPT are compare-exchanges between a thread's own registers, the strides below
// 32*IPT are one 64-bit lane exchange per element (partner lane = lane ^ stride/IPT), and only the three stages
// whose stride crosses warps go through shared memory (element r of thread t at [r][t]: conflict-free).  The
// shared-memory network it replaces met at a block barrier after every stage and was issue-bound on LDS/STS
// and its bank conflicts.  Longer lists (up to
// kTileSortCap) keep the shared-memory network.
constexpr int kSortThreads = 128;
constexpr int kSortRegCap = kSortThreads * 8;

template <int IPT>
__device__ __forceinline__ void sort_tile_in_registers(uint64_t* s_key, int n, const uint64_t* __restrict__ src)
{
    constexpr int M = kSortThreads * IPT;
    const int tid = threadIdx.x, lane = tid & 31;
    // coalesced load, then the thread's IPT consecutive elements
    for (int k = tid; k < M; k += kSortThreads) s_key[k] = k < n ? src[k] : 0xFFFFFFFFFFFFFFFFull;
    __syncthreads();
    uint64_t key[IPT];
#pragma unroll
    for (int r = 0; r < IPT; r++) key[r] = s_key[tid * IPT + r];
    __syncthreads();
#pragma unroll
    for (int size = 2; size <= M; size <<= 1) {
#pragma unroll
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            if (stride >= 32 * IPT) {                                  // partner in another warp
#pragma unroll
                for (int r = 0; r < IPT; r++) s_key[r * kSortThreads + tid] = key[r];
                __syncthreads();
                const int ptid = tid ^ (stride / IPT);
                const bool keep_min = ((tid & (stride / IPT)) == 0) == (((tid * IPT) & size) == 0);
#pragma unroll
                for (int r = 0; r < IPT; r++) {
                    const uint64_t y = s_key[r * kSortThreads + ptid];
                    if ((key[r] > y) == keep_min) key[r] = y;
                }
                __syncthreads();
            } else if (stride >= IPT) {                                // partner in another lane of this warp
                const int lmask = stride / IPT;
                const bool keep_min = ((lane & lmask) == 0) == (((tid * IPT) & size) == 0);
#pragma unroll
                for (int r = 0; r < IPT; r++) {
                    const uint64_t y = __shfl_xor_sync(0xffffffffu, key[r], lmask);
                    if ((key[r] > y) == keep_min) key[r] = y;
                }
            } else {                                                   // both in this thread's registers
#pragma unroll
                for (int r = 0; r < IPT; r++) {
                    if ((r & stride) == 0) {
                        const bool up = (((tid * IPT + r) & size) == 0);
                        const uint64_t x = key[r], y = key[r + stride];
                        if ((x > y) == up) { key[r] = y; key[r + stride] = x; }
                    }
                }
            }
        }
    }
#pragma unroll
    for (int r = 0; r < IPT; r++) s_key[tid * IPT + r] = key[r];
    __syncthreads();
}

__global__ void __launch_bounds__(kSortThreads)
tile_sort_gather_kernel(int gx, int rows, int shard_count, int shard_index, const uint2* __restrict__ ranges,
                        const uint64_t* __restrict__ pairs, const Record* __restrict__ records,
                        uint64_t* __restrict__ keys_sorted, uint32_t* __restrict__ point_list,
                        Record* __restrict__ sorted)
{
    extern __shared__ uint64_t s_key[];
    const int tid = threadIdx.x;
    const int tile_x = blockIdx.x % gx;
    const int tile_y = (blockIdx.x / gx) * shard_count + shard_index;
    const uint32_t tile = (uint32_t)(tile_y * gx + tile_x);
    const uint2 range = ranges[tile];
    const int n = (int)(range.y - range.x);
    if (n == 0) return;
    if (n <= kSortThreads) sort_tile_in_registers<1>(s_key, n, pairs + range.x);
    else if (n <= kSortThreads * 2) sort_tile_in_registers<2>(s_key, n, pairs + range.x);
    else if (n <= kSortThreads * 4) sort_tile_in_registers<4>(s_key, n, pairs + range.x);
    else if (n <= kSortRegCap) sort_tile_in_registers<8>(s_key, n, pairs + range.x);
    else {
        int m = 32;
        while (m < n) m <<= 1;
        for (int k = tid; k < m; k += kSortThreads) s_key[k] = k < n ? pairs[range.x + k] : 0xFFFFFFFFFFFFFFFFull;
        __syncthreads();
        for (int size = 2; size <= m; size <<= 1) {
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                for (int k = tid; k < (m >> 1); k += kSortThreads) {
                    const int lo = 2 * k - (k & (stride - 1));             // index of the lower partner
                    const int hi = lo + stride;
                    const bool up = (lo & size) == 0;
                    const uint64_t x = s_key[lo], y = s_key[hi];
                    if ((x > y) == up) { s_key[lo] = y; s_key[hi] = x; }
                }
                __syncthreads();
            }
        }
    }
    for (int k = tid; k < n; k += kSortThreads) {
        const uint64_t key = s_key[k];
        const uint32_t g = (uint32_t)key, dbits = (uint32_t)(key >> 32);
        const size_t pos = (size_t)range.x + k;
        keys_sorted[pos] = ((uint64_t)tile << 32) | dbits;
        point_list[pos] = g;
        const float4* src = reinterpret_cast<const float4*>(records + g);
        const float4 a = __ldg(src), b = __ldg(src + 1), c = __ldg(src + 2);
        const uint32_t kb = sorted_kbits(__float_as_uint(b.w), block_mask16(a, b, tile_x, tile_y));
        float4* dst = reinterpret_cast<float4*>(sorted + pos);
        dst[0] = a;
        dst[1] = make_float4(b.x, b.y, b.z, __uint_as_float(kb));
        dst[2] = c;
    }
}

int launch_binning(const h3dgs_raster_args& a, const int32_t* radii, const float* depths, const uint32_t* offsets,
                   const Record* records, int64_t D, uint8_t* bin, const BinLayout& bl, uint32_t* ranges,
                   cudaStream_t s)
{
    const int W = a.image_width, H = a.image_height;
    const int gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
    H3_CUDA(cudaMemsetAsync(ranges, 0, (size_t)gx * gy * 2 * sizeof(uint32_t), s));
    if (D == 0 || a.P == 0) return H3DGS_OK;
    uint64_t* keys_u = (uint64_t*)(bin + bl.keys_unsorted);
    uint64_t* keys_s = (uint64_t*)(bin + bl.keys_sorted);
    uint32_t* vals_u = (uint32_t*)(bin + bl.vals_unsorted);
    uint32_t* vals_s = (uint32_t*)(bin + bl.vals_sorted);
    { ProfScope prof(H3DGS_STAGE_DUPLICATE, s);
    duplicate_with_keys_kernel<<<(a.P + 255) / 256, 256, 0, s>>>(a.P, W, H, a.shard_count > 0 ? a.shard_count : 1,
                                                                 a.shard_count > 0 ? a.shard_index : 0, radii, depths,
                                                                 offsets, records, keys_u, vals_u);
    H3_LAUNCHED("duplicate_with_keys", a.debug, s); }
    int tile_bits = 0;
    while ((1 << tile_bits) < gx * gy) tile_bits++;
    size_t temp = bl.sort_temp_bytes;
    { ProfScope prof(H3DGS_STAGE_SORT, s);
    H3_CUDA(cub::DeviceRadixSort::SortPairs(bin + bl.sort_temp, temp, keys_u, keys_s, vals_u, vals_s, D, 0,
                                            32 + tile_bits, s));
    H3_LAUNCHED("radix_sort", a.debug, s); }
    { ProfScope prof(H3DGS_STAGE_RANGES, s);
    identify_tile_ranges_kernel<<<(unsigned)((D + 255) / 256), 256, 0, s>>>(D, keys_s, ranges);
    H3_LAUNCHED("identify_tile_ranges", a.debug, s); }
    { ProfScope prof(H3DGS_STAGE_GATHER, s);
    gather_records_kernel<<<(unsigned)((D + 255) / 256), 256, 0, s>>>(D, vals_s, keys_s, gx, records,
                                                                       (Record*)(bin + bl.sorted_records));
    H3_LAUNCHED("gather_records", a.debug, s); }
    return H3DGS_OK;
}

int launch_tile_scan(const h3dgs_raster_args& a, const uint32_t* tile_count, uint32_t* ranges, ScanInfo* info,
                     uint32_t cap_entries, uint32_t cap_list, cudaStream_t s)
{
    const int gx = (a.image_width + kTile - 1) / kTile, gy = (a.image_height + kTile - 1) / kTile;
    ProfScope prof(H3DGS_STAGE_SCAN, s);
    tile_scan_kernel<<<1, 1024, 0, s>>>(gx * gy, tile_count, (uint2*)ranges, info, cap_entries, cap_list);
    H3_LAUNCHED("tile_scan", a.debug, s);
    return H3DGS_OK;
}

int launch_tile_binning(const h3dgs_raster_args& a, const int32_t* radii, const float* depths, const Record* records,
                        int64_t D, uint32_t max_count, uint8_t* bin, const BinLayout& bl, const uint32_t* ranges,
                        const ScanInfo* info, uint32_t* tile_count, cudaStream_t s)
{
    if (D == 0 || a.P == 0) return H3DGS_OK;
    const int W = a.image_width, H = a.image_height;
    const int gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
    const int sc = a.shard_count > 0 ? a.shard_count : 1, si = a.shard_count > 0 ? a.shard_index : 0;
    const int rows = (gy + sc - 1 - si) / sc;
    uint2* pairs = (uint2*)(bin + bl.keys_unsorted);
    { ProfScope prof(H3DGS_STAGE_DUPLICATE, s);
    emit_to_tiles_kernel<<<(a.P + 255) / 256, 256, 0, s>>>(a.P, W, H, sc, si, radii, depths, records, (const uint2*)ranges,
                                                           info, tile_count, pairs);
    H3_LAUNCHED("emit_to_tiles", a.debug, s); }
    int m = kSortThreads;                                       // the register sort stages at least 128 keys
    while (m < (int)max_count) m <<= 1;
    const size_t smem = (size_t)m * sizeof(uint64_t);
    if (smem > 48 * 1024)     // per device, idempotent: only the rare long lists need the opt-in
        H3_CUDA(cudaFuncSetAttribute(tile_sort_gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     kTileSortCap * (int)sizeof(uint64_t)));
    { ProfScope prof(H3DGS_STAGE_SORT, s);
    tile_sort_gather_kernel<<<gx * rows, kSortThreads, smem, s>>>(gx, rows, sc, si, (const uint2*)ranges, (const uint64_t*)pairs, records,
                                                         (uint64_t*)(bin + bl.keys_sorted), (uint32_t*)(bin + bl.vals_sorted),
                                                         (Record*)(bin + bl.sorted_records));
    H3_LAUNCHED("tile_sort_gather", a.debug, s); }
    return H3DGS_OK;
}

GeomLayout geom_layout(int P) {
    GeomLayout l; size_t o = 0; const size_t n = (size_t)(P > 0 ? P : 1);
    l.depths = o; o = align_up(o + n * 4);
    l.tiles_touched = o; o = align_up(o + n * 4);
    l.offsets = o; o = align_up(o + n * 4);
    l.rank_mask = o; o = align_up(o + n);
    l.records = o; o = align_up(o + n * sizeof(Record));
    l.scan_temp_bytes = scan_temp_bytes(P);
    l.scan_temp = o; o = align_up(o + l.scan_temp_bytes);
    l.total = o;
    return l;
}
BinLayout bin_layout(int64_t D) {
    BinLayout l; size_t o = 0; const size_t n = (size_t)(D > 0 ? D : 1);
    l.keys_unsorted = o; o = align_up(o + n * 8);
    l.keys_sorted = o; o = align_up(o + n * 8);
    l.vals_unsorted = o; o = align_up(o + n * 4);
    l.vals_sorted = o; o = align_up(o + n * 4);
    l.sort_temp_bytes = sort_temp_bytes(D);
    l.sort_temp = o; o = align_up(o + l.sort_temp_bytes);
    l.sorted_records = o; o = align_up(o + (n + 1) * sizeof(Record));
    l.total = o;
    return l;
}
ImgLayout img_layout(int W, int H) {
    ImgLayout l; size_t o = 0;
    const size_t px = (size_t)W * H;
    const size_t tiles = (size_t)((W + kTile - 1) / kTile) * ((H + kTile - 1) / kTile);
    l.final_T = o; o = align_up(o + px * 4);
    l.n_contrib = o; o = align_up(o + px * 4);
    l.ranges = o; o = align_up(o + tiles * 8);
    l.tile_max_contrib = o; o = align_up(o + tiles * 4);
    l.tile_count = o; o = align_up(o + tiles * 4);
    l.scan_info = o; o = align_up(o + sizeof(ScanInfo));
    l.total = o;
    return l;
}

}  // namespace h3dgs
