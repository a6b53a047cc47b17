// api.cu -- the extern "C" entry points declared in include/h3dgs.h: argument checks
// (same exclusivity rules the reference's Python shim enforces), state-buffer
// carving, and the stage sequence.  No torch types; device pointers only.
#include <stdarg.h>
#include <string.h>
#include <algorithm>
#include <mutex>
#include <vector>
#include "common.cuh"

namespace h3dgs {

static thread_local char g_err[1024] = "";
int64_t g_launches = 0;
#ifdef H3_SIMT_EMU
long long g_emu_stats[16] = {0};
#endif

void set_error(const char* fmt, ...) {
    va_list ap; va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// ---- stage profiler ----
struct ProfRec { int stage; cudaEvent_t e0, e1; };
static bool g_prof_on = false;
static std::vector<ProfRec> g_prof_pending;
static std::vector<cudaEvent_t> g_prof_pool;
static double g_prof_ms[H3DGS_STAGE_COUNT];
static int64_t g_prof_n[H3DGS_STAGE_COUNT];
static cudaEvent_t g_prof_open[H3DGS_STAGE_COUNT];
static std::mutex g_prof_mu;

static cudaEvent_t prof_event() {
    if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
    cudaEvent_t e; cudaEventCreate(&e); return e;
}
// stage events are timing events: they cannot be recorded into a stream that is being captured
static bool capturing(cudaStream_t s) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    return cudaStreamIsCapturing(s, &st) != cudaSuccess || st != cudaStreamCaptureStatusNone;
}
void prof_begin(int stage, cudaStream_t s) {
    if (!g_prof_on || capturing(s)) return;
    std::lock_guard<std::mutex> lk(g_prof_mu);
    cudaEvent_t e = prof_event();
    cudaEventRecord(e, s);
    g_prof_open[stage] = e;
}
void prof_end(int stage, cudaStream_t s) {
    if (!g_prof_on || capturing(s)) return;
    std::lock_guard<std::mutex> lk(g_prof_mu);
    cudaEvent_t e = prof_event();
    cudaEventRecord(e, s);
    g_prof_pending.push_back({stage, g_prof_open[stage], e});
}
static void prof_drain() {
    for (auto& r : g_prof_pending) {
        float ms = 0.f;
        cudaEventSynchronize(r.e1);
        if (cudaEventElapsedTime(&ms, r.e0, r.e1) == cudaSuccess) { g_prof_ms[r.stage] += ms; g_prof_n[r.stage]++; }
        g_prof_pool.push_back(r.e0); g_prof_pool.push_back(r.e1);
    }
    g_prof_pending.clear();
}

// ---- side stream: zero-filling the full-size gradients (0.7 GB in scatter mode, pure DRAM
// traffic) overlaps the issue-bound per-tile replay instead of preceding the chain rule ----
struct SideStream { cudaStream_t s = nullptr; cudaEvent_t fork = nullptr, join = nullptr; };
static SideStream g_side[64];
static int side_stream(SideStream** out) {
    int dev = 0;
    H3_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64) { set_error("device index %d out of range", dev); return H3DGS_EINVAL; }
    SideStream& ss = g_side[dev];
    if (!ss.s) {
        H3_CUDA(cudaStreamCreateWithFlags(&ss.s, cudaStreamNonBlocking));
        H3_CUDA(cudaEventCreateWithFlags(&ss.fork, cudaEventDisableTiming));
        H3_CUDA(cudaEventCreateWithFlags(&ss.join, cudaEventDisableTiming));
    }
    *out = &ss;
    return H3DGS_OK;
}

// Once work has been forked onto the side stream, EVERY exit path of the entry point -- error returns included -- must
// make the caller's stream wait for it: the caller may free or reuse the buffers the side work still writes.
struct SideJoin {
    SideStream* ss = nullptr; cudaStream_t main = nullptr; bool armed = false;
    void arm(SideStream* s_, cudaStream_t m) { ss = s_; main = m; armed = true; }
    ~SideJoin() {
        if (!armed) return;
        // a fresh record on the side stream covers everything enqueued there so far (idempotent with the explicit joins)
        if (cudaEventRecord(ss->join, ss->s) == cudaSuccess) cudaStreamWaitEvent(main, ss->join, 0);
    }
};

static void* g_pinned[64] = {nullptr};
int pinned_scratch(void** out) {
    int dev = 0;
    H3_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64) { set_error("device index %d out of range", dev); return H3DGS_EINVAL; }
    if (!g_pinned[dev]) H3_CUDA(cudaHostAlloc(&g_pinned[dev], 64, cudaHostAllocDefault));
    *out = g_pinned[dev];
    return H3DGS_OK;
}

static int check_args(const h3dgs_raster_args* a) {
    if (!a) { set_error("args is NULL"); return H3DGS_EINVAL; }
    if (a->P < 0 || a->image_width <= 0 || a->image_height <= 0) { set_error("bad sizes P=%d W=%d H=%d", a->P, a->image_width, a->image_height); return H3DGS_EINVAL; }
    if ((a->shs == nullptr) == (a->colors_precomp == nullptr) && a->P > 0) {
        set_error("Please provide excatly one of either SHs or precomputed colors!"); return H3DGS_EINVAL;
    }
    const bool have_sr = a->scales != nullptr && a->rotations != nullptr;
    const bool any_sr = a->scales != nullptr || a->rotations != nullptr;
    if (a->P > 0 && ((have_sr && a->cov3D_precomp) || (!any_sr && !a->cov3D_precomp) || (any_sr && !have_sr))) {
        set_error("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!"); return H3DGS_EINVAL;
    }
    if (a->shs && (a->sh_degree < 0 || a->sh_degree > 3 || (a->sh_degree + 1) * (a->sh_degree + 1) > a->sh_coeffs || a->sh_coeffs > 16)) {
        set_error("sh_degree %d does not fit %d SH coefficients", a->sh_degree, a->sh_coeffs); return H3DGS_EINVAL;
    }
    if ((a->interpolation_weights == nullptr) != (a->num_node_kids == nullptr)) {
        set_error("interpolation_weights and num_node_kids must be given together"); return H3DGS_EINVAL;
    }
    if ((a->render_indices == nullptr) != (a->parent_indices == nullptr)) {
        set_error("render_indices and parent_indices must be given together"); return H3DGS_EINVAL;
    }
    if (a->render_indices && (!a->interpolation_weights || a->num_source <= 0 || a->colors_precomp || a->cov3D_precomp)) {
        set_error("render_indices needs interpolation_weights/num_node_kids, num_source > 0 and SH + scale/rotation inputs");
        return H3DGS_EINVAL;
    }
    if (a->shard_count > 1 && (a->shard_index < 0 || a->shard_index >= a->shard_count)) {
        set_error("bad tile shard %d/%d", a->shard_index, a->shard_count); return H3DGS_EINVAL;
    }
    if (a->bin_capacity < 0 || a->sort_capacity < 0 || a->sort_capacity > kTileSortCap) {
        set_error("bad capacities: bin %lld, sort %d (max %d)", (long long)a->bin_capacity, a->sort_capacity, kTileSortCap);
        return H3DGS_EINVAL;
    }
    if (a->peer_count > 1) {
        const int n = a->peer_count;
        if (n != a->shard_count || n > H3DGS_MAX_PEERS || (n & (n - 1)) || a->grad_cyclic_log2 < 5 || a->grad_cyclic_log2 > 24 || a->do_depth) {
            set_error("peer mode needs peer_count == shard_count in {2,4,8}, 5 <= grad_cyclic_log2 <= 24, do_depth off (got %d/%d, log2 %d)",
                      n, a->shard_count, a->grad_cyclic_log2);
            return H3DGS_EINVAL;
        }
        for (int r = 0; r < n; r++)
            if ((r == a->shard_index && !a->peer_image[r]) || !a->peer_stage[r]) { set_error("peer mode: peer_image[shard_index] / peer_stage[%d] is NULL", r); return H3DGS_EINVAL; }
    }
    if (a->bin_capacity > 0 && a->debug) { set_error("capacity mode has no host synchronisation: debug must be off"); return H3DGS_EINVAL; }
    if (!a->means3D && a->P > 0) { set_error("means3D is NULL"); return H3DGS_EINVAL; }
    if (!a->bg || !a->viewmatrix || !a->projmatrix || !a->campos) { set_error("bg/viewmatrix/projmatrix/campos must be device pointers"); return H3DGS_EINVAL; }
    return H3DGS_OK;
}

}  // namespace h3dgs

using namespace h3dgs;

extern "C" int h3dgs_profile_enable(int on) { std::lock_guard<std::mutex> lk(g_prof_mu); prof_drain(); g_prof_on = on != 0; return H3DGS_OK; }
extern "C" int h3dgs_profile_reset(void) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    prof_drain();
    for (int i = 0; i < H3DGS_STAGE_COUNT; i++) { g_prof_ms[i] = 0; g_prof_n[i] = 0; }
    return H3DGS_OK;
}
extern "C" int h3dgs_profile_read(int stage, double* total_ms, int64_t* launches) {
    if (stage < 0 || stage >= H3DGS_STAGE_COUNT) { set_error("bad stage %d", stage); return H3DGS_EINVAL; }
    std::lock_guard<std::mutex> lk(g_prof_mu);
    prof_drain();
    if (total_ms) *total_ms = g_prof_ms[stage];
    if (launches) *launches = g_prof_n[stage];
    return H3DGS_OK;
}
extern "C" const char* h3dgs_stage_name(int stage) {
    static const char* names[H3DGS_STAGE_COUNT] = {"preprocess", "scan", "key_emission", "sort", "identify_tile_ranges",
        "gather_records", "render_forward", "render_backward", "preprocess_backward", "lod_cut", "lod_weights",
        "preprocess_color", "sh_backward"};
    return (stage >= 0 && stage < H3DGS_STAGE_COUNT) ? names[stage] : "?";
}
extern "C" const char* h3dgs_last_error(void) { return g_err; }
extern "C" int h3dgs_version(void) { return H3DGS_VERSION; }
extern "C" int64_t h3dgs_launch_count(void) { return g_launches; }
extern "C" size_t h3dgs_backward_scratch_bytes(int32_t P) { return align_up((size_t)(P > 0 ? P : 1) * kAccum * sizeof(float)); }

extern "C" int h3dgs_rasterize_forward(const h3dgs_raster_args* a, h3dgs_alloc_fn alloc, void* user,
                                       float* out_color, int32_t* out_radii, float* out_invdepth,
                                       int64_t* num_rendered, void* stream)
{
    int rc = check_args(a);
    if (rc) return rc;
    if (!alloc || (!out_color && a->peer_count <= 1) || (!out_radii && a->P > 0) || (a->do_depth && !out_invdepth)) {
        set_error("missing output buffer or alloc callback"); return H3DGS_EINVAL;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const int P = a->P;
    const GeomLayout gl = geom_layout(P);
    uint8_t* geom = (uint8_t*)alloc(user, 0, gl.total);
    const ImgLayout il = img_layout(a->image_width, a->image_height);
    uint8_t* img = (uint8_t*)alloc(user, 2, il.total);
    if (!geom || !img) { set_error("alloc callback returned NULL"); return H3DGS_ENOMEM; }
    float* depths = (float*)(geom + gl.depths);
    uint32_t* tiles = (uint32_t*)(geom + gl.tiles_touched);
    uint32_t* offsets = (uint32_t*)(geom + gl.offsets);
    Record* records = (Record*)(geom + gl.records);

    // per-tile histogram (filled by K1) -> ranges (tile_scan writes ScanInfo itself)
    uint32_t* tile_count = (uint32_t*)(img + il.tile_count);
    ScanInfo* info = (ScanInfo*)(img + il.scan_info);
    uint32_t* ranges = (uint32_t*)(img + il.ranges);
    const int gxy = ((a->image_width + kTile - 1) / kTile) * ((a->image_height + kTile - 1) / kTile);
    // one memset covers the histogram and ScanInfo (adjacent regions of the image state)
    H3_CUDA(cudaMemsetAsync(tile_count, 0, (size_t)((uint8_t*)info - (uint8_t*)tile_count) + sizeof(ScanInfo), s));
    (void)gxy;
    rc = launch_preprocess(*a, out_radii, depths, tiles, geom + gl.rank_mask, records, tile_count, info, s);
    if (rc) return rc;
    // SH -> RGB only feeds record.c (read again by the record gather): run it on the side stream,
    // overlapped with the tile scan, the num_rendered round trip and key emission
    SideStream* ss = nullptr;
    SideJoin side_guard;
    const bool side_color = !a->colors_precomp && P > 0 && !a->debug;
    if (side_color) {
        rc = side_stream(&ss);
        if (rc) return rc;
        H3_CUDA(cudaEventRecord(ss->fork, s));
        H3_CUDA(cudaStreamWaitEvent(ss->s, ss->fork, 0));
        side_guard.arm(ss, s);
        rc = launch_preprocess_color(*a, out_radii, tiles, records, ss->s);
        if (rc) return rc;
        H3_CUDA(cudaEventRecord(ss->join, ss->s));
    } else {
        rc = launch_preprocess_color(*a, out_radii, tiles, records, s);
        if (rc) return rc;
    }
    const bool capacity_mode = a->bin_capacity > 0;
    const uint32_t cap_list = (uint32_t)(a->sort_capacity > 0 ? a->sort_capacity : kTileSortCap);
    rc = launch_tile_scan(*a, tile_count, ranges, info, capacity_mode ? (uint32_t)std::min<int64_t>(a->bin_capacity, 0xFFFFFFFFll) : 0u,
                          cap_list, s);
    if (rc) return rc;
    ScanInfo hinfo;
    if (capacity_mode) {
        // sizes fixed by the caller; a frame that does not fit raises ScanInfo::overflow on the device
        hinfo.D = (uint32_t)std::min<int64_t>(a->bin_capacity, 0xFFFFFFFFll); hinfo.max_count = cap_list; hinfo.overflow = 0; hinfo.prefilter_bad = 0;
    } else {
        // The reference API sizes the binning buffer from num_rendered: one D2H + sync.
        void* pin = nullptr;
        rc = pinned_scratch(&pin);
        if (rc) return rc;
        H3_CUDA(cudaMemcpyAsync(pin, info, sizeof(ScanInfo), cudaMemcpyDeviceToHost, s));
        H3_CUDA(cudaStreamSynchronize(s));
        hinfo = *static_cast<const ScanInfo*>(pin);
        if (hinfo.prefilter_bad) {       // the reference's kernel traps here ("Point is filtered although prefiltered is set")
            set_error("Point is filtered although prefiltered is set. This shouldn't happen!"); return H3DGS_EINVAL;
        }
    }
    const int64_t D = (int64_t)hinfo.D;
    if (num_rendered) *num_rendered = D;
    const BinLayout bl = bin_layout(D);
    uint8_t* bin = (uint8_t*)alloc(user, 1, bl.total);
    if (!bin) { set_error("alloc callback returned NULL"); return H3DGS_ENOMEM; }
    if (hinfo.max_count <= (uint32_t)kTileSortCap) {
        if (side_color) H3_CUDA(cudaStreamWaitEvent(s, ss->join, 0));  // colours are needed by the record gather
        rc = launch_tile_binning(*a, out_radii, depths, records, D, hinfo.max_count, bin, bl, ranges, info, tile_count, s);
        if (rc) return rc;
    } else {
        // a tile list too long for the shared-memory sort: global stable radix sort (CUB), same order
        rc = launch_scan(tiles, offsets, P, geom + gl.scan_temp, gl.scan_temp_bytes, s, a->debug);
        if (rc) return rc;
        if (side_color) H3_CUDA(cudaStreamWaitEvent(s, ss->join, 0));
        rc = launch_binning(*a, out_radii, depths, offsets, records, D, bin, bl, ranges, s);
        if (rc) return rc;
    }
    rc = launch_render_forward(*a, ranges, (const Record*)(bin + bl.sorted_records), out_color, out_invdepth,
                               (float*)(img + il.final_T), (uint32_t*)(img + il.n_contrib),
                               (uint32_t*)(img + il.tile_max_contrib), s);
    return rc;
}

extern "C" int h3dgs_rasterize_backward(const h3dgs_raster_args* a, const int32_t* radii, const void* geom_state,
                                        const void* binning_state, const void* image_state, int64_t D,
                                        const float* dL_dcolor, const float* dL_dinvdepth, float* dL_dmeans3D,
                                        float* dL_dmeans2D, float* dL_dsh, float* dL_dcolors_precomp,
                                        float* dL_dopacities, float* dL_dscales, float* dL_drotations,
                                        float* dL_dcov3D, void* scratch, int phases, void* stream)
{
    int rc = check_args(a);
    if (rc) return rc;
    if (a->P == 0) return H3DGS_OK;                      // nothing rendered: all outputs have zero rows
    if (!geom_state || !binning_state || !image_state || ((phases & 1) && !dL_dcolor) || !scratch || !radii) {
        set_error("backward: missing saved state / scratch"); return H3DGS_EINVAL;
    }
    if ((phases & (2 | 4)) && (!dL_dmeans3D || !dL_dmeans2D || !dL_dopacities || (a->shs && !dL_dsh) ||
        (a->scales && (!dL_dscales || !dL_drotations)) || (a->cov3D_precomp && !dL_dcov3D))) {
        set_error("backward: missing gradient output"); return H3DGS_EINVAL;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const GeomLayout gl = geom_layout(a->P);
    const BinLayout bl = bin_layout(D);
    const ImgLayout il = img_layout(a->image_width, a->image_height);
    const uint8_t* geom = (const uint8_t*)geom_state;
    const uint8_t* bin = (const uint8_t*)binning_state;
    const uint8_t* img = (const uint8_t*)image_state;
    float* accum = (float*)scratch;
    h3dgs_raster_args b = *a;
    if (!dL_dinvdepth && (phases & 1)) b.do_depth = 0;
    bool zero_joined = true;
    SideStream* ss = nullptr;
    SideJoin side_guard;
    // scatter mode: gradients have num_source rows and must start from zero.  The fill (0.7 GB on config #3) runs on the side
    // stream beside the issue-bound replay; a caller that splits the phases asks for it with the replay (phases = 1 | 4) and
    // tells the chain-rule call that it has happened (phases = 2 | 8) -- otherwise it would sit between the two, exposed
    const bool fill_now = a->render_indices && (((phases & 2) && !(phases & 8)) || (phases & 4));
    if (fill_now) {
        rc = side_stream(&ss);
        if (rc) return rc;
        const size_t N = (size_t)a->num_source;
        H3_CUDA(cudaEventRecord(ss->fork, s));              // outputs may still be in use by earlier work on s
        H3_CUDA(cudaStreamWaitEvent(ss->s, ss->fork, 0));
        side_guard.arm(ss, s);
        H3_CUDA(cudaMemsetAsync(dL_dmeans3D, 0, N * 3 * sizeof(float), ss->s));
        H3_CUDA(cudaMemsetAsync(dL_dopacities, 0, N * sizeof(float), ss->s));
        H3_CUDA(cudaMemsetAsync(dL_dsh, 0, N * (size_t)a->sh_coeffs * 3 * sizeof(float), ss->s));
        H3_CUDA(cudaMemsetAsync(dL_dscales, 0, N * 3 * sizeof(float), ss->s));
        H3_CUDA(cudaMemsetAsync(dL_drotations, 0, N * 4 * sizeof(float), ss->s));
        H3_CUDA(cudaEventRecord(ss->join, ss->s));
        zero_joined = false;
    }
    if (phases & 1) H3_CUDA(cudaMemsetAsync(accum, 0, (size_t)a->P * kAccum * sizeof(float), s));
    if (D > 0 && (phases & 1)) {
        rc = launch_render_backward(b, (const uint32_t*)(img + il.ranges), (const Record*)(bin + bl.sorted_records),
                                    (const uint32_t*)(bin + bl.vals_sorted), (const float*)(img + il.final_T),
                                    (const uint32_t*)(img + il.n_contrib), (const uint32_t*)(img + il.tile_max_contrib),
                                    dL_dcolor, dL_dinvdepth, accum, s);
        if (rc) return rc;
    }
    if ((phases & 1) && a->peer_count > 1) {
        // peer mode: the partial rows of Gaussians other ranks own go into the owners' staging areas (posted stores over NVLink)
        rc = launch_peer_push(b, geom + gl.rank_mask, accum, s);
        if (rc) return rc;
    }
    if (!(phases & 2)) return H3DGS_OK;
    if (!zero_joined && !a->debug && !a->colors_precomp) {
        // scatter mode: every output is an atomic reduction, so the SH kernel (side stream, right
        // after its zero-fill) and the covariance kernel (main stream) run concurrently
        H3_CUDA(cudaEventRecord(ss->fork, s));                           // accum is complete at this point of s
        H3_CUDA(cudaStreamWaitEvent(ss->s, ss->fork, 0));
        rc = launch_sh_backward(b, radii, geom + gl.rank_mask, (const Record*)(geom + gl.records), accum, dL_dmeans3D, dL_dsh, ss->s);
        if (rc) return rc;
        H3_CUDA(cudaStreamWaitEvent(s, ss->join, 0));                    // zero-fill done before our own reductions
        H3_CUDA(cudaEventRecord(ss->join, ss->s));
        rc = launch_preprocess_backward(b, radii, geom + gl.rank_mask, (const Record*)(geom + gl.records), accum, dL_dmeans3D, dL_dmeans2D,
                                        dL_dsh, dL_dcolors_precomp, dL_dopacities, dL_dscales, dL_drotations, dL_dcov3D, s);
        if (rc) return rc;
        H3_CUDA(cudaStreamWaitEvent(s, ss->join, 0));
        return H3DGS_OK;
    }
    if (!zero_joined) H3_CUDA(cudaStreamWaitEvent(s, ss->join, 0));
    rc = launch_preprocess_backward(b, radii, geom + gl.rank_mask, (const Record*)(geom + gl.records), accum, dL_dmeans3D, dL_dmeans2D,
                                    dL_dsh, dL_dcolors_precomp, dL_dopacities, dL_dscales, dL_drotations, dL_dcov3D, s);
    if (rc) return rc;
    return launch_sh_backward(b, radii, geom + gl.rank_mask, (const Record*)(geom + gl.records), accum, dL_dmeans3D, dL_dsh, s);
}

extern "C" int h3dgs_state_layout(int32_t P, int32_t W, int32_t H, int64_t D, const void* geom_state,
                                  const void* binning_state, const void* image_state, h3dgs_state_view* out)
{
    if (!out) { set_error("out is NULL"); return H3DGS_EINVAL; }
    const GeomLayout gl = geom_layout(P);
    const BinLayout bl = bin_layout(D);
    const ImgLayout il = img_layout(W, H);
    const uint8_t* geom = (const uint8_t*)geom_state;
    const uint8_t* bin = (const uint8_t*)binning_state;
    const uint8_t* img = (const uint8_t*)image_state;
    memset(out, 0, sizeof(*out));
    if (geom) {
        out->depths = (const float*)(geom + gl.depths);
        out->tiles_touched = (const uint32_t*)(geom + gl.tiles_touched);
        out->point_offsets = (const uint32_t*)(geom + gl.offsets);
        out->records = (const float*)(geom + gl.records);
    }
    if (bin) {
        out->keys_sorted = (const uint64_t*)(bin + bl.keys_sorted);
        out->point_list = (const uint32_t*)(bin + bl.vals_sorted);
    }
    if (img) {
        out->ranges = (const uint32_t*)(img + il.ranges);
        out->final_T = (const float*)(img + il.final_T);
        out->n_contrib = (const uint32_t*)(img + il.n_contrib);
        out->scan_info = (const uint32_t*)(img + il.scan_info);
    }
    return H3DGS_OK;
}

#ifdef H3_SIMT_EMU
extern "C" long long* h3dgs_emu_stats(void) { return h3dgs::g_emu_stats; }     // emulation build only (tests/emul)
#endif
