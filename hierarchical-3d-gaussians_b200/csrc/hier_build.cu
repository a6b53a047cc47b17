// hier_build.cu -- the hierarchy creator (the GaussianHierarchyCreator stage of scripts/full_train.py:185-200): P trained
// Gaussians -> a binary LOD hierarchy of N = 2P - 1 nodes with one Gaussian row per node, in the arrays write_hierarchy
// takes.  The contract (topology, node order, merge rule, boxes) is include/h3dgs.h h3dgs_build_hierarchy; it is this
// project's own rule, not a restatement of upstream's.
//
// Step 1 here: check_bbox_kernel checks the input (EINVAL flag) and takes the bounding box of the positions
// (order-preserving uint keys, every word reduced with atomicMax from 0) -> read back; the quantisation scale in fp32
// on the host.  Steps 2-8 (Morton keys, radix tree, BFS order, leaves, the bottom-up merge) are the tree build of
// hier_tree.cuh, with the input Gaussians as the leaves.  An offline tool, so it synchronises twice.
// Deterministic: the only atomics are the order-independent max reductions of step 1.  This file is compiled with
// -fmad=false: the Morton quantisation is pinned fp32 arithmetic.
#include "hier_tree.cuh"

namespace h3dgs {
namespace {

__global__ void __launch_bounds__(256) check_bbox_kernel(int P, const float* __restrict__ xyz, const float* __restrict__ log_scales,
                                                         const float* __restrict__ rotations, const float* __restrict__ opacities,
                                                         uint32_t* __restrict__ hdr) {
    float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    uint32_t bad = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
        bool ok = true;
        for (int a = 0; a < 3; a++) {
            const float x = xyz[3 * (size_t)i + a];
            const float ls = log_scales[3 * (size_t)i + a];
            ok = ok && isfinite(x) && isfinite(ls) && ls <= kMaxLogScale;
            if (isfinite(x)) { lo[a] = fminf(lo[a], x); hi[a] = fmaxf(hi[a], x); }
        }
        for (int a = 0; a < 4; a++) ok = ok && isfinite(rotations[4 * (size_t)i + a]);
        const float o = opacities[i];
        if (!ok || !(o >= 0.f) || !isfinite(o)) bad = 1;
    }
    for (int a = 0; a < 3; a++) { lo[a] = warp_min(lo[a]); hi[a] = warp_max(hi[a]); }
    bad = __any_sync(kFull, bad) ? 1u : 0u;
    if ((threadIdx.x & 31) == 0) {
        for (int a = 0; a < 3; a++) { atomicMax(hdr + a, ~f2key(lo[a])); atomicMax(hdr + 3 + a, f2key(hi[a])); }
        if (bad) atomicMax(hdr + 6, 1u);
    }
}

struct In { const float *xyz, *log_scales, *rotations, *opacities, *shs; };

// the creator's leaves: a copy of input row s, its moments and its box
struct InputLeaves {
    In in;
    __device__ __forceinline__ void operator()(int p, int s, int32_t* nd, const Out& out, double* __restrict__ mom,
                                               double* __restrict__ shm) const {
        nd[0] = 0;
        out.source[p] = s;
        const float* x = in.xyz + 3 * (size_t)s;
        const float* ls = in.log_scales + 3 * (size_t)s;
        const float* r = in.rotations + 4 * (size_t)s;
        for (int a = 0; a < 3; a++) { out.xyz[3 * (size_t)p + a] = x[a]; out.log_scales[3 * (size_t)p + a] = ls[a]; }
        for (int a = 0; a < 4; a++) out.rotations[4 * (size_t)p + a] = r[a];
        const float o = in.opacities[s];
        out.opacities[p] = o;
        const float* sh = in.shs + kSH * (size_t)s;
        for (int c = 0; c < kSH; c++) { out.shs[kSH * (size_t)p + c] = sh[c]; shm[kSH * (size_t)p + c] = (double)sh[c]; }
        double C[6];
        double* m = mom + kMoments * (size_t)p;
        m[0] = gauss_moments(ls, r, o, C);
        for (int a = 0; a < 3; a++) m[1 + a] = (double)x[a];
        for (int e = 0; e < 6; e++) m[4 + e] = C[e];
        gauss_box(x, C, out.boxes + 8 * (size_t)p);
    }
};

}  // namespace
}  // namespace h3dgs

using namespace h3dgs;

extern "C" size_t h3dgs_build_hierarchy_scratch_bytes(int64_t P) {
    return (P >= 1 && P <= (int64_t(1) << 30)) ? build_layout(P).total : 0;
}

extern "C" int h3dgs_build_hierarchy(int32_t P, const float* xyz, const float* log_scales, const float* rotations,
                                     const float* opacities, const float* shs, float* out_xyz, float* out_shs,
                                     float* out_opacities, float* out_log_scales, float* out_rotations, int32_t* out_nodes,
                                     float* out_boxes, int32_t* out_source, void* scratch, void* stream) {
    if (P < 1 || P > (1 << 30) || !xyz || !log_scales || !rotations || !opacities || !shs || !out_xyz || !out_shs ||
        !out_opacities || !out_log_scales || !out_rotations || !out_nodes || !out_boxes || !out_source || !scratch) {
        set_error("build_hierarchy: bad arguments (P = %d)", P); return H3DGS_EINVAL;
    }
    if (reinterpret_cast<uintptr_t>(out_boxes) % 16 != 0) {
        set_error("build_hierarchy: out_boxes must be 16-byte aligned"); return H3DGS_EINVAL;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const BuildLayout l = build_layout(P);
    uint8_t* base = static_cast<uint8_t*>(scratch);
    int32_t* hdr = reinterpret_cast<int32_t*>(base + l.hdr);
    int32_t host[8];

    // 1. input check and bounding box -> quantisation
    H3_CUDA(cudaMemsetAsync(hdr, 0, kHdrWords * sizeof(int32_t), s));
    check_bbox_kernel<<<min(blocks(P, 256), 1024), 256, 0, s>>>(P, xyz, log_scales, rotations, opacities, reinterpret_cast<uint32_t*>(hdr));
    H3_LAUNCHED("hier_check_bbox", 0, s);
    H3_CUDA(cudaMemcpyAsync(host, hdr, 8 * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    H3_CUDA(cudaStreamSynchronize(s));
    if (host[6]) {
        set_error("build_hierarchy: a non-finite position, log-scale or rotation, a log-scale above 300, or a negative or "
                  "non-finite opacity");
        return H3DGS_EINVAL;
    }

    // 2.-8. the tree over the input Gaussians
    Out out{out_xyz, out_shs, out_opacities, out_log_scales, out_rotations, out_boxes, out_nodes, out_source};
    return build_tree(P, xyz, quant_of(host), l, base, InputLeaves{In{xyz, log_scales, rotations, opacities, shs}}, out, s,
                      "build_hierarchy");
}
