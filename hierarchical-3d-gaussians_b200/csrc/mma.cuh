// mma.cuh -- the TF32 tensor-core and cp.async wrappers of the LPIPS convolutions (lpips.cu), for sm_90a.
// Kept in one header, as tma.cuh is, so that the CPU emulation build of the sources can replace it.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace h3dgs {

// fp32 -> TF32 (10 mantissa bits), round to nearest with ties away from zero; the result is an fp32 bit pattern
__device__ __forceinline__ uint32_t to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}

// d += A (16x8, row) * B (8x8, col), TF32 operands, fp32 accumulate.  Fragments per the PTX ISA (g = lane / 4,
// t = lane % 4): a = {A[g][t], A[g+8][t], A[g][t+4], A[g+8][t+4]}, b = {B[t][g], B[t+4][g]},
// d = {D[g][2t], D[g][2t+1], D[g+8][2t], D[g+8][2t+1]}
__device__ __forceinline__ void mma_tf32_16x8x8(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// 16-byte global -> shared copy; zero-fills the destination when !valid (src is not read then)
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)),
                 "l"(gmem_src), "r"(valid ? 16 : 0)
                 : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

}  // namespace h3dgs
