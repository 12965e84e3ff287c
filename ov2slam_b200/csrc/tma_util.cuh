// TMA (cp.async.bulk.tensor) + mbarrier helpers shared by the image kernels (sm_90a).
// One elected thread issues a bulk tensor copy that lands a box of a tiled tensor map in shared memory and
// completes on an mbarrier; out-of-bounds parts of the box are zero-filled.  Measured rule (scripts/tma_probe.cu):
// for uint8 maps the box must START on a 16-byte boundary of the innermost dimension.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace tma {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "TMA_WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra TMA_WAIT_DONE;\n"
        "bra TMA_WAIT_LOOP;\n"
        "TMA_WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(phase) : "memory");
}
// The same wait with a suspend-time hint: the waiting threads sleep instead of spinning.  For grid FAST's one-copy cells
// the spin was 7.6 % of the kernel's instructions.
__device__ __forceinline__ void mbar_wait_suspend(uint64_t* bar, uint32_t phase) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "TMA_WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, 0x989680;\n"
        "@P1 bra TMA_WAIT_DONE;\n"
        "bra TMA_WAIT_LOOP;\n"
        "TMA_WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(phase) : "memory");
}
__device__ __forceinline__ void load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int x, int y, int z) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z)
                 : "memory");
}

typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static inline encode_tiled_fn encoder() {
    static encode_tiled_fn fn = []() -> encode_tiled_fn {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            return nullptr;
        return (encode_tiled_fn)p;
    }();
    return fn;
}

// 3-D uint8 map {W, H, frames} with row pitch / frame stride in bytes and box {bw, bh, 1}; false when the base
// address / strides do not meet the 16-byte rules or the driver lacks the entry point.
static inline bool make_u8_3d(CUtensorMap* map, const void* base, int w, int h, int frames, size_t pitch, size_t fstride, int bw, int bh) {
    encode_tiled_fn enc = encoder();
    if (!enc || ((uintptr_t)base % 16) != 0 || pitch % 16 != 0 || fstride % 16 != 0 || bw > 256 || bh > 256 || bw % 16 != 0) return false;
    cuuint64_t dims[3] = {(cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)frames};
    cuuint64_t strides[2] = {(cuuint64_t)pitch, (cuuint64_t)fstride};
    cuuint32_t box[3] = {(cuuint32_t)bw, (cuuint32_t)bh, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace tma
