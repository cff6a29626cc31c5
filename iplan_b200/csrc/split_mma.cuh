// Split-f16 tensor-core building blocks shared by lin64_mma.cuh (learner.cu) and behavior_fc.cu: an fp32 pair split into
// f16 hi + lo halves, and one mma.sync.m16n8k16 (f16 in, fp32 accumulate).  A product is hi*hi + lo*hi + hi*lo, which
// keeps ~2^-22 relative accuracy.  Included INSIDE namespace iplan, after <cuda_fp16.h>.
#pragma once

__device__ __forceinline__ void l64_split(float x, float y, uint32_t& hi, uint32_t& lo) {
    const __half2 h = __floats2half2_rn(x, y);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(x - hf.x, y - hf.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ void l64_mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
