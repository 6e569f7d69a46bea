// wunet_wgmma.cuh — sm_90a device helpers shared by the tensor-core kernels (wunet_tc.cu, wunet_tc_f16.cu: inference forward;
// wunet_train_tc.cu: bf16 and tf32 training convolutions). Raw PTX; forms taken
// from the PTX ISA as shipped in CUDA 12.9.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include <type_traits>

namespace wunet {

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t pack_bf16(float a, float b)
{
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&h);
}

// wgmma (sm_90a): a warpgroup-wide asynchronous MMA whose operands come from shared memory through descriptors and whose
// accumulators are registers of the issuing warpgroup.
// Shared-memory descriptor of a K-major, 128B-swizzled operand (8-row groups 1024 B apart), as (lo, hi) words:
//   lo = (addr >> 4) | LBO(1) << 16,  hi = SBO(1024 >> 4) | SWIZZLE_128B(1) << 30, base_offset 0.
// The swizzle acts on absolute shared-memory address bits, so a start address advanced by whole 128-byte rows (the tap
// shift of the implicit GEMM) or by 32 bytes (the next K16 step) addresses the TMA-written tile correctly.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// D[64 x N] += A[64 x 16] * B[N x 16]^T, bf16 operands, fp32 accumulators, N = 16, 32, ..., 128. The B descriptor addresses
// N K-major rows of 128 B (8-row groups 1024 B apart). The f32 fragment is that of m64n16k16 per 16-column block, concatenated:
// column block nb is d[8 nb .. 8 nb + 7].
// imm-trans-a / imm-trans-b (TA, TB) = 1: that operand is MN-major ("transposed"): each 128-byte row of the tile holds 64
// consecutive M (or N) elements of ONE K index, 8-row K groups SBO apart (the [position][channel] tiles of the weight gradient,
// whose K axis is the position). 0: K-major, as in the inference kernels.
template <int N, int TA, int TB> struct WgmmaBf16;
template <int TA, int TB> struct WgmmaBf16<16, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[8], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%8, %10};\n\tmov.b64 db, {%9, %10};\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7"
            "}, da, db, p, 1, 1, %11, %12;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};
template <int TA, int TB> struct WgmmaBf16<32, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[16], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%16, %18};\n\tmov.b64 db, {%17, %18};\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
            "}, da, db, p, 1, 1, %19, %20;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};
template <int TA, int TB> struct WgmmaBf16<48, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[24], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%24, %26};\n\tmov.b64 db, {%25, %26};\n\t"
            "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23"
            "}, da, db, p, 1, 1, %27, %28;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};
template <int TA, int TB> struct WgmmaBf16<64, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[32], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%32, %34};\n\tmov.b64 db, {%33, %34};\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
            "}, da, db, p, 1, 1, %35, %36;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};
template <int TA, int TB> struct WgmmaBf16<80, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[40], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%40, %42};\n\tmov.b64 db, {%41, %42};\n\t"
            "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39"
            "}, da, db, p, 1, 1, %43, %44;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};
template <int TA, int TB> struct WgmmaBf16<96, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[48], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%48, %50};\n\tmov.b64 db, {%49, %50};\n\t"
            "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
            "}, da, db, p, 1, 1, %51, %52;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};
template <int TA, int TB> struct WgmmaBf16<112, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[56], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%56, %58};\n\tmov.b64 db, {%57, %58};\n\t"
            "wgmma.mma_async.sync.aligned.m64n112k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
            "%48, %49, %50, %51, %52, %53, %54, %55"
            "}, da, db, p, 1, 1, %59, %60;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};
template <int TA, int TB> struct WgmmaBf16<128, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[64], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%64, %66};\n\tmov.b64 db, {%65, %66};\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
            "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
            "}, da, db, p, 1, 1, %67, %68;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};

// The same forms with fp16 operands (wgmma ...f32.f16.f16: same layouts, descriptors and rate as bf16)
template <int N, int TA, int TB> struct WgmmaF16;
template <int TA, int TB> struct WgmmaF16<16, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[8], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%8, %10};\n\tmov.b64 db, {%9, %10};\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7"
            "}, da, db, p, 1, 1, %11, %12;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};
template <int TA, int TB> struct WgmmaF16<32, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[16], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%16, %18};\n\tmov.b64 db, {%17, %18};\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
            "}, da, db, p, 1, 1, %19, %20;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};
template <int TA, int TB> struct WgmmaF16<48, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[24], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%24, %26};\n\tmov.b64 db, {%25, %26};\n\t"
            "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23"
            "}, da, db, p, 1, 1, %27, %28;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};
template <int TA, int TB> struct WgmmaF16<64, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[32], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%32, %34};\n\tmov.b64 db, {%33, %34};\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
            "}, da, db, p, 1, 1, %35, %36;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};
template <int TA, int TB> struct WgmmaF16<80, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[40], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%40, %42};\n\tmov.b64 db, {%41, %42};\n\t"
            "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39"
            "}, da, db, p, 1, 1, %43, %44;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};
template <int TA, int TB> struct WgmmaF16<96, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[48], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%48, %50};\n\tmov.b64 db, {%49, %50};\n\t"
            "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
            "}, da, db, p, 1, 1, %51, %52;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};
template <int TA, int TB> struct WgmmaF16<112, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[56], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%56, %58};\n\tmov.b64 db, {%57, %58};\n\t"
            "wgmma.mma_async.sync.aligned.m64n112k16.f32.f16.f16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
            "%48, %49, %50, %51, %52, %53, %54, %55"
            "}, da, db, p, 1, 1, %59, %60;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};
template <int TA, int TB> struct WgmmaF16<128, TA, TB> {
    static __device__ __forceinline__ void mma(float (&d)[64], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%64, %66};\n\tmov.b64 db, {%65, %66};\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
            "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
            "}, da, db, p, 1, 1, %67, %68;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "r"(a_lo), "r"(b_lo), "r"(hi), "n"(TA), "n"(TB)
            : "memory");
    }
};

// E: the operand element type, __nv_bfloat16 or __half
template <int N, int TA = 0, int TB = 0, typename E = __nv_bfloat16>
__device__ __forceinline__ void wgmma_m64nNk16(float (&d)[N / 2], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
{
    if constexpr (std::is_same<E, __half>::value) WgmmaF16<N, TA, TB>::mma(d, a_lo, b_lo, hi);
    else WgmmaBf16<N, TA, TB>::mma(d, a_lo, b_lo, hi);
}

// D[64 x N] += A[64 x 8] * B[N x 8]^T, tf32 operands (fp32 words; the MMA reads the top 19 bits), fp32 accumulators,
// N = 16 .. 64. Both operands K-major: the PTX has no transpose immediates for 32-bit operand types. A 128-byte swizzled row
// holds 32 fp32 K elements, so one K8 step is 32 bytes, the same descriptor advance as a bf16 K16 step. Same f32 fragment as
// wgmma_m64nNk16.
template <int N> struct WgmmaTf32;
template <> struct WgmmaTf32<16> {
    static __device__ __forceinline__ void mma(float (&d)[8], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%8, %10};\n\tmov.b64 db, {%9, %10};\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {"
            "%0, %1, %2, %3, %4, %5, %6, %7"
            "}, da, db, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "r"(a_lo), "r"(b_lo), "r"(hi)
            : "memory");
    }
};
template <> struct WgmmaTf32<32> {
    static __device__ __forceinline__ void mma(float (&d)[16], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%16, %18};\n\tmov.b64 db, {%17, %18};\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
            "}, da, db, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "r"(a_lo), "r"(b_lo), "r"(hi)
            : "memory");
    }
};
template <> struct WgmmaTf32<48> {
    static __device__ __forceinline__ void mma(float (&d)[24], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%24, %26};\n\tmov.b64 db, {%25, %26};\n\t"
            "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23"
            "}, da, db, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "r"(a_lo), "r"(b_lo), "r"(hi)
            : "memory");
    }
};
template <> struct WgmmaTf32<64> {
    static __device__ __forceinline__ void mma(float (&d)[32], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\tsetp.ne.b32 p, 1, 0;\n\tmov.b64 da, {%32, %34};\n\tmov.b64 db, {%33, %34};\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
            "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
            "}, da, db, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "r"(a_lo), "r"(b_lo), "r"(hi)
            : "memory");
    }
};

template <int N>
__device__ __forceinline__ void wgmma_m64nNk8_tf32(float (&d)[N / 2], uint32_t a_lo, uint32_t b_lo, uint32_t hi)
{
    WgmmaTf32<N>::mma(d, a_lo, b_lo, hi);
}

}  // namespace

}  // namespace wunet
