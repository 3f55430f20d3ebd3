// Quantised attention on sm_90a warpgroup MMAs: qattention_kernel's two-pass algorithm (integer scores, exp2-domain
// softmax with the calibrated step, P codes as hi/lo byte planes, integer PV, row sums from an all-ones V^T row) with
//   * S = Q K^T as wgmma m64n64 (k32 on 8-bit codes, or k16 f16 x f16 -> f32 on fp16 centred codes - qk_f16 - whose
//     integer scores are exact), Q fragments in registers, the K tile in shared memory;
//   * O += P V as wgmma m64nNV k32 (u8 P codes in registers, V^T tile in shared memory), NV = d + 8 rounded up to a
//     wgmma width (the extra rows: the all-ones row, then zeros);
//   * K, V^T and the zq*rowsum(k) slice staged by TMA / bulk copies through an ATW_STAGES-deep mbarrier ring (one load
//     per (pass, key tile); pass 0 needs no V^T).  The consumer warp that releases a stage last refills it.
// Two consumer warpgroups, 64 query rows each, running the loads L = 0 .. 2*ntiles-1 in order, one loop per pass;
// for d <= 40 two CTAs share an SM (MINB = 2, <= 128 registers).  The softmax works on fp32 scores: the fp16 operands'
// accumulators as they are (exact integers), and the 8-bit codes' int32 sums converted without I2F.  The per-warp
// accumulator fragment of wgmma m64nN is the m16n8 fragment of mma.sync repeated over N / 8 column tiles, and the register A operand has the m16n8k32 layout, so the softmax code
// below is qattention_kernel's, operating on the same registers.  V^T keeps its 16-key byte permutation
// (att_vt_perm): with it, the P fragments built from the S accumulators are the A operand without shuffles.
#pragma once
#include "attention.cuh"
#include "ptx.cuh"

namespace qd {

__device__ __forceinline__ void wgmma_ra_s8s8_n64(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ra_u8u8_n64(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k32.s32.u8.u8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ra_f16_n64(float* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ra_u8u8_n24(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %17, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n24k32.s32.u8.u8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11}, {%12, %13, %14, %15}, %16, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ra_u8s8_n24(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %17, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n24k32.s32.u8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11}, {%12, %13, %14, %15}, %16, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ra_u8u8_n32(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.u8.u8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ra_u8s8_n32(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.u8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ra_u8u8_n48(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %29, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k32.s32.u8.u8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, {%24, %25, %26, %27}, %28, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ra_u8s8_n48(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %29, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k32.s32.u8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, {%24, %25, %26, %27}, %28, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ra_u8s8_n64(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k32.s32.u8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ra_u8u8_n80(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %45, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n80k32.s32.u8.u8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, {%40, %41, %42, %43}, %44, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ra_u8s8_n80(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %45, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n80k32.s32.u8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, {%40, %41, %42, %43}, %44, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ra_u8u8_n96(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %53, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k32.s32.u8.u8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, {%48, %49, %50, %51}, %52, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ra_u8s8_n96(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %53, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k32.s32.u8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, {%48, %49, %50, %51}, %52, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ra_u8u8_n112(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %61, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n112k32.s32.u8.u8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55}, {%56, %57, %58, %59}, %60, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_ra_u8s8_n112(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %61, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n112k32.s32.u8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55}, {%56, %57, %58, %59}, %60, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

constexpr int ATW_STAGES = 4;
constexpr int ATW_THREADS = ATT_WARPS * 32;       // two warpgroups
// PV width: d + 8 (the all-ones row sits at row d) rounded up to a wgmma N for 8-bit operands
__host__ __device__ constexpr int atw_nv(int DV) {
  return DV + 8 <= 24 ? 24 : DV + 8 <= 32 ? 32 : DV + 8 <= 48 ? 48 : DV + 8 <= 64 ? 64 : DV + 8 <= 80 ? 80 : DV + 8 <= 96 ? 96 : 112;
}
struct AtwSmem {
  int k_bytes, v_bytes, z_off, bar_off, total;
};
// per stage: K tile 64 x P bytes (P-byte swizzle), V^T tile NV x 64 bytes (64-byte swizzle), 256 bytes of row sums
__host__ __device__ inline AtwSmem atw_smem(int P, int NV) {
  AtwSmem l;
  l.k_bytes = (ATT_BN * P + 1023) / 1024 * 1024;
  l.v_bytes = (NV * ATT_BN + 1023) / 1024 * 1024;
  l.z_off = ATW_STAGES * (l.k_bytes + l.v_bytes);
  l.bar_off = l.z_off + ATW_STAGES * ATT_BN * 4;
  l.total = l.bar_off + ATW_STAGES * 8 + ATW_STAGES * 4 + 1024;   // full barriers, release counters, alignment slack
  return l;
}
// sm_90 shared-memory descriptor for a K-major tile of `row_bytes`-byte rows stored with the matching TMA swizzle
__device__ __forceinline__ uint64_t atw_desc(uint32_t addr, int row_bytes) {
  const uint64_t layout = row_bytes == 128 ? 1 : row_bytes == 64 ? 2 : 3;
  uint64_t d = (uint64_t)((addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)((8 * row_bytes) >> 4) << 32;
  d |= layout << 62;
  return d;
}

template <int N, bool VS>
__device__ __forceinline__ void atw_pv(uint32_t* d, const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  if constexpr (VS) {
    if constexpr (N == 24) wgmma_ra_u8s8_n24(d, a, db, scale_d);
    else if constexpr (N == 32) wgmma_ra_u8s8_n32(d, a, db, scale_d);
    else if constexpr (N == 48) wgmma_ra_u8s8_n48(d, a, db, scale_d);
    else if constexpr (N == 64) wgmma_ra_u8s8_n64(d, a, db, scale_d);
    else if constexpr (N == 80) wgmma_ra_u8s8_n80(d, a, db, scale_d);
    else if constexpr (N == 96) wgmma_ra_u8s8_n96(d, a, db, scale_d);
    else wgmma_ra_u8s8_n112(d, a, db, scale_d);
  } else {
    if constexpr (N == 24) wgmma_ra_u8u8_n24(d, a, db, scale_d);
    else if constexpr (N == 32) wgmma_ra_u8u8_n32(d, a, db, scale_d);
    else if constexpr (N == 48) wgmma_ra_u8u8_n48(d, a, db, scale_d);
    else if constexpr (N == 64) wgmma_ra_u8u8_n64(d, a, db, scale_d);
    else if constexpr (N == 80) wgmma_ra_u8u8_n80(d, a, db, scale_d);
    else if constexpr (N == 96) wgmma_ra_u8u8_n96(d, a, db, scale_d);
    else wgmma_ra_u8u8_n112(d, a, db, scale_d);
  }
}

// DQ: bytes of the padded QK^T reduction (multiple of 32, <= P); DV: head dim d; P: per-head pitch of Q / K in bytes
// (32 / 64 / 128, also the K tile's swizzle span).
template <int DQ, int DV, bool QK_SIGNED, bool V_SIGNED, bool SM16, bool F16, int MINB>
__global__ void __launch_bounds__(ATW_THREADS, MINB)
qattention_wg_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                     const qd_attention_desc p, int P) {
  constexpr int NV = atw_nv(DV);
  constexpr int NKC = DQ / 32;      // 32-byte k-steps of QK^T
  constexpr int NDT = DV / 8 + 1;   // n8 tiles of the output + the row-sum tile
  constexpr int RB = F16 ? 2 * DV : DV;   // bytes of one head's Q / K row
  static_assert(!F16 || DV <= 64, "fp16 Q / K operands: d <= 64 keeps |S| below 2^22");
  static_assert(DV <= 96, "8-bit codes: the raw scores must stay below 2^23 (unsigned) / 2^22 (signed)");
  // Accumulator of S = Q K^T: the exact fp32 score on fp16 operands; the raw int32 sum on 8-bit codes, made fp32 without
  // I2F (which shares the quarter-rate pipe with ex2): the bits of MB + raw are the float MB + raw, exact for unsigned
  // codes (MB = 2^23, 0 <= raw <= 255^2 * 96 < 2^23) and signed ones (MB = 1.5 * 2^23, |raw| <= 128^2 * 96 < 2^22).
  // zq * rowsum(k) goes through the same add (attention_wg_eligible keeps it in that range), and the difference of two
  // floats of [2^22, 2^24) with unit spacing is the exact score.
  using SV = std::conditional_t<F16, float, uint32_t>;
  constexpr uint32_t MB = QK_SIGNED ? 0x4B400000u : 0x4B000000u;
  extern __shared__ uint8_t atw_raw[];
  uint8_t* smem = atw_raw + (((smem_u32(atw_raw) + 1023u) & ~1023u) - smem_u32(atw_raw));
  const AtwSmem lay = atw_smem(P, NV);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + lay.bar_off);
  int* released = reinterpret_cast<int*>(full + ATW_STAGES);   // per stage: consumer-warp releases so far

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int bh = blockIdx.y;
  const int b = bh / p.heads, h = bh - b * p.heads;
  const int row0 = blockIdx.x * ATT_BM + warp * 16;
  const int ntiles = (p.Tk + ATT_BN - 1) / ATT_BN;
  const int nloads = 2 * ntiles;      // (pass, tile) in order
  const bool has_zq = !F16 && p.zq != 0;
  const int* zrk_g = reinterpret_cast<const int*>(p.ws) + (long long)bh * (long long)att_ws_stride(p.Tk);

  // ---- V^T rows d .. NV-1 of every stage: the all-ones row, then zeros (TMA writes rows 0 .. d-1 only).  A row of
  // equal bytes is the same under any swizzle.
  for (int i = threadIdx.x; i < ATW_STAGES * (NV - DV) * ATT_BN; i += ATW_THREADS) {
    const int s = i / ((NV - DV) * ATT_BN), r = (i / ATT_BN) % (NV - DV) + DV, c = i % ATT_BN;
    smem[ATW_STAGES * lay.k_bytes + s * lay.v_bytes + r * ATT_BN + c] = r == DV ? 1 : 0;
  }
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    for (int s = 0; s < ATW_STAGES; ++s) {
      mbar_init(&full[s], 1);
      released[s] = 0;
    }
    fence_mbar_init();
  }
  fence_proxy_async();     // the generic writes above -> visible to the tensor cores
  __syncthreads();

  auto issue = [&](int L) {           // one thread: load number L into stage L % ATW_STAGES
    const int s = L % ATW_STAGES, pass = L / ntiles, tile = L - pass * ntiles;
    const int j0 = tile * ATT_BN;
    const uint32_t bytes = (uint32_t)(ATT_BN * P) + (pass ? (uint32_t)(ATT_BN * DV) : 0u) + (has_zq ? ATT_BN * 4u : 0u);
    mbar_arrive_expect_tx(&full[s], bytes);
    tma_load_2d(smem + s * lay.k_bytes, &tmK, &full[s], h * P, b * p.Tk + j0);
    if (pass) tma_load_2d(smem + ATW_STAGES * lay.k_bytes + s * lay.v_bytes, &tmV, &full[s], j0, bh * DV);
    if (has_zq) bulk_load_1d(smem + lay.z_off + s * ATT_BN * 4, zrk_g + j0, ATT_BN * 4, &full[s]);
  };
  if (threadIdx.x == 0)
    for (int L = 0; L < ATW_STAGES && L < nloads; ++L) issue(L);

  // ---- Q fragments (rows g, g+8 of this warp's 16-row slab) in the m16n8k32 / m16n8k16 A layout: bytes 4t.. and
  // 16+4t.. of every 32-byte k-chunk; zero beyond the head's row (the K tile may hold the next head's bytes there).
  // At d = 48 (8-bit and fp16 operands alike) ptxas of CUDA 12.9 hands the registers of fragments that stay live across
  // the key loop to the P fragments of the first PV wgmma, so every later S = Q K^T read P codes as Q: the kernel then
  // loads the fragments again for every key tile (L1 hits), which keeps them out of the loop's live set.
  constexpr bool QRELOAD = DV == 48;
  uint32_t qf[NKC][4];
  const uint8_t* qbase = reinterpret_cast<const uint8_t*>(p.q) + (long long)b * p.Tq * p.ld_q + p.q_off + h * p.head_stride_q;
  const uint8_t* q0 = qbase + (long long)min(row0 + g, p.Tq - 1) * p.ld_q;
  const uint8_t* q1 = qbase + (long long)min(row0 + g + 8, p.Tq - 1) * p.ld_q;
  auto load_q = [&]() {
#pragma unroll
    for (int kc = 0; kc < NKC; ++kc) {
      const int c0 = kc * 32 + 4 * t, c1 = c0 + 16;
      qf[kc][0] = c0 < RB ? *reinterpret_cast<const uint32_t*>(q0 + c0) : 0u;
      qf[kc][1] = c0 < RB ? *reinterpret_cast<const uint32_t*>(q1 + c0) : 0u;
      qf[kc][2] = c1 < RB ? *reinterpret_cast<const uint32_t*>(q0 + c1) : 0u;
      qf[kc][3] = c1 < RB ? *reinterpret_cast<const uint32_t*>(q1 + c1) : 0u;
    }
  };
  if constexpr (!QRELOAD) load_q();
  const float c = p.sim_scale * 1.4426950408889634f;
  const bool ragged = (p.Tk % ATT_BN) != 0;
  float mi0 = -INFINITY, mi1 = -INFINITY;
  float l0 = 0.f, l1 = 0.f;

  // S(L) = Q K^T for this warpgroup, 64 x 64, once load L has landed; this warp's 16 rows land in s[nt][0..3]
  // (m16n8 fragments)
  auto issue_s = [&](SV (&s)[8][4], int L) {
    const int st = L % ATW_STAGES;
    if constexpr (QRELOAD) load_q();
    mbar_wait(&full[st], (uint32_t)(L / ATW_STAGES) & 1u);
    const uint64_t dK = atw_desc(smem_u32(smem + st * lay.k_bytes), P);
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < NKC; ++kc) {
      if constexpr (F16) wgmma_ra_f16_n64(&s[0][0], qf[kc], dK + (uint64_t)(2 * kc), kc ? 1u : 0u);
      else if constexpr (QK_SIGNED) wgmma_ra_s8s8_n64(&s[0][0], qf[kc], dK + (uint64_t)(2 * kc), kc ? 1u : 0u);
      else wgmma_ra_u8u8_n64(&s[0][0], qf[kc], dK + (uint64_t)(2 * kc), kc ? 1u : 0u);
    }
    wgmma_commit();
  };
  // After the wait that retired S(L): the fp32 scores, keys beyond Tk at -inf (no share of the row maximum, the row sum
  // or the P codes, whatever the codes are).
  auto scores = [&](SV (&s)[8][4], float (&f)[8][4], int L) {
    wgmma_fence_regs(reinterpret_cast<SV (&)[32]>(s));
    const int tile = L % ntiles, st = L % ATW_STAGES;
    if constexpr (F16) {
#pragma unroll
      for (int i = 0; i < 32; ++i) f[i >> 2][i & 3] = s[i >> 2][i & 3];
    } else {
      const uint32_t* sZrk = reinterpret_cast<const uint32_t*>(smem + lay.z_off + st * ATT_BN * 4);
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        float z0 = __uint_as_float(MB), z1 = z0;
        if (has_zq) {
          const uint2 z = *reinterpret_cast<const uint2*>(sZrk + 8 * nt + 2 * t);
          z0 = __uint_as_float(z.x + MB);
          z1 = __uint_as_float(z.y + MB);
        }
        f[nt][0] = __uint_as_float(s[nt][0] + MB) - z0; f[nt][1] = __uint_as_float(s[nt][1] + MB) - z1;
        f[nt][2] = __uint_as_float(s[nt][2] + MB) - z0; f[nt][3] = __uint_as_float(s[nt][3] + MB) - z1;
      }
    }
    if (ragged && tile == ntiles - 1) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int j = tile * ATT_BN + 8 * nt + 2 * t;
        if (j >= p.Tk) { f[nt][0] = -INFINITY; f[nt][2] = -INFINITY; }
        if (j + 1 >= p.Tk) { f[nt][1] = -INFINITY; f[nt][3] = -INFINITY; }
      }
    }
  };

  // Release load R; the last of the 8 warps to do so refills the stage, so no warp waits for another.
  auto release = [&](int R) {
    __syncwarp();
    if (lane == 0) {
      const int s = R % ATW_STAGES;
      __threadfence_block();
      const int n = atomicAdd(&released[s], 1);
      if (n == ATT_WARPS * (R / ATW_STAGES + 1) - 1 && R + ATW_STAGES < nloads) {
        __threadfence_block();
        issue(R + ATW_STAGES);
      }
    }
  };

  // One S register set per warp and every wgmma retired before the next is issued: for d <= 40 that fits 128 registers
  // (two CTAs per SM, whose warps hide each other's latencies) without spills or wgmma serialisation.  Overlapping
  // S(L+1) with the softmax of S(L) needs a second S set (pass 0) or P and S live together (pass 1); ptxas of CUDA 12.9
  // then spills or serialises the wgmmas at that register cap (DESIGN §6).
  // ---- pass 0: row maxima and sums.  The O accumulators are not live yet.  Load L (K and the zq * rowsum(k) slice) is
  // released as soon as its scores are read, before the exp2 work.
  for (int L = 0; L < ntiles; ++L) {
    SV sacc[8][4];
    issue_s(sacc, L);
    wgmma_wait<0>();
    float f[8][4];
    scores(sacc, f, L);
    release(L);
    float tm0 = f[0][0], tm1 = f[0][2];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      tm0 = fmaxf(tm0, fmaxf(f[nt][0], f[nt][1]));
      tm1 = fmaxf(tm1, fmaxf(f[nt][2], f[nt][3]));
    }
    tm0 = fmaxf(tm0, __shfl_xor_sync(0xffffffffu, tm0, 1));
    tm0 = fmaxf(tm0, __shfl_xor_sync(0xffffffffu, tm0, 2));
    tm1 = fmaxf(tm1, __shfl_xor_sync(0xffffffffu, tm1, 1));
    tm1 = fmaxf(tm1, __shfl_xor_sync(0xffffffffu, tm1, 2));
    if (tm0 > mi0) { l0 *= (mi0 == -INFINITY) ? 0.f : ex2_approx((mi0 - tm0) * c); mi0 = tm0; }
    if (tm1 > mi1) { l1 *= (mi1 == -INFINITY) ? 0.f : ex2_approx((mi1 - tm1) * c); mi1 = tm1; }
    const float b0 = -mi0 * c, b1 = -mi1 * c;
    float a0 = 0.f, a1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      a0 += ex2_approx(fmaf(f[nt][0], c, b0)) + ex2_approx(fmaf(f[nt][1], c, b0));
      a1 += ex2_approx(fmaf(f[nt][2], c, b1)) + ex2_approx(fmaf(f[nt][3], c, b1));
    }
    l0 += a0;
    l1 += a1;
  }

  // ---- pass 1: P codes packed straight into A fragments (byte planes), then O += P V on the warpgroup
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float off0 = -mi0 * c + log2f(1.0f / (l0 * p.delta_w));
  const float off1 = -mi1 * c + log2f(1.0f / (l1 * p.delta_w));
  const float pmax = (float)p.p_qmax;
  const QuantK oqk = make_quantk(p.oq);
  // code words of S(L): 1.5 * 2^23 + round(min(p, qmax)), the code in the low 16 bits
  auto codes = [&](SV (&s)[8][4], uint32_t (&cw)[8][4], int L) {
    float f[8][4];
    scores(s, f, L);
#pragma unroll
    for (int i = 0; i < 32; ++i)
      cw[i >> 2][i & 3] = __float_as_uint(fminf(ex2_approx(fmaf(f[i >> 2][i & 3], c, (i & 2) ? off1 : off0)), pmax) + 12582912.0f);
  };
  // P codes as A fragments (byte planes) of m64nNk32: k-chunk kc holds key tiles 4kc .. 4kc+3
  uint32_t plo[2][4], phi[2][4];
  auto pack = [&](const uint32_t (&cw)[8][4]) {
#pragma unroll
    for (int kc = 0; kc < 2; ++kc) {
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int ntA = 4 * kc + 2 * half, ntB = ntA + 1;
        const uint32_t cd[8] = {cw[ntA][0], cw[ntA][1], cw[ntB][0], cw[ntB][1], cw[ntA][2], cw[ntA][3], cw[ntB][2], cw[ntB][3]};
        plo[kc][2 * half] = __byte_perm(__byte_perm(cd[0], cd[1], 0x0040), __byte_perm(cd[2], cd[3], 0x0040), 0x5410);
        plo[kc][2 * half + 1] = __byte_perm(__byte_perm(cd[4], cd[5], 0x0040), __byte_perm(cd[6], cd[7], 0x0040), 0x5410);
        if constexpr (SM16) {
          phi[kc][2 * half] = __byte_perm(__byte_perm(cd[0], cd[1], 0x0051), __byte_perm(cd[2], cd[3], 0x0051), 0x5410);
          phi[kc][2 * half + 1] = __byte_perm(__byte_perm(cd[4], cd[5], 0x0051), __byte_perm(cd[6], cd[7], 0x0051), 0x5410);
        }
      }
    }
  };
  uint32_t olo[NV / 2], ohi[SM16 ? NV / 2 : 1];     // zeroed by the first PV (scale_d = 0)
  for (int L = ntiles; L < nloads; ++L) {
    SV sacc[8][4];
    uint32_t cw[8][4];
    issue_s(sacc, L);
    wgmma_wait<0>();
    codes(sacc, cw, L);
    pack(cw);
    const uint64_t dV = atw_desc(smem_u32(smem + ATW_STAGES * lay.k_bytes + (L % ATW_STAGES) * lay.v_bytes), ATT_BN);
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < 2; ++kc) {
      const uint32_t acc = (kc || L > ntiles) ? 1u : 0u;
      atw_pv<NV, V_SIGNED>(olo, plo[kc], dV + (uint64_t)(2 * kc), acc);
      if constexpr (SM16) atw_pv<NV, V_SIGNED>(ohi, phi[kc], dV + (uint64_t)(2 * kc), acc);
    }
    wgmma_commit();
    wgmma_wait<0>();
    release(L);
  }
#pragma unroll
  for (int i = 0; i < NV / 2; ++i) asm volatile("" : "+r"(olo[i])::"memory");
#pragma unroll
  for (int i = 0; i < (SM16 ? NV / 2 : 1); ++i) asm volatile("" : "+r"(ohi[i])::"memory");

  // ---- write O: (256*hi + lo - zv * rowsum) * out_scale.  Row sums: column d (tile NDT - 1, t == 0).
  float rs0 = (float)(int)olo[4 * (NDT - 1)], rs1 = (float)(int)olo[4 * (NDT - 1) + 2];
  if constexpr (SM16) { rs0 += 256.0f * (float)(int)ohi[4 * (NDT - 1)]; rs1 += 256.0f * (float)(int)ohi[4 * (NDT - 1) + 2]; }
  rs0 = __shfl_sync(0xffffffffu, rs0, lane & ~3);
  rs1 = __shfl_sync(0xffffffffu, rs1, lane & ~3);
  const int r0 = row0 + g, r1 = row0 + g + 8;
  const float z0 = (float)p.zv * rs0, z1 = (float)p.zv * rs1;
#pragma unroll
  for (int nd = 0; nd < NDT - 1; ++nd) {
    const int col = h * DV + 8 * nd + 2 * t;
    float v0 = (float)(int)olo[4 * nd], v1 = (float)(int)olo[4 * nd + 1], v2 = (float)(int)olo[4 * nd + 2], v3 = (float)(int)olo[4 * nd + 3];
    if constexpr (SM16) {
      v0 += 256.0f * (float)(int)ohi[4 * nd]; v1 += 256.0f * (float)(int)ohi[4 * nd + 1];
      v2 += 256.0f * (float)(int)ohi[4 * nd + 2]; v3 += 256.0f * (float)(int)ohi[4 * nd + 3];
    }
    const float y0 = (v0 - z0) * p.out_scale, y1 = (v1 - z0) * p.out_scale;
    const float y2 = (v2 - z1) * p.out_scale, y3 = (v3 - z1) * p.out_scale;
    if (p.out) {
      if (r0 < p.Tq) *reinterpret_cast<float2*>(p.out + ((long long)b * p.Tq + r0) * p.ld_out + col) = make_float2(y0, y1);
      if (r1 < p.Tq) *reinterpret_cast<float2*>(p.out + ((long long)b * p.Tq + r1) * p.ld_out + col) = make_float2(y2, y3);
    }
    if (p.out_q) {
      uint8_t* oq = reinterpret_cast<uint8_t*>(p.out_q);
      if (r0 < p.Tq)
        *reinterpret_cast<uint16_t*>(oq + ((long long)b * p.Tq + r0) * p.ld_out_q + col) =
            (uint16_t)(quant_code(y0, oqk) | (quant_code(y1, oqk) << 8));
      if (r1 < p.Tq)
        *reinterpret_cast<uint16_t*>(oq + ((long long)b * p.Tq + r1) * p.ld_out_q + col) =
            (uint16_t)(quant_code(y2, oqk) | (quant_code(y3, oqk) << 8));
    }
  }
}

}  // namespace qd
