// Shared device-side pieces of the wgmma GEMM kernel (gemm_tc.cu): PTX wrappers (mbarrier, TMA, wgmma), shared-memory
// descriptors, the hi/lo split helpers with their scale-miss report (also used by the normaliser kernels, rms_kernels.cu, which
// write operand planes too) and the epilogue parameter block.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include "common.cuh"
#include "kernels.h"

namespace ase {

constexpr int TC_KPAD = 32;               // fp32 words: K padding of workspace planes (128 bytes, the prep kernels' granularity)
constexpr int TC_THREADS = 384;           // warpgroup 0: TMA producer; warpgroups 1, 2: MMA + epilogue, BM / 2 tile rows each

// Operand-plane formats.  H = false: TF32 hi/lo planes stored as fp32 words (.tf32, K = 8 per MMA, both operands K-major).
// H = true: SCALED FP16 hi/lo planes (.f16, K = 16 per MMA, twice the MMA rate and half the plane bytes): each tensor is
// multiplied by a per-tensor power of two that puts its max |x| in [2^8, 2^9) before the split, so hi + lo carries 22
// significant bits for every element within 2^-22 of the tensor max (absolute floor 2^-25 / scale); the epilogue multiplies
// by the two inverse scales (exact).  In both formats a k-block is ONE 128-byte swizzle row per operand row (four MMA k-slices),
// so the shared memory tiles, the TMA transaction bytes and the 12-MMAs-per-k-block-and-m64 structure are identical.
template <bool H> struct TcFmt {
  static constexpr int BK = H ? 64 : 32;              // elements per k-block (128 bytes)
  // MN-major operands (FP16 planes only)
  static constexpr int MN_BOX = 64;                   // MN elements per MN-major TMA box row (128 bytes)
  static constexpr int MN_BOX_BYTES = 8192;           // BK k-rows x 128 bytes
  static constexpr int MN_KSTEP = 2048;               // bytes between the MN-major k-slices of consecutive MMAs (16 k-rows)
};
constexpr int TC_M64_BYTES = 8192;        // one m64 block of an A plane in both layouts: 64 K-major 128-byte rows / one MN-major box

// ------------------------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra.uni WAIT_DONE;\n"
      "bra.uni WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(addr), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// Programmatic dependent launch: the GEMMs are launched with programmatic stream serialization, so a CTA of the NEXT kernel may
// be scheduled (on an SM the previous kernel no longer needs) and run its prologue -- barrier init, tensor-map
// prefetch -- while the previous kernel's last wave is still computing.  launch_dependents lets our own successor do the same;
// wait blocks until the predecessor grid has completed and its writes are visible: nothing before it touches global memory.
__device__ __forceinline__ void pdl_sync() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
// ------------------------------------------------------------------------------------------ wgmma (sm_90a)
// A warpgroup (4 consecutive warps) issues asynchronous MMAs of 64 rows x N columns into fp32 REGISTERS; operands come from
// shared memory through 64-bit descriptors.  fence before the first MMA that reads / writes registers touched by other code,
// commit closes a group, wait<N> blocks until at most N groups are pending.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// m64nNk16 (FP16 planes; TA / TB = 1: operand stored MN-major) and m64nNk8 (TF32 planes, both operands K-major), D += A.B^T
// (scale_d = 0: D = A.B^T)
template <int TA, int TB>
__device__ __forceinline__ void wg_f16_n128(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, %68;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wg_f16_n64(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, %35, %36;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}
__device__ __forceinline__ void wg_tf32_n128(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wg_tf32_n64(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}

// Shared-memory matrix descriptor (PTX ISA "Matrix Descriptor Format" for wgmma):
//   bits [0,14) start address >> 4 | [16,30) LBO >> 4 | [32,46) SBO >> 4 | [62,64) layout type (1 = SWIZZLE_128B)
// Every tile is 1024-byte aligned, so the base-offset field stays 0.
// K-major: 8-row x 128 B swizzle atoms, SBO = 1024 between 8-row groups, LBO unused (1); the k-slices of one k-block are
// 32 bytes apart along the swizzled row.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// MN-major 16-bit operands (FP16 planes only: wgmma transposes 16-bit types alone): the canonical SWIZZLE_128B layout
// ((8,n),(8,k)):((1,LBO),(8,SBO)) in 16-byte units.  A TMA box is [64 k-rows x 64 mn] = 8 KB with the 16-byte chunks of row r
// XORed with r mod 8; LBO = distance between 64-wide MN blocks (one box, 8192), SBO = distance between 8-row k groups (1024);
// a K = 16 MMA slice is two k groups (2048 bytes).
__device__ __forceinline__ uint64_t make_smem_desc_mn_h(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)(8192 >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
template <bool MN>
__device__ __forceinline__ uint64_t tc_desc(uint32_t base, int k) {
  return MN ? make_smem_desc_mn_h(base + k * TcFmt<true>::MN_KSTEP) : make_smem_desc(base + k * 32);
}

// scale that puts amax into [2^(top-1), 2^top); 1 for an all-zero / non-finite tensor.  Absolute split error 2^-25 / scale
// = 2^-(24+top) of the tensor max.  TOP_SITE leaves 2^7 of headroom below the FP16 maximum for scales PREDICTED from the
// previous call's max; TOP_EXACT is for a scale derived from the very tensor being split.
constexpr int TOP_SITE = 9, TOP_EXACT = 13;
__device__ __forceinline__ float scale_from_amax(float amax, int top) {
  if (!(amax > 0.0f) || !(amax < 3.0e38f)) return 1.0f;
  int e; frexpf(amax, &e);                      // amax = m * 2^e, m in [0.5, 1)
  return ldexpf(1.0f, max(-100, min(100, top - e)));
}

// ------------------------------------------------------------------------------------------ the hi/lo split (every writer of planes)
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  uint32_t h, l;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(x));
  hi = __uint_as_float(h);
  const float r = x - hi;                       // exact
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(r));
  lo = __uint_as_float(l);
}
// FP16 format: xs is the value already multiplied by its scale
__device__ __forceinline__ void split_f16(float xs, __half& hi, __half& lo) {
  hi = __float2half_rn(xs);
  lo = __float2half_rn(xs - __half2float(hi));   // the residual is exact in fp32
}
// two elements at once: cvt.rn.f16x2.f32 (F2FP, full rate) instead of two scalar F2F conversions (quarter-rate pipe; ncu r01:
// the store phase stalled on MIO at the F2Fs); the residuals are exact in fp32.  Returns the packed hi / lo half2 words.
__device__ __forceinline__ void split_f16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(a, b);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}
// FP16 format, end of a pass that wrote planes with scale s: m is the thread's running max |x|.  The warp's max goes into amax_out
// (the scale source of the next call) and a scale that does not fit the data is reported in the sticky flag: bit 0 when a scaled
// value exceeds 60000 (never saturate silently), bit 1 when the site only ever saw all-zero tensors and now there is data.  Both
// pointers may be null.  The warp shuffles: call it from every lane of the warp.
__device__ __forceinline__ void report_scale_miss(float m, float s, unsigned* amax_out, unsigned* flag) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.0f) {
    if (amax_out) atomicMax(amax_out, __float_as_uint(m));        // non-negative floats order like their uint bits
    if (flag && !(m * s <= 60000.0f)) atomicOr(flag, 1u);
    if (flag && s == 0.0f) atomicOr(flag, 2u);
  }
}

// explicit shared-space accesses for the staging tile (a generic pointer makes the compiler emit LD.E / ST.E with their longer latency)
__device__ __forceinline__ float4 lds128(const float* p) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(smem_u32(p)));
  return v;
}

struct TcEpi {
  float* C; int64_t ldc;
  int M, N, K;
  int kb_total, kb_per_split;
  float alpha;
  const float* bias;
  int act;
  const float* mask_src; int64_t ldm; int mask_mode;
  int accumulate;
  float* colsum;                           // optional: colsum[n] += sum_m C[m,n] (bias gradient of the layer whose dZ this GEMM produces)
  void* Chi; void* Clo; int64_t ldp;       // optional hi/lo planes of C (operand cache for the consumers of C): fp32 words (TF32) or halfs
  const float* a_inv; const float* b_inv;  // FP16 planes: device pointers to the operands' inverse scales (null = 1)
  const float* c_scale;                    // FP16 planes of C: device pointer to the scale they are written with
  unsigned* c_amax;                        // optional: atomicMax of |C| (as uint bits) -- the scale source for the consumers of C
  unsigned* flag;                          // FP16 planes of C written with a PREDICTED scale: sticky overflow flag (bit 0)
  uint32_t* relu_bits; int64_t ldrb;       // optional: bit (n % 32) of word n / 32 of row m := C[m,n] > 0
  const uint32_t* mask_bits; int64_t ldmb; // optional: replaces mask_src for mask_mode 1 (same bit layout)
  int skip_c;                              // the planes are the only consumers of C: no fp32 store
  int debug;   // experiments only (env ASE_TC_DEBUG): 1 skip the whole store phase, 4 skip correction MMAs,
               // 16 skip mask loads, 32 skip plane stores, 64 skip column-sum atomics, 128 skip the fp32 C store,
               // 256 generic store phase only, 512 pin the tile height to 128 rows (gemm_tc_plan),
               // 1024 one tile per CTA (no persistent tile loop)
};

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

}  // namespace ase
