// wgmma GEMM for sm_90a with fp32-class accuracy: three tensor-core MMAs per product on hi/lo operand planes.
//
//   C[M,N] = epi(alpha * A . B^T),  A = A_hi + A_lo, B = B_hi + B_lo
//   A.B^T ~= A_hi.B_hi + A_lo.B_hi + A_hi.B_lo       (dropped A_lo.B_lo term is 2^-22 relative)
//
// Plane formats (template parameter H): scaled FP16 halfs (.f16, backend 2, default) or fp32 words holding TF32 values
// (.tf32, backend 1).  FP16 planes are kept in the tensors' natural row-major layout and read K-major or MN-major by TMA /
// wgmma descriptors -- nothing is transposed -- and are normally WRITTEN by the epilogue of the GEMM that produces the tensor.
// wgmma reads 32-bit operands K-major only, so a TF32 operand stored [K, rows] is split into K-major planes by its prep pass.
//
// Kernel (gemm_tc_kernel, BM x BN output tile, BM = 256 or 128, BN = 128 or 64, chosen by gemm_tc_plan): warpgroup 0 = TMA
// producer into a shared-memory ring with mbarrier completion; warpgroups 1, 2 = BM / 2 rows each: wgmma into register
// fragments, every (k-block, m64 block)'s partial -- corrections and A_hi.B_hi -- added into fp32 registers with
// round-to-nearest adds -- the tensor core's own accumulation truncates.
// Store phase: bias / ReLU / tanh / mask (fp32 or 1-bit), optional fp32 C, half planes (predicted power-of-two scale), ReLU
// activity bits, max |C|, fused column sums, split-K fp32 RED.  Interior, aligned 128-column tiles are stored straight from
// the accumulator fragments (epilogue_frag: no staging tile, no CTA-wide barrier, one quad shuffle per value pair so that a
// lane stores 4 consecutive columns); every other tile goes registers -> shared staging tile -> coalesced pass (epilogue_rows).
// Descriptor formats follow the PTX ISA "Matrix Descriptor Format" for wgmma.  DESIGN.md section 5 has the numerics.
#include <cuda.h>
#include <cuda_fp16.h>
#include <vector>
#include <unordered_map>
#include <string.h>
#include <stdlib.h>
#include "common.cuh"
#include "kernels.h"
#include "tc_common.cuh"

namespace ase {


// Phase 2 of the epilogue, shared by the tile shapes: a warp writes rows [row0, row0+nrows) of the staged tile; a row is
// written as BNT/4 float4 by consecutive lanes (full 128-byte lines); bias / activation / mask operands are read with the
// same coalesced mapping; optional hi/lo planes of C, the ReLU activity bits, the running max |C| and the fused column sums
// (bias gradient; reduced over the tile's rows in shared memory first: s_colsum[BNT], zeroed by the caller) ride along.
// Every lane stays in both loops for the whole tile (columns past N are predicated off): the bit packing shuffles need all 32.
template <bool H>
__device__ __forceinline__ void epilogue_rows(const TcEpi& e, const float* cs, int cs_ld, float* s_colsum, int row0, int nrows, int BNT, int m0, int n0, int lane) {
  const bool vec_ok = ((e.ldc & 3) == 0) && ((reinterpret_cast<uintptr_t>(e.C) & 15) == 0) &&
                      (!e.mask_mode || e.mask_bits || (((e.ldm & 3) == 0) && ((reinterpret_cast<uintptr_t>(e.mask_src) & 15) == 0)));
  const bool add_bias = e.bias && (!e.accumulate || blockIdx.z == 0);
  const uintptr_t pal = H ? 7 : 15;         // 4 plane elements per lane: 8 bytes (halfs) / 16 bytes (fp32 words)
  const bool pvec = e.Chi && ((e.ldp & 3) == 0) && ((reinterpret_cast<uintptr_t>(e.Chi) & pal) == 0) && ((reinterpret_cast<uintptr_t>(e.Clo) & pal) == 0);
  const float cscale = (H && e.Chi && e.c_scale) ? *e.c_scale : 1.0f;
  const bool use_bits = e.mask_mode == 1 && e.mask_bits != nullptr;
  const int nib_shift = 4 * (lane & 7);
  float amax = 0.0f;
#pragma unroll 1
  for (int cc = lane * 4; cc < ((BNT + 127) & ~127); cc += 128) {          // same trip count for every lane (BNT = 64: lanes 16.. idle along)
    const int n = n0 + cc;
    // columns of this lane's group inside the output.  The full-group test is a separate comparison: folded into the clamp,
    // ptxas (CUDA 12.9, sm_90a) derived it from the min/max instruction's predicate output, which also fires for rem == 0
    const int rem = (cc < BNT) ? e.N - n : 0;
    const bool full = rem >= 4;
    const int nvalid = full ? 4 : (rem > 0 ? rem : 0);
    float bv[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (add_bias) for (int j = 0; j < nvalid; ++j) bv[j] = e.bias[n + j];
    float cs4[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll 4
    for (int r = 0; r < nrows; ++r) {
      const int row = row0 + r, m = m0 + row;
      if (m >= e.M) break;                 // warp-uniform
      const float4 t = (cc < BNT) ? lds128(cs + row * cs_ld + cc) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      float x[4] = {t.x + bv[0], t.y + bv[1], t.z + bv[2], t.w + bv[3]};
      float* cp = e.C + (int64_t)m * e.ldc + n;
      if (e.accumulate) {
        if (vec_ok && full) asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(cp), "f"(x[0]), "f"(x[1]), "f"(x[2]), "f"(x[3]) : "memory");
        else for (int j = 0; j < nvalid; ++j) atomicAdd(cp + j, x[j]);
        continue;
      }
      if (e.act == 1) { for (int j = 0; j < 4; ++j) x[j] = fmaxf(x[j], 0.0f); }
      else if (e.act == 2) { for (int j = 0; j < 4; ++j) x[j] = tanhf(x[j]); }
      if (e.relu_bits) {                   // 8 lanes x 4 columns = one 32-bit word of the row's activity mask
        uint32_t w = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) w |= (j < nvalid && x[j] > 0.0f) ? (1u << j) : 0u;
        w <<= nib_shift;
        w |= __shfl_xor_sync(0xffffffffu, w, 1); w |= __shfl_xor_sync(0xffffffffu, w, 2); w |= __shfl_xor_sync(0xffffffffu, w, 4);
        if ((lane & 7) == 0 && nvalid > 0) e.relu_bits[(int64_t)m * e.ldrb + (n >> 5)] = w;
      }
      if (use_bits) {
        const uint32_t w = (nvalid > 0 && !(e.debug & 16)) ? e.mask_bits[(int64_t)m * e.ldmb + (n >> 5)] >> nib_shift : 0xFu;
#pragma unroll
        for (int j = 0; j < 4; ++j) x[j] = ((w >> j) & 1u) ? x[j] : 0.0f;
      } else if (e.mask_mode && !(e.debug & 16) && nvalid > 0) {
        const float* mp = e.mask_src + (int64_t)m * e.ldm + n;
        float mv[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        if (vec_ok && full) { const float4 q = *reinterpret_cast<const float4*>(mp); mv[0] = q.x; mv[1] = q.y; mv[2] = q.z; mv[3] = q.w; }
        else for (int j = 0; j < nvalid; ++j) mv[j] = mp[j];
        if (e.mask_mode == 1) { for (int j = 0; j < 4; ++j) x[j] = (mv[j] > 0.0f) ? x[j] : 0.0f; }
        else { for (int j = 0; j < 4; ++j) x[j] *= (1.0f - mv[j] * mv[j]); }
      }
      if (e.skip_c || (e.debug & 128)) {}
      else if (vec_ok && full) *reinterpret_cast<float4*>(cp) = make_float4(x[0], x[1], x[2], x[3]);
      else for (int j = 0; j < nvalid; ++j) cp[j] = x[j];
#pragma unroll
      for (int j = 0; j < 4; ++j) { cs4[j] += x[j]; if (j < nvalid) amax = fmaxf(amax, fabsf(x[j])); }
      if (e.Chi && !(e.debug & 32) && nvalid > 0) {       // the consumers of C read these planes directly through TMA: no separate split pass
        if (!H) {
          float h[4], l[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) split_tf32(x[j], h[j], l[j]);
          float* hp = (float*)e.Chi + (int64_t)m * e.ldp + n; float* lp = (float*)e.Clo + (int64_t)m * e.ldp + n;
          if (pvec && full) { *reinterpret_cast<float4*>(hp) = make_float4(h[0], h[1], h[2], h[3]); *reinterpret_cast<float4*>(lp) = make_float4(l[0], l[1], l[2], l[3]); }
          else for (int j = 0; j < nvalid; ++j) { hp[j] = h[j]; lp[j] = l[j]; }
        } else {
          uint2 hv, lv;
          split_f16x2(x[0] * cscale, x[1] * cscale, hv.x, lv.x); split_f16x2(x[2] * cscale, x[3] * cscale, hv.y, lv.y);
          __half* hp = (__half*)e.Chi + (int64_t)m * e.ldp + n; __half* lp = (__half*)e.Clo + (int64_t)m * e.ldp + n;
          if (pvec && full) { *reinterpret_cast<uint2*>(hp) = hv; *reinterpret_cast<uint2*>(lp) = lv; }
          else {
            const uint32_t hw[2] = {hv.x, hv.y}, lw[2] = {lv.x, lv.y};
            for (int j = 0; j < nvalid; ++j) {
              hp[j] = __ushort_as_half((unsigned short)(hw[j >> 1] >> (16 * (j & 1))));
              lp[j] = __ushort_as_half((unsigned short)(lw[j >> 1] >> (16 * (j & 1))));
            }
          }
        }
      }
    }
    if (e.colsum && !e.accumulate && !(e.debug & 64)) for (int j = 0; j < nvalid; ++j) atomicAdd(s_colsum + cc + j, cs4[j]);   // shared-memory atomics
  }
  if ((e.c_amax || (H && e.Chi && e.flag)) && !e.accumulate) report_scale_miss(amax, cscale, e.c_amax, (H && e.Chi) ? e.flag : nullptr);
}

// Interior, aligned tiles of BN = 128 without split-K accumulation take the fragment store phase (epilogue_frag below); the
// staged, generic epilogue_rows above handles everything else.  The host asks the same question for a whole launch (tile 0 of a
// launch whose M and N are whole tiles) to decide whether it may run the persistent kernel.
__host__ __device__ __forceinline__ bool epilogue_frag_ok(const TcEpi& e, int m0, int n0, int bm, int bn, bool H) {
  if (e.accumulate || m0 + bm > e.M || n0 + bn > e.N) return false;
  if ((e.ldc & 3) || (reinterpret_cast<uintptr_t>(e.C) & 15)) return false;
  if (e.bias && (reinterpret_cast<uintptr_t>(e.bias) & 15)) return false;
  if (e.Chi && (!H || (e.ldp & 7) || (reinterpret_cast<uintptr_t>(e.Chi) & 15) || (reinterpret_cast<uintptr_t>(e.Clo) & 15))) return false;
  if (e.mask_mode && !(e.mask_mode == 1 && e.mask_bits) && ((e.ldm & 3) || (reinterpret_cast<uintptr_t>(e.mask_src) & 15))) return false;
  return true;
}

// Fragment store phase: every consumer thread applies the epilogue to the accumulators it holds and stores them itself -- no
// staging tile, no CTA-wide barrier, so a warpgroup starts storing while the other one still computes, and the operand ring is
// never touched.  m64n128 fragment layout: thread t of a warpgroup holds rows 16 (t/32) + (t%32)/4 and + 8 of each m64 block and
// the column pairs 8 j + 2 (t%4), j = 0..15.  Per 16-column group (two j) the lanes of a quad swap one pair with their
// neighbour (shfl.xor 1): even lanes then own columns 2 q .. 2 q + 3 of the group, odd lanes 8 + 2 (q - 1) .. + 3, so a lane
// stores one float4 of C and one uint2 per half plane, and a quad writes whole 32-byte sectors.  A lane's four columns are
// one nibble of the row's 32-column activity word: two groups are OR-ed over the quad into the whole word, and lane q stores
// the word of the thread's q-th row; mask words are read whole by every lane.  Column sums: the thread's rows first, then the
// warp's 8 row lanes (shfl.xor 4 / 8 / 16), then shared-memory atomics into s_colsum.
// Every element sees the operations of epilogue_rows in the same order, so C, the planes and the activity bits are
// bit-identical to it; the multiplies and the bias add are spelled __fmul_rn / __fadd_rn because here -- with no shared-memory
// round trip between them -- the compiler would contract them into an FMA.
// The per-thread arrays of epilogue_frag.  A struct, not a bare array: the compiler merges the stack slots of equally typed bare
// arrays of the functions it inlines into the kernel, epilogue_rows indexes its float[4] / uint32_t[2] arrays dynamically, and a
// merged slot keeps every store of epilogue_frag's (register-resident) arrays alive as local-memory traffic.
template <class T, int N> struct FragArr {
  T v[N];
  __device__ __forceinline__ T& operator[](int i) { return v[i]; }
  __device__ __forceinline__ const T& operator[](int i) const { return v[i]; }
};

template <bool H, int NH>
__device__ __forceinline__ void epilogue_frag(const TcEpi& e, float (&acc)[NH][64], float* s_colsum, int m0, int n0, int wg, int t) {
  constexpr int NROW = 2 * NH;                               // rows per thread; row k is 64 (k / 2) + 8 (k % 2) below the first
  constexpr unsigned FULL = 0xffffffffu;
  const int lane = t & 31, q = lane & 3;
  const bool odd = q & 1;
  const int cq = ((q & 1) << 3) | ((q & 2) << 1);            // this lane's 4 columns inside a 16-column group: 0, 8, 4, 12
  const int64_t m = m0 + wg * NH * 64 + 16 * (t >> 5) + (lane >> 2);
  const int n = n0 + cq;
  // FP16 planes: undo the operands' power-of-two scales (two exact multiplies; their product alone could underflow)
  const float s1 = (H && e.a_inv) ? *e.a_inv : 1.0f;
  const float s2 = e.alpha * ((H && e.b_inv) ? *e.b_inv : 1.0f);
  const float cscale = (H && e.Chi && e.c_scale) ? *e.c_scale : 1.0f;
  const bool use_bits = e.mask_mode == 1 && e.mask_bits != nullptr;
  const uint32_t* mb = use_bits ? e.mask_bits + m * e.ldmb + (n0 >> 5) : nullptr;
  float* cp = e.C + m * e.ldc + n;
  __half* hp = (H && e.Chi) ? (__half*)e.Chi + m * e.ldp + n : nullptr;
  __half* lp = (H && e.Chi) ? (__half*)e.Clo + m * e.ldp + n : nullptr;
  const float* mp = (e.mask_mode && !use_bits) ? e.mask_src + m * e.ldm + n : nullptr;
  const float* bp = e.bias ? e.bias + n : nullptr;
  FragArr<uint32_t, NROW> mw, mwn;                             // the rows' mask words: the next 32 columns' are in flight
#pragma unroll
  for (int k = 0; k < NROW; ++k) { mw[k] = 0; mwn[k] = 0; }
  if (use_bits) {
#pragma unroll
    for (int k = 0; k < NROW; ++k) mw[k] = __ldg(mb + (64 * (k >> 1) + 8 * (k & 1)) * e.ldmb);
  }
  float amax = 0.0f;
  FragArr<uint32_t, NROW> rbw;                              // the rows' activity words: two groups each
#pragma unroll
  for (int k = 0; k < NROW; ++k) rbw[k] = 0;
  // One 16-column group (fragment column blocks j = 2 g, 2 g + 1) per trip of a ROLLED loop: the group is always read from
  // the first 8 registers of each m64 block and the rest move down by 8 at the end of the trip (56 MOVs per block).  Unrolled
  // over the 8 groups the store phase is ~120 KB of straight-line code that every warp walks once per tile, and it ran at
  // the speed of the instruction fetch: twice as long as the staged store phase it replaces.
#pragma unroll 1
  for (int g = 0; g < 8; ++g) {
    const int w = g >> 1;                                    // 32 columns: one word of activity / mask bits per row
    if (use_bits && !(g & 1) && w < 3) {
#pragma unroll
      for (int k = 0; k < NROW; ++k) mwn[k] = __ldg(mb + (64 * (k >> 1) + 8 * (k & 1)) * e.ldmb + w + 1);
    }
    const int c = 16 * g, sh = 16 * (g & 1) + cq;          // sh: this lane's nibble of the word
    FragArr<float, 4> bv = {{0.0f, 0.0f, 0.0f, 0.0f}};
    if (bp) { const float4 b4 = *reinterpret_cast<const float4*>(bp + c); bv[0] = b4.x; bv[1] = b4.y; bv[2] = b4.z; bv[3] = b4.w; }
    FragArr<float, 4> csum = {{0.0f, 0.0f, 0.0f, 0.0f}};
#pragma unroll
    for (int k = 0; k < NROW; ++k) {
      const int64_t ro = 64 * (k >> 1) + 8 * (k & 1);
      const float* a = acc[k >> 1] + 2 * (k & 1);          // a[0..1]: block 2 g, a[4..5]: block 2 g + 1
      const float r0 = __shfl_xor_sync(FULL, odd ? a[0] : a[4], 1), r1 = __shfl_xor_sync(FULL, odd ? a[1] : a[5], 1);
      FragArr<float, 4> x;
      x[0] = odd ? r0 : a[0]; x[1] = odd ? r1 : a[1]; x[2] = odd ? a[4] : r0; x[3] = odd ? a[5] : r1;
#pragma unroll
      for (int j = 0; j < 4; ++j) x[j] = __fadd_rn(__fmul_rn(s2, __fmul_rn(s1, x[j])), bv[j]);
      if (e.act == 1) {
#pragma unroll
        for (int j = 0; j < 4; ++j) x[j] = fmaxf(x[j], 0.0f);
      } else if (e.act == 2) {
#pragma unroll
        for (int j = 0; j < 4; ++j) x[j] = tanhf(x[j]);
      }
      if (e.relu_bits) {
        uint32_t nib = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) nib |= (x[j] > 0.0f) ? (1u << j) : 0u;
        rbw[k] |= nib << sh;
      }
      if (use_bits) {
#pragma unroll
        for (int j = 0; j < 4; ++j) x[j] = ((mw[k] >> (sh + j)) & 1u) ? x[j] : 0.0f;
      } else if (mp) {
        const float4 q4 = *reinterpret_cast<const float4*>(mp + ro * e.ldm + c);
        const FragArr<float, 4> mv = {{q4.x, q4.y, q4.z, q4.w}};
        if (e.mask_mode == 1) {
#pragma unroll
          for (int j = 0; j < 4; ++j) x[j] = (mv[j] > 0.0f) ? x[j] : 0.0f;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) x[j] *= (1.0f - mv[j] * mv[j]);
        }
      }
      if (!e.skip_c) *reinterpret_cast<float4*>(cp + ro * e.ldc + c) = make_float4(x[0], x[1], x[2], x[3]);
#pragma unroll
      for (int j = 0; j < 4; ++j) { csum[j] += x[j]; amax = fmaxf(amax, fabsf(x[j])); }
      if (H && hp) {
        uint2 hv, lv;
        split_f16x2(x[0] * cscale, x[1] * cscale, hv.x, lv.x); split_f16x2(x[2] * cscale, x[3] * cscale, hv.y, lv.y);
        *reinterpret_cast<uint2*>(hp + ro * e.ldp + c) = hv;
        *reinterpret_cast<uint2*>(lp + ro * e.ldp + c) = lv;
      }
    }
    if (e.colsum) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float v = csum[j];
        v += __shfl_xor_sync(FULL, v, 4); v += __shfl_xor_sync(FULL, v, 8); v += __shfl_xor_sync(FULL, v, 16);
        if (lane < 4) atomicAdd(s_colsum + c + cq + j, v);
      }
    }
    if (e.relu_bits && (g & 1)) {
      uint32_t word = 0;
#pragma unroll
      for (int k = 0; k < NROW; ++k) {
        uint32_t v = rbw[k];
        v |= __shfl_xor_sync(FULL, v, 1); v |= __shfl_xor_sync(FULL, v, 2);
        if (q == k) word = v;
        rbw[k] = 0;
      }
      if (q < NROW) e.relu_bits[(m + 64 * (q >> 1) + 8 * (q & 1)) * e.ldrb + (n0 >> 5) + w] = word;
    }
    if (g & 1) {
#pragma unroll
      for (int k = 0; k < NROW; ++k) mw[k] = mwn[k];
    }
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
      for (int i = 0; i < 56; ++i) acc[h][i] = acc[h][i + 8];
  }
  if (e.c_amax || (H && e.Chi && e.flag)) report_scale_miss(amax, cscale, e.c_amax, (H && e.Chi) ? e.flag : nullptr);
}

// Ring depth per tile shape: as many stages as fit in ~200 KB of the 227 KB an H100 block may use
template <int BM, int BN> constexpr int tc_stages() { return (200 * 1024) / (256 * (BM + BN)); }

template <int BM, int BN, int STAGES>
struct TcSmem {
  static constexpr int A_BYTES = BM * 128;                   // per plane: one 128-byte k-block row per operand row
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;
  // [2][BN] fp32 column sums, behind the barriers: never over the ring.  The persistent kernel alternates the two slots by tile
  static constexpr int COLSUM_OFF = STAGES * STAGE_BYTES + 256;
  static constexpr int TOTAL = COLSUM_OFF + 2 * 512 + 1024 /*align slack*/;
  static_assert(BM * (BN + 4) * 4 <= STAGES * STAGE_BYTES, "the generic store phase's staging tile lives over the ring");
};

// one 64 x BN MMA over k-slice k (32 bytes of K) of a k-block; sd = 0 starts a fresh accumulator
template <int BN, bool AMN, bool BMN, bool H>
__device__ __forceinline__ void wg_mma(float (&d)[BN / 2], uint32_t a, uint32_t b, int k, int sd) {
  const uint64_t da = tc_desc<AMN>(a, k), db = tc_desc<BMN>(b, k);
  if constexpr (H) {
    if constexpr (BN == 128) wg_f16_n128<AMN, BMN>(d, da, db, sd); else wg_f16_n64<AMN, BMN>(d, da, db, sd);
  } else {
    if constexpr (BN == 128) wg_tf32_n128(d, da, db, sd); else wg_tf32_n64(d, da, db, sd);
  }
}

// fp32-exact accumulation ("accumulate outside the tensor core", Ootomo & Yokota 2022): the tensor core adds into its
// accumulator with truncation, which over K/8 x 3 sequential MMAs costs ~1e-5 absolute on O(1) sums -- enough to flip ReLU
// masks against the fp32 reference.  So the tensor core accumulates only WITHIN one k-block of 64 halfs / 32 TF32 words:
// per m64 block the 8 correction MMAs (A_lo.B_hi, A_hi.B_lo; 2^-11 of the main term, the first one starting a fresh
// fragment) come first, then the 4 main MMAs A_hi.B_hi add into the same partial, and the partial is added into the fp32
// accumulator with round-to-nearest FADDs.  The main term sees 4 truncating adds per rounded add (one more than with a fresh
// main partial) and the corrections no longer truncate across all of K.
//
// Warp specialisation: warpgroup 0 (register budget lowered to 40) is the TMA producer into a STAGES-deep shared-memory ring
// with mbarrier completion; warpgroups 1 and 2 (232 registers) each own BM / 2 rows of the BM x BN tile as BM / 128 m64
// blocks -- at BM = 256 two 64 x BN accumulators plus one partial, 192 registers at BN = 128 -- issue their wgmma, and run
// the store phase.  While one warpgroup waits for its partial and adds it, the other's MMAs keep the tensor core busy.
//
// PERSIST = false: one tile per CTA, blockIdx = (n tile, m tile, K split).  PERSIST = true (launches whose every tile takes the
// fragment store phase, see gemm_tc): min(tiles, SMs) CTAs, CTA b computes the linear tiles b, b + gridDim.x, ... in the same
// raster order (n fastest, then m).  Barrier set-up, tensor-map prefetch and the PDL wait happen once per CTA, the ring's
// stage index and phase parity run on over all of the CTA's k-blocks, and the producer issues the next tile's k-blocks as soon
// as stages free up -- the fragment store phase never touches the ring, so the next tile's first stages land under it.
template <int BM, int BN, int STAGES, bool AMN, bool BMN, bool H, bool PERSIST>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmAhi, const __grid_constant__ CUtensorMap tmAlo,
               const __grid_constant__ CUtensorMap tmBhi, const __grid_constant__ CUtensorMap tmBlo, const TcEpi e) {
  static_assert(H || (!AMN && !BMN), "TF32 wgmma reads K-major operands only");
  static_assert(BM == 128 || BM == 256, "tile height");
  static_assert(!PERSIST || (H && BN == 128), "the persistent kernel stores every tile from the fragments");
  using SM = TcSmem<BM, BN, STAGES>;
  using F = TcFmt<H>;
  constexpr int R = BN / 2;                        // fragment registers per thread (64 x BN fp32 over 128 threads)
  constexpr int NH = BM / 128;                     // m64 blocks per consumer warpgroup
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * SM::STAGE_BYTES);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kb_begin = PERSIST ? 0 : blockIdx.z * e.kb_per_split;
  const int nkb = PERSIST ? e.kb_total : min(e.kb_per_split, e.kb_total - kb_begin);
  const int tiles_n = PERSIST ? e.N / BN : 1;      // persistent launches have whole tiles in M and N
  const int ntiles = PERSIST ? (e.M / BM) * tiles_n : 1;
  const int tile0 = PERSIST ? (int)blockIdx.x : 0, tile_step = PERSIST ? (int)gridDim.x : 1;
  auto tile_m0 = [&](int tile) { return PERSIST ? (tile / tiles_n) * BM : (int)blockIdx.y * BM; };
  auto tile_n0 = [&](int tile) { return PERSIST ? (tile % tiles_n) * BN : (int)blockIdx.x * BN; };

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmAhi)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmAlo)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmBhi)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmBlo)) : "memory");
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }   // 2 consumer warpgroups release a stage
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  float* s_colsum = reinterpret_cast<float*>(smem + SM::COLSUM_OFF);   // per-tile column sums, [2][BN]
  if (threadIdx.x < 2 * BN) s_colsum[threadIdx.x] = 0.0f;
  __syncthreads();
  pdl_sync();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && lane == 0) {
      int it = 0;                                  // k-blocks issued over all tiles: ring stage and phase
      for (int tile = tile0; tile < ntiles; tile += tile_step) {
        const int m0 = tile_m0(tile), n0 = tile_n0(tile);
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          mbar_wait(&empty[s], ph ^ 1);
          mbar_expect_tx(&full[s], SM::STAGE_BYTES);
          uint8_t* st = smem + s * SM::STAGE_BYTES;
          const int k0 = (kb_begin + kb) * F::BK;
          if (!AMN) {          // K-major planes [rows, K]: one box of BM rows x one k-block
            tma_load_2d(st, &tmAhi, &full[s], k0, m0);
            tma_load_2d(st + SM::A_BYTES, &tmAlo, &full[s], k0, m0);
          } else {             // MN-major planes [K, rows]: boxes of BK k-rows x 128 bytes of m
#pragma unroll
            for (int b = 0; b < BM / F::MN_BOX; ++b) {
              tma_load_2d(st + b * F::MN_BOX_BYTES, &tmAhi, &full[s], m0 + b * F::MN_BOX, k0);
              tma_load_2d(st + SM::A_BYTES + b * F::MN_BOX_BYTES, &tmAlo, &full[s], m0 + b * F::MN_BOX, k0);
            }
          }
          if (!BMN) {
            tma_load_2d(st + 2 * SM::A_BYTES, &tmBhi, &full[s], k0, n0);
            tma_load_2d(st + 2 * SM::A_BYTES + SM::B_BYTES, &tmBlo, &full[s], k0, n0);
          } else {
#pragma unroll
            for (int b = 0; b < BN / F::MN_BOX; ++b) {
              tma_load_2d(st + 2 * SM::A_BYTES + b * F::MN_BOX_BYTES, &tmBhi, &full[s], n0 + b * F::MN_BOX, k0);
              tma_load_2d(st + 2 * SM::A_BYTES + SM::B_BYTES + b * F::MN_BOX_BYTES, &tmBlo, &full[s], n0 + b * F::MN_BOX, k0);
            }
          }
        }
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int wg = (warp >> 2) - 1;                  // consumer warpgroup: tile rows [wg BM/2, (wg + 1) BM/2)
  const int t = threadIdx.x & 127;
  const int et = threadIdx.x - 128;                // 0..255 within the consumer warps
  const bool corrections = !(e.debug & 4);
#pragma unroll 1
  for (int tile = tile0; tile < ntiles; tile += tile_step) {
    const int ti = tile / tile_step;                 // tiles this CTA has done (tile0 < tile_step)
    float acc[NH][R], part[R];
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
      for (int j = 0; j < R; ++j) acc[h][j] = 0.0f;
    // The first MMA of a k-block starts a fresh partial under a run-time predicate, so the compiler takes the partial as read
    // there: without this, the last tile's partial would stay live across the store phase (64 registers: spills at BM = 256)
    if constexpr (PERSIST) {
#pragma unroll
      for (int j = 0; j < R; ++j) part[j] = 0.0f;
    }
    for (int kb = 0; kb < nkb; ++kb) {
      const int it = ti * nkb + kb;                  // k-blocks consumed over all tiles: ring stage and phase
      const int s = it % STAGES;
      mbar_wait(&full[s], (it / STAGES) & 1);
      const uint32_t sa = smem_u32(smem + s * SM::STAGE_BYTES);
      const uint32_t b_hi = sa + 2 * SM::A_BYTES, b_lo = b_hi + SM::B_BYTES;
#pragma unroll
      for (int h = 0; h < NH; ++h) {
        // m64 block wg NH + h starts (wg NH + h) x 8 KB into each A plane in both layouts
        const uint32_t a_hi = sa + (wg * NH + h) * TC_M64_BYTES, a_lo = a_hi + SM::A_BYTES;
        wg_fence();
        if (corrections) {
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            wg_mma<BN, AMN, BMN, H>(part, a_lo, b_hi, k, k > 0 ? 1 : 0);
            wg_mma<BN, AMN, BMN, H>(part, a_hi, b_lo, k, 1);
          }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) wg_mma<BN, AMN, BMN, H>(part, a_hi, b_hi, k, (corrections || k > 0) ? 1 : 0);
        wg_commit();
        wg_wait<0>();
        if (h == NH - 1 && t == 0) mbar_arrive(&empty[s]);   // every MMA reading this stage is done
#pragma unroll
        for (int j = 0; j < R; ++j) acc[h][j] += part[j];    // round-to-nearest fp32 accumulation across k-blocks
      }
    }
    const int m0 = tile_m0(tile), n0 = tile_n0(tile);
    // Column sums: the persistent kernel alternates the two slots by tile.  Tile i + 2 reaches slot i & 1 only after every
    // consumer thread passed the barrier below for tile i + 1, i.e. after it flushed and zeroed its column of tile i.
    float* cs_slot = s_colsum + (PERSIST ? (ti & 1) * BN : 0);
    bool frag = PERSIST;
    if constexpr (BN == 128 && !PERSIST) frag = epilogue_frag_ok(e, m0, n0, BM, BN, H) && !(e.debug & 256);
    if (frag) {
      if constexpr (BN == 128) { if (!(e.debug & 1)) epilogue_frag<H, NH>(e, acc, cs_slot, m0, n0, wg, t); }
    } else if constexpr (!PERSIST) {
      // Generic store phase.  Phase 1: accumulators -> shared staging tile [BM][BN+4] over the idle ring (every TMA load was
      // consumed; the barrier waits for the other warpgroup's last MMAs).  Fragment layout of m64nN: thread t holds rows
      // 16 (t/32) + (t%32)/4 (+8) and column pairs 8 j + 2 (t%4).
      asm volatile("bar.sync 1, 256;" ::: "memory");      // the 8 consumer warps only
      float* cs = reinterpret_cast<float*>(smem);
      constexpr int CS_LD = BN + 4;
      // FP16 planes: undo the operands' power-of-two scales (two exact multiplies; their product alone could underflow)
      const float s1 = (H && e.a_inv) ? *e.a_inv : 1.0f;
      const float s2 = e.alpha * ((H && e.b_inv) ? *e.b_inv : 1.0f);
#pragma unroll
      for (int h = 0; h < NH; ++h) {
        const int row = (wg * NH + h) * 64 + 16 * (t >> 5) + ((t & 31) >> 2);
        float* c0 = cs + row * CS_LD + 2 * (t & 3);
#pragma unroll
        for (int j = 0; j < R / 4; ++j) {
          const float* a = acc[h] + 4 * j;
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(smem_u32(c0 + 8 * j)), "f"(s2 * (s1 * a[0])), "f"(s2 * (s1 * a[1])) : "memory");
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(smem_u32(c0 + 8 * CS_LD + 8 * j)), "f"(s2 * (s1 * a[2])), "f"(s2 * (s1 * a[3])) : "memory");
        }
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      // Phase 2: coalesced epilogue -- consumer warp w owns rows [w BM/8, (w + 1) BM/8)
      constexpr int NRW = BM / 8;
      if (!(e.debug & 1)) epilogue_rows<H>(e, cs, CS_LD, s_colsum, (warp - 4) * NRW, NRW, BN, m0, n0, lane);
    }
    if (e.colsum && !e.accumulate) {
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (et < BN && n0 + et < e.N) atomicAdd(e.colsum + n0 + et, cs_slot[et]);
      if (PERSIST && et < BN) cs_slot[et] = 0.0f;
    }
  }
}

// ------------------------------------------------------------------------------------------ operand prep

// split src[rows, cols] (ld) into zero-padded hi/lo planes [rows_p, cols_p]
__global__ void __launch_bounds__(256)
tc_prep_kernel(const float* __restrict__ src, int64_t ld, int rows, int cols, int rows_p, int cols_p, float* __restrict__ hi,
               float* __restrict__ lo) {
  const int64_t total = (int64_t)rows_p * cols_p;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / cols_p), c = (int)(i - (int64_t)r * cols_p);
    float h = 0.0f, l = 0.0f;
    if (r < rows && c < cols) split_tf32(src[(int64_t)r * ld + c], h, l);
    hi[i] = h; lo[i] = l;
  }
}

// The same split of a source stored TRANSPOSED, [cols, rows] (ld): planes[r][c] = split(src[c * ld + r]).  32 x 32 tiles pass
// through shared memory so that both the reads (along r) and the plane writes (along c) are coalesced.  rows_p and cols_p are
// multiples of 32; block 32 x 8, grid (rows_p / 32, cols_p / 32).
__global__ void __launch_bounds__(256)
tc_prep_t_kernel(const float* __restrict__ src, int64_t ld, int rows, int cols, int cols_p, float* __restrict__ hi,
                 float* __restrict__ lo) {
  __shared__ float tile[32][33];
  const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32, tx = threadIdx.x;
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int c = c0 + j, r = r0 + tx;
    tile[j][tx] = (r < rows && c < cols) ? src[(int64_t)c * ld + r] : 0.0f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int64_t o = (int64_t)(r0 + j) * cols_p + c0 + tx;
    float h, l;
    split_tf32(tile[tx][j], h, l);
    hi[o] = h; lo[o] = l;
  }
}

// FP16 format: max |src| of every item's [rows, cols] view into its amax slot.  blockIdx.y = item, blockIdx.x = slice of it.
template <int N>
__global__ void __launch_bounds__(256)
tc_amax_kernel(const TcPrepList<N> l) {
  const TcPrepItem it = l.item[blockIdx.y];
  const int64_t total = (int64_t)it.rows * it.cols;
  float m = 0.0f;
  if (it.cols == it.ld) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(it.src[i]));
  } else {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
      const int r = (int)(i / it.cols), c = (int)(i - (int64_t)r * it.cols);
      m = fmaxf(m, fabsf(it.src[(int64_t)r * it.ld + c]));
    }
  }
  report_scale_miss(m, 1.0f, it.amax, nullptr);      // no flag: the max only
}

// FP16 format: split every item into its half planes, 4 consecutive columns per thread (ldp is a multiple of 8); blockIdx.y = item,
// blockIdx.x = slice of it.  Two modes, both without a host sync:
//   exact     : the scale is derived from the max already in the item's amax slot and published with its inverse in scale[0..1]
//               for the epilogues of the GEMMs that consume these planes;
//   predicted : scale[0] holds the scale derived from the previous call's max at this site; this pass tracks the current max into
//               the amax slot for the next call and reports a scale miss in `flag`.
// scale_copy, if set, receives the scale and its inverse (0 for a zero scale): a copy that outlives the site's slot.
template <int N>
__global__ void __launch_bounds__(256)
tc_split_h_kernel(const TcPrepList<N> l, int exact, int top, unsigned* __restrict__ flag) {
  const TcPrepItem it = l.item[blockIdx.y];
  float s;
  if (exact) {
    s = scale_from_amax(__uint_as_float(*it.amax), top);
    if (blockIdx.x == 0 && threadIdx.x == 0) { it.scale[0] = s; it.scale[1] = 1.0f / s; }
  } else s = it.scale[0];
  if (it.scale_copy && blockIdx.x == 0 && threadIdx.x == 0) { it.scale_copy[0] = s; it.scale_copy[1] = (s != 0.0f) ? 1.0f / s : 0.0f; }
  __half* hi = (__half*)it.hi; __half* lo = (__half*)it.lo;
  const int c4n = it.ldp >> 2;
  const int64_t total = (int64_t)it.rows_p * c4n;
  const bool vec = ((it.ld & 3) == 0) && ((reinterpret_cast<uintptr_t>(it.src) & 15) == 0);
  float m = 0.0f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / c4n), c = (int)(i - (int64_t)r * c4n) * 4;
    float x[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (r < it.rows) {
      const float* sp = it.src + (int64_t)r * it.ld + c;
      if (vec && c + 4 <= it.cols) { const float4 t = *reinterpret_cast<const float4*>(sp); x[0] = t.x; x[1] = t.y; x[2] = t.z; x[3] = t.w; }
      else for (int j = 0; j < 4; ++j) if (c + j < it.cols) x[j] = sp[j];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) m = fmaxf(m, fabsf(x[j]));
    uint2 hv, lv;
    split_f16x2(x[0] * s, x[1] * s, hv.x, lv.x); split_f16x2(x[2] * s, x[3] * s, hv.y, lv.y);
    *reinterpret_cast<uint2*>(hi + (int64_t)r * it.ldp + c) = hv;
    *reinterpret_cast<uint2*>(lo + (int64_t)r * it.ldp + c) = lv;
  }
  if (!exact) report_scale_miss(m, s, it.amax, flag);
}

// FP16 format, start of every top-level call: fold the maxima tracked during the previous call into the sites' scales (the
// prediction for this call), check that the previous prediction did not lose precision, and clear the maxima.
__global__ void __launch_bounds__(256)
tc_site_update_kernel(unsigned* __restrict__ amax, float* __restrict__ scale, int n, float* __restrict__ static_scale, float static_value,
                      unsigned* __restrict__ flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) { static_scale[0] = static_value; static_scale[1] = 1.0f / static_value; }
  if (i >= n) return;
  const float a = __uint_as_float(amax[i]);
  const float s0 = scale[2 * i];
  if (a > 0.0f) {
    if (s0 != 0.0f && a * s0 < 0.015625f) atomicOr(flag, 2u);        // the tensor shrank by > 2^14 .. 2^15 since the last call: the split lost bits
    const float s = scale_from_amax(a, TOP_SITE);
    scale[2 * i] = s; scale[2 * i + 1] = 1.0f / s;
    amax[i] = 0u;
  }                                          // a site that only ever saw all-zero tensors keeps scale 0 (zero planes, zero inverse)
}

// ------------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  }
  return fn;
}

// cuTensorMapEncodeTiled costs microseconds and the learner re-issues the same ~230 maps every minibatch: memoise.
struct MapKey {
  const void* base; int rows, cols; int64_t ld; int box_rows; int mn;     // mn: bit 0 = MN-major, bit 1 = half planes
  bool operator==(const MapKey& o) const { return base == o.base && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows && mn == o.mn; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = (size_t)k.base;
    h ^= (size_t)k.rows * 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
    h ^= (size_t)k.cols * 0xC2B2AE3D27D4EB4Full + (h << 6) + (h >> 2);
    h ^= (size_t)k.ld * 0x165667B19E3779F9ull + (size_t)k.box_rows * 31 + (size_t)k.mn;
    return h;
  }
};
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash>& map_cache() { static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> c; return c; }

// 2D map over [rows, cols] elements (cols contiguous, row stride ld elements); the box is one 128-byte row chunk
// (32 fp32 words / 64 halfs) x box_rows, 128-byte swizzle
static int encode_cached(CUtensorMap* tm, const void* base, int rows, int cols, int64_t ld, int box_rows, bool mn_major, bool half) {
  MapKey k{base, rows, cols, ld, box_rows, (mn_major ? 1 : 0) | (half ? 2 : 0)};
  auto& c = map_cache();
  auto it = c.find(k);
  if (it != c.end()) { memcpy(tm, &it->second, sizeof(CUtensorMap)); return ASE_OK; }
  PFN_encodeTiled enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled not available from the driver"); return ASE_ERR_UNSUPPORTED; }
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)ld * (half ? 2 : 4)};
  cuuint32_t box[2] = {half ? 64u : 32u, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  if (mn_major && !half) { set_error("wgmma GEMM: TF32 planes cannot be read MN-major"); return ASE_ERR_INVALID; }
  CUresult r = enc(tm, half ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(%d x %d, ld %lld, box %d) failed with CUresult %d", rows, cols, (long long)ld, box_rows, (int)r); return ASE_ERR_CUDA; }
  if (c.size() > 8192) c.clear();
  c.emplace(k, *tm);
  return ASE_OK;
}

static inline int pad_to(int x, int m) { return (x + m - 1) / m * m; }

// planes are padded to whole tiles in both dimensions (zero filled by the prep kernel), M to the tallest tile (256 rows)
// (the FP16 format needs half of it: [*, pad(K, 64)] halfs <= [*, pad(K, 32)] words; the first TC_WS_HEAD bytes hold the
// amax / scale slots of a registry-less call)
// amax / scale slots of a registry-less call).  The plane slots are sized in fp32 words of K padded to 32 in BOTH formats:
// the split passes and gemm_tc place the planes with tc_ws_slots, the one layout gemm_tc_workspace_bytes sums up.
constexpr int64_t TC_WS_HEAD = 1024;
constexpr int TC_MPAD = 256;
struct TcWsSlots { int64_t a, b; };      // bytes of one A plane slot / one B plane slot
static TcWsSlots tc_ws_slots(int M, int N, int K) {
  const int64_t Mp = pad_to(M, TC_MPAD), Np = pad_to(N, 128), Kw = pad_to(K, TC_KPAD);
  return {align_up(Mp * Kw * 4, 1024), align_up(Np * Kw * 4, 1024)};
}
int64_t gemm_tc_workspace_bytes(int M, int N, int K) {
  const TcWsSlots s = tc_ws_slots(M, N, K);
  return TC_WS_HEAD + 2 * s.a + 2 * s.b;
}

// a missing / small / misaligned workspace is an ERROR, never a silent fallback
int gemm_tc_check_workspace(const AseGemmParams& p) {
  if (!p.workspace || p.workspace_bytes < gemm_tc_workspace_bytes(p.M, p.N, p.K)) {
    set_error("wgmma GEMM %dx%dx%d: workspace %lld bytes < required %lld", p.M, p.N, p.K, (long long)p.workspace_bytes,
              (long long)gemm_tc_workspace_bytes(p.M, p.N, p.K));
    return ASE_ERR_WORKSPACE;
  }
  if (reinterpret_cast<uintptr_t>(p.workspace) & 1023) { set_error("wgmma GEMM: workspace must be 1024-byte aligned"); return ASE_ERR_WORKSPACE; }
  return ASE_OK;
}

// TF32 operand with `rows` = its M/N extent and reduction length K, stored [rows, K] (trans == 0) or [K, rows] (trans == 1):
// K-major planes [rows_p, Kp] either way
static int prep_operand(const float* src, int64_t ld, int trans, int rows, int K, int rows_p, int Kp, float* hi, float* lo, cudaStream_t st) {
  if (trans) {
    tc_prep_t_kernel<<<dim3(rows_p / 32, Kp / 32), dim3(32, 8), 0, st>>>(src, ld, rows, K, Kp, hi, lo);
  } else {
    const int64_t total = (int64_t)rows_p * Kp;
    tc_prep_kernel<<<(int)imin64((total + 255) / 256, NUM_SMS * 16), 256, 0, st>>>(src, ld, rows, K, rows_p, Kp, hi, lo);
  }
  ASE_LAUNCH_OK();
  return ASE_OK;
}

// FP16 format: split one tensor into half planes.  With a predicted scale (scale_known: the site's scale from the previous call)
// one pass also tracks the tensor's max for the next call.  Else the scale is exact, from the max in it.amax, which a max pass
// computes first unless max_known (the GEMM that wrote the tensor tracked it).
static int materialize_h(const TcPrepItem& it, bool scale_known, bool max_known, unsigned* flag, int top, cudaStream_t st) {
  const TcPrepList<1> l{{it}};
  if (!scale_known && !max_known) {
    const int64_t total = (int64_t)it.rows * it.cols;
    tc_amax_kernel<1><<<(int)imin64((total + 1023) / 1024, NUM_SMS * 8), 256, 0, st>>>(l);
    ASE_LAUNCH_OK();
  }
  const int64_t total = (int64_t)it.rows_p * (it.ldp / 4);
  tc_split_h_kernel<1><<<(int)imin64((total + 255) / 256, NUM_SMS * 16), 256, 0, st>>>(l, scale_known ? 0 : 1, top, flag);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

// Optional per-launch timing of the main kernel (bench.py's live roofline measurement): CUDA events recorded on
// the launching stream around every gemm_tc_kernel launch; read back (with a sync) by ase_gemm_tc_profile_read.
struct TcProfile {
  bool on = false;
  std::vector<cudaEvent_t> ev;   // pairs
  size_t used = 0;
  double flops = 0.0;
};
static TcProfile g_prof;

static void prof_mark(cudaStream_t st) {
  if (g_prof.used == g_prof.ev.size()) {
    cudaEvent_t e;
    if (cudaEventCreate(&e) != cudaSuccess) { g_prof.on = false; return; }
    g_prof.ev.push_back(e);
  }
  cudaEventRecord(g_prof.ev[g_prof.used++], st);
}

static int tc_pdl() {   // env ASE_TC_PDL=0 launches the GEMMs fully stream-serialised
  static int v = -1;
  if (v < 0) { const char* d = getenv("ASE_TC_PDL"); v = d ? (atoi(d) != 0) : 1; }
  return v;
}

template <int BM, int BN, bool AMN, bool BMN, bool H, bool PERSIST>
static int launch_tc(const CUtensorMap& ah, const CUtensorMap& al, const CUtensorMap& bh, const CUtensorMap& bl, const TcEpi& e,
                     int splits, cudaStream_t st) {
  constexpr int STAGES = tc_stages<BM, BN>();
  using SM = TcSmem<BM, BN, STAGES>;
  static bool attr_set = false;
  if (!attr_set) {
    ASE_CUDA_OK(cudaFuncSetAttribute(gemm_tc_kernel<BM, BN, STAGES, AMN, BMN, H, PERSIST>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::TOTAL));
    attr_set = true;
  }
  const dim3 grid = PERSIST ? dim3(min((e.M / BM) * (e.N / BN), NUM_SMS)) : dim3(ceil_div(e.N, BN), ceil_div(e.M, BM), splits);
  const bool prof = g_prof.on;
  if (prof) prof_mark(st);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = dim3(TC_THREADS); cfg.dynamicSmemBytes = SM::TOTAL; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = tc_pdl();
  cfg.attrs = attr; cfg.numAttrs = 1;
  ASE_CUDA_OK(cudaLaunchKernelEx(&cfg, gemm_tc_kernel<BM, BN, STAGES, AMN, BMN, H, PERSIST>, ah, al, bh, bl, e));
  if (prof) { prof_mark(st); g_prof.flops += 2.0 * (double)e.M * (double)e.N * (double)e.K; }
  ASE_LAUNCH_OK();
  return ASE_OK;
}

template <int BM, int BN, bool H, bool PERSIST = false>
static int launch_tc_major(bool amn, bool bmn, const CUtensorMap& ah, const CUtensorMap& al, const CUtensorMap& bh, const CUtensorMap& bl,
                           const TcEpi& e, int splits, cudaStream_t st) {
  if constexpr (!H) {
    if (amn || bmn) { set_error("wgmma GEMM: TF32 operand planes must be K-major"); return ASE_ERR_INVALID; }
    return launch_tc<BM, BN, false, false, false, false>(ah, al, bh, bl, e, splits, st);
  } else {
    if (!amn && !bmn) return launch_tc<BM, BN, false, false, true, PERSIST>(ah, al, bh, bl, e, splits, st);
    if (!amn && bmn) return launch_tc<BM, BN, false, true, true, PERSIST>(ah, al, bh, bl, e, splits, st);
    if (amn && !bmn) return launch_tc<BM, BN, true, false, true, PERSIST>(ah, al, bh, bl, e, splits, st);
    return launch_tc<BM, BN, true, true, true, PERSIST>(ah, al, bh, bl, e, splits, st);
  }
}

static int tc_debug() {   // env ASE_TC_DEBUG: experiment bits, see TcEpi::debug
  static int v = -1;
  if (v < 0) { const char* d = getenv("ASE_TC_DEBUG"); v = d ? atoi(d) : 0; }
  return v;
}

// Tile plan of one tensor-core GEMM: the tile height BM, the tile width BN and the number of K splits.  BN = 128, or 64
// when N <= 64.  (BM, splits) minimise a launch-time model: whole waves of one-CTA-per-SM launches times the per-CTA time
//   TC_CTA_FIXED + (k-blocks per split + TC_CTA_STORE) x BM BN / 128^2,
// in units of one k-block of a 128 x 128 tile (12 MMAs per consumer warpgroup and m64 block): a CTA pays a fixed start (first TMA
// round trip, barrier set-up) and a store phase that grows with its area.  Every extra split adds 3 % for its RED pass over C.
// split_k > 1 (with accumulate) is taken as given, 0 / 1 is none; split_k < 0 (TC_SPLIT_AUTO, with accumulate: the learner's
// dW GEMMs) lets the model pick up to 64 splits of at least 4 k-blocks each: the learner's small dW outputs (a few 128-row
// tiles over K = 4096 .. 32768) need 16-64 splits to give every SM a CTA.  Without accumulate there is no split-K.
constexpr double TC_CTA_FIXED = 1.0, TC_CTA_STORE = 1.0;
TcPlan gemm_tc_plan(int M, int N, int K, int accumulate, int split_k, int sms, bool f16) {
  TcPlan best{128, N > 64 ? 128 : 64, 1};
  const int kb_total = ceil_div(K, f16 ? TcFmt<true>::BK : TcFmt<false>::BK);
  int smin = 1, smax = 1;
  if (accumulate && split_k > 1) smin = smax = min(split_k, kb_total);
  else if (accumulate && split_k < 0) smax = max(1, min(64, kb_total / 4));
  const int bm_max = (tc_debug() & 512) ? 128 : 256;
  double best_cost = 1e300;
  for (int bm = 128; bm <= bm_max; bm *= 2) {
    for (int s = smin; s <= smax; ++s) {
      const int kbs = ceil_div(kb_total, s), splits = ceil_div(kb_total, kbs);    // as launched: no empty split
      const int64_t ctas = (int64_t)ceil_div(M, bm) * ceil_div(N, best.bn) * splits;
      const double area = (double)bm * best.bn / (128.0 * 128.0);
      const double cost = (double)ceil_div(ctas, (int64_t)sms) * (TC_CTA_FIXED + (kbs + TC_CTA_STORE) * area) * (1.0 + 0.03 * splits);
      if (cost < best_cost - 1e-9) { best_cost = cost; best.bm = bm; best.splits = splits; }
    }
  }
  return best;
}

// ---------------------------------------------------------------------------------------------------------
// Operand-plane registry: fp32 buffers whose TF32 hi/lo planes are kept next to them so that a tensor is split at
// most once (by the epilogue of the GEMM that produced it, or by one prep pass on first use) no matter how many
// GEMMs consume it, in either major-ness.  Host-side bookkeeping in stream-issue order (single stream).
// ---------------------------------------------------------------------------------------------------------
PlaneBuf* PlaneRegistry::find(const float* p) {
  for (int i = 0; i < n; ++i)
    if (p >= b[i].base && p < b[i].base + b[i].capacity) return &b[i];
  return nullptr;
}
void PlaneRegistry::add(const float* base, int64_t capacity, float* hi, float* lo, int64_t plane_capacity) {
  if (n >= MAX) return;
  PlaneBuf& x = b[n++];
  x.base = base; x.capacity = capacity; x.hi = hi; x.lo = lo; x.plane_capacity = plane_capacity;
  x.ld = 0; x.rows = x.cols = 0; x.ldp = 0; x.scale_ptr = nullptr; x.drop();
}
PlaneBuf* PlaneRegistry::declare(const float* base, int64_t ld, int rows, int cols) {
  PlaneBuf* x = find(base);
  if (!x || x->base != base) return nullptr;
  x->drop();
  const int64_t ldp = f16 ? (cols + 7) / 8 * 8 : (cols + 3) / 4 * 4;
  if ((int64_t)rows * ldp > (f16 ? 2 : 1) * x->plane_capacity) return nullptr;
  x->ld = ld; x->rows = rows; x->cols = cols; x->ldp = ldp; x->valid = true;
  if (f16) { x->is_static = true; x->scale_ptr = static_scale; }
  return x;
}
void* PlaneRegistry::plane(const PlaneBuf* x, bool lo, int64_t r0, int64_t c0) const {
  float* p = lo ? x->lo : x->hi;
  const int64_t off = r0 * x->ldp + c0;
  return f16 ? (void*)((__half*)p + off) : (void*)(p + off);
}
void PlaneRegistry::invalidate(const float* p) { if (PlaneBuf* x = find(p)) x->drop(); }
void PlaneRegistry::invalidate_range(const float* lo_, const float* hi_) {
  for (int i = 0; i < n; ++i) if (b[i].base >= lo_ && b[i].base < hi_) b[i].drop();
}
int PlaneRegistry::begin_call(cudaStream_t st, int base) {
  call_base = base; gemm_index = 0;
  if (!f16) return ASE_OK;
  if (reset_pending) {      // new parameters: every scale is re-derived exactly on this call, nothing is compared with the old ones
    ASE_CUDA_OK(cudaMemsetAsync(amax, 0, (size_t)SITES * 12, st));      // amax[SITES] + scale[SITES][2] are contiguous
    reset_pending = false;
  }
  for (int i = 0; i < SITES; ++i) { if (touched[i]) { known[i] = true; touched[i] = false; } }
  for (int i = 0; i < n; ++i) {
    b[i].amax_site = -1;                                 // maxima tracked by GEMM epilogues are only meaningful within one call
    // planes written by a GEMM epilogue refer to their site's scale slot, which is re-predicted right now: drop them
    // (planes split by a prep pass -- the weights -- carry their own copy of the scale and stay valid)
    if (b[i].valid && !b[i].is_static && b[i].scale_ptr >= scale && b[i].scale_ptr < scale + 2 * SITES) b[i].valid = false;
    if (b[i].is_static) { b[i].valid = false; b[i].is_static = false; }
  }
  tc_site_update_kernel<<<ceil_div(SITES, 256), 256, 0, st>>>(amax, scale, SITES, static_scale, STATIC_SCALE, flag);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

// (Re)split every listed weight tensor [rows, cols] (contiguous) into its registered planes: one launch (two on the first call
// after the parameters were announced: exact maxima first).  Sites are fixed per tensor (WEIGHT_SITE0 + i).
int PlaneRegistry::prep_weights(const float* const* src, const int* rows, const int* cols, int count, cudaStream_t st) {
  if (!f16 || count <= 0) return ASE_OK;
  TcPrepBatch batch; int nb = 0; bool all_known = true;
  for (int i = 0; i < count && nb < TcPrepBatch::MAX; ++i) {
    PlaneBuf* x = find(src[i]);
    if (!x || x->base != src[i]) continue;
    const int64_t ldp = (cols[i] + 7) / 8 * 8;
    if ((int64_t)rows[i] * ldp > 2 * x->plane_capacity) continue;
    const int site = WEIGHT_SITE0 + i;
    if (site >= SITES) break;
    x->ld = cols[i]; x->rows = rows[i]; x->cols = cols[i]; x->ldp = ldp; x->valid = true; x->is_static = false; x->amax_site = -1; x->fp32_stale = false;
    x->scale_ptr = bscale + 2 * (x - b);
    batch.item[nb++] = {src[i], cols[i], rows[i], cols[i], rows[i], (int)ldp, x->hi, x->lo, amax + site, scale + 2 * site, bscale + 2 * (x - b)};
    all_known = all_known && known[site];
    touched[site] = true;
  }
  if (nb == 0) return ASE_OK;
  dim3 grid(48, nb);      // 28 MB of weights per optimizer step: 48 slices x 16 tensors keep every SM several blocks deep
  if (!all_known) {
    tc_amax_kernel<<<grid, 256, 0, st>>>(batch);
    ASE_LAUNCH_OK();
  }
  tc_split_h_kernel<<<grid, 256, 0, st>>>(batch, all_known ? 0 : 1, TOP_SITE, flag);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

struct OpView { const void* hi; const void* lo; int64_t ldp; bool ok; const float* scale; };

// View [nat_rows, nat_cols] (ld) at `ptr` as planes.  Geometry of a registered buffer is whatever its last full
// writer declared; a first read of a buffer without valid planes splits the WHOLE declared buffer once.
// site: this reader's scale site (FP16 format; used when the buffer's max is not already tracked at its producer's site).
static int resolve_operand(PlaneRegistry* reg, const float* ptr, int64_t ld, int nat_rows, int nat_cols, OpView* v, int site, cudaStream_t st) {
  v->ok = false; v->scale = nullptr;
  if (!reg) return ASE_OK;
  PlaneBuf* x = reg->find(ptr);
  if (!x) return ASE_OK;
  const bool H = reg->f16;
  const int pal = H ? 8 : 4;                 // plane leading dimensions / column offsets: 16-byte granules
  if (!x->valid) {
    if (x->fp32_stale) { set_error("wgmma GEMM: a planes-only tensor lost its planes before it was consumed"); return ASE_ERR_INVALID; }
    // adopt the reader's geometry if it starts at the buffer base (inputs written by non-GEMM kernels, weights)
    if (ptr != x->base) return ASE_OK;
    if (!H) {
      const int64_t ldp = pad_to(nat_cols, 4);
      if ((int64_t)nat_rows * ldp > x->plane_capacity || (int64_t)(nat_rows - 1) * ld + nat_cols > x->capacity) return ASE_OK;
      x->ld = ld; x->rows = nat_rows; x->cols = nat_cols; x->ldp = ldp;
      const int64_t total = (int64_t)nat_rows * ldp;
      tc_prep_kernel<<<(int)imin64((total + 255) / 256, NUM_SMS * 16), 256, 0, st>>>(ptr, ld, nat_rows, nat_cols, nat_rows, (int)ldp, x->hi, x->lo);
      ASE_LAUNCH_OK();
    } else {
      int rc;
      float* bs = reg->bscale + 2 * (x - reg->b);      // the buffer's own copy of the scale: survives the next begin_call
      if (x->amax_site >= 0) {
        // written earlier in this call by a GEMM whose scale was not known yet: it declared the geometry and tracked max |C|
        const int ts = x->amax_site;
        x->ldp = pad_to(x->cols, 8);
        const TcPrepItem it{ptr, x->ld, x->rows, x->cols, x->rows, (int)x->ldp, x->hi, x->lo, reg->amax + ts, reg->scale + 2 * ts, bs};
        if ((rc = materialize_h(it, false, true, nullptr, TOP_SITE, st))) return rc;
      } else {
        // written by a non-GEMM kernel (or accumulated into): split the reader's view with this reader's site
        const int64_t ldp = pad_to(nat_cols, 8);
        if (site < 0 || (int64_t)nat_rows * ldp > 2 * x->plane_capacity || (int64_t)(nat_rows - 1) * ld + nat_cols > x->capacity) return ASE_OK;
        x->ld = ld; x->rows = nat_rows; x->cols = nat_cols; x->ldp = ldp;
        const TcPrepItem it{ptr, ld, nat_rows, nat_cols, nat_rows, (int)ldp, x->hi, x->lo, reg->amax + site, reg->scale + 2 * site, bs};
        if ((rc = materialize_h(it, reg->known[site], false, reg->flag, TOP_SITE, st))) return rc;
        reg->touched[site] = true;
      }
      x->scale_ptr = bs; x->is_static = false;
    }
    x->valid = true;
  }
  if (ld != x->ld) return ASE_OK;
  const int64_t off = ptr - x->base;
  const int64_t r0 = off / x->ld, c0 = off - r0 * x->ld;
  if ((c0 & (pal - 1)) || r0 + nat_rows > x->rows || c0 + nat_cols > x->cols) return ASE_OK;
  v->hi = reg->plane(x, false, r0, c0); v->lo = reg->plane(x, true, r0, c0);
  if (H) v->scale = x->scale_ptr;
  v->ldp = x->ldp; v->ok = true;
  return ASE_OK;
}

int gemm_tc(const AseGemmParams& p, cudaStream_t st, PlaneRegistry* reg) {
  const bool H = p.backend == 2;             // scaled FP16 hi/lo planes instead of TF32 ones
  if (reg && reg->f16 != H) { set_error("wgmma GEMM: plane registry format does not match backend %d", p.backend); return ASE_ERR_INVALID; }
  const int BK = H ? TcFmt<true>::BK : TcFmt<false>::BK;
  const TcPlan plan = gemm_tc_plan(p.M, p.N, p.K, p.accumulate, p.split_k, NUM_SMS, H);
  const int BN = plan.bn;
  const int a_box = plan.bm;
  // workspace planes: whole tiles of rows (one tile height, 256, for every plan), K to 128 bytes (the prep kernels' granularity)
  const int Mp = pad_to(p.M, TC_MPAD), Np = pad_to(p.N, 128), Kp = pad_to(p.K, H ? 2 * TC_KPAD : TC_KPAD);
  int rc;
  // ---- operands: cached planes when the buffer is registered, else a split pass into the shared workspace
  OpView va, vb;
  const int a_rows = p.a_trans ? p.K : p.M, a_cols = p.a_trans ? p.M : p.K;
  const int b_rows = p.b_trans ? p.K : p.N, b_cols = p.b_trans ? p.N : p.K;
  // FP16 format: scale sites of this GEMM (A, B, C); without a registry the workspace head holds two transient slots
  const int site_a = (H && reg) ? reg->site(0) : -1, site_b = (H && reg) ? reg->site(1) : -1, site_c = (H && reg) ? reg->site(2) : -1;
  if (H && reg) { if (site_c < 0) { set_error("wgmma FP16 GEMM: more GEMMs in one call than scale sites"); return ASE_ERR_WORKSPACE; } reg->gemm_index++; }
  // TF32 planes are only read K-major: an operand stored [K, rows] is split transposed into the workspace instead
  if ((rc = resolve_operand((H || !p.a_trans) ? reg : nullptr, p.A, p.lda, a_rows, a_cols, &va, site_a, st))) return rc;
  if ((rc = resolve_operand((H || !p.b_trans) ? reg : nullptr, p.B, p.ldb, b_rows, b_cols, &vb, site_b, st))) return rc;
  if (reg) {      // a planes-only tensor (fp32 store elided) can only be consumed through its planes / activity bits: anything else is a bug, not a fallback
    auto stale = [&](const float* ptr) { PlaneBuf* x = ptr ? reg->find(ptr) : nullptr; return x && x->fp32_stale; };
    if ((!va.ok && stale(p.A)) || (!vb.ok && stale(p.B)) || (p.mask_src && p.mask_mode && !(p.mask_mode == 1 && p.mask_bits) && stale(p.mask_src))) {
      set_error("wgmma GEMM %dx%dx%d: an operand's fp32 copy was elided (c_planes_only) but it is not consumed through its planes", p.M, p.N, p.K);
      return ASE_ERR_INVALID;
    }
  }
  CUtensorMap ah, al, bh, bl;
  char* ws = (char*)p.workspace;
  if (!va.ok || !vb.ok) { if ((rc = gemm_tc_check_workspace(p))) return rc; }
  unsigned* t_amax[2] = {nullptr, nullptr}; float* t_scale[2] = {nullptr, nullptr}; bool t_pred[2] = {false, false};
  if (H && (!va.ok || !vb.ok)) {
    if (reg) {
      const int sites[2] = {site_a, site_b};
      for (int i = 0; i < 2; ++i) {
        if (i == 0 ? va.ok : vb.ok) continue;
        t_amax[i] = reg->amax + sites[i]; t_scale[i] = reg->scale + 2 * sites[i]; t_pred[i] = reg->known[sites[i]]; reg->touched[sites[i]] = true;
      }
    } else {
      ASE_CUDA_OK(cudaMemsetAsync(ws, 0, 2 * sizeof(unsigned), st));
      t_amax[0] = (unsigned*)ws; t_amax[1] = (unsigned*)ws + 1; t_scale[0] = (float*)(ws + 16); t_scale[1] = (float*)(ws + 32);
    }
  }
  unsigned* oflag = (H && reg) ? reg->flag : nullptr;
  char* wsp = ws + TC_WS_HEAD;
  // plane slots of the workspace layout.  (They used to be placed at Mp x Kp fp32 words with the FP16 format's K padding to 64,
  // which for K % 64 in (0, 32] reached past the workspace the caller sized with gemm_tc_workspace_bytes.)
  const TcWsSlots slots = tc_ws_slots(p.M, p.N, p.K);
  if (va.ok) {
    // TRUE extents over a (sub-)view of the planes: TMA zero-fills everything outside [a_rows, a_cols]
    if ((rc = encode_cached(&ah, va.hi, a_rows, a_cols, va.ldp, p.a_trans ? BK : a_box, p.a_trans != 0, H)) ||
        (rc = encode_cached(&al, va.lo, a_rows, a_cols, va.ldp, p.a_trans ? BK : a_box, p.a_trans != 0, H))) return rc;
  } else {
    float* Ahi = (float*)wsp; float* Alo = (float*)(wsp + slots.a);
    if (!H) { if ((rc = prep_operand(p.A, p.lda, p.a_trans, p.M, p.K, Mp, Kp, Ahi, Alo, st))) return rc; }
    else {
      const TcPrepItem it{p.A, p.lda, a_rows, a_cols, p.a_trans ? Kp : Mp, p.a_trans ? Mp : Kp, Ahi, Alo, t_amax[0], t_scale[0], nullptr};
      if ((rc = materialize_h(it, t_pred[0], false, oflag, reg ? TOP_SITE : TOP_EXACT, st))) return rc;
      va.scale = t_scale[0];
    }
    if (!p.a_trans || !H) { if ((rc = encode_cached(&ah, Ahi, Mp, Kp, Kp, a_box, false, H)) || (rc = encode_cached(&al, Alo, Mp, Kp, Kp, a_box, false, H))) return rc; }
    else            { if ((rc = encode_cached(&ah, Ahi, Kp, Mp, Mp, BK, true, H)) || (rc = encode_cached(&al, Alo, Kp, Mp, Mp, BK, true, H))) return rc; }
  }
  if (vb.ok) {
    if ((rc = encode_cached(&bh, vb.hi, b_rows, b_cols, vb.ldp, p.b_trans ? BK : BN, p.b_trans != 0, H)) ||
        (rc = encode_cached(&bl, vb.lo, b_rows, b_cols, vb.ldp, p.b_trans ? BK : BN, p.b_trans != 0, H))) return rc;
  } else {
    char* wb = wsp + 2 * slots.a;
    float* Bhi = (float*)wb; float* Blo = (float*)(wb + slots.b);
    if (!H) { if ((rc = prep_operand(p.B, p.ldb, p.b_trans, p.N, p.K, Np, Kp, Bhi, Blo, st))) return rc; }
    else {
      const TcPrepItem it{p.B, p.ldb, b_rows, b_cols, p.b_trans ? Kp : Np, p.b_trans ? Np : Kp, Bhi, Blo, t_amax[1], t_scale[1], nullptr};
      if ((rc = materialize_h(it, t_pred[1], false, oflag, reg ? TOP_SITE : TOP_EXACT, st))) return rc;
      vb.scale = t_scale[1];
    }
    if (!p.b_trans || !H) { if ((rc = encode_cached(&bh, Bhi, Np, Kp, Kp, BN, false, H)) || (rc = encode_cached(&bl, Blo, Np, Kp, Kp, BN, false, H))) return rc; }
    else            { if ((rc = encode_cached(&bh, Bhi, Kp, Np, Np, BK, true, H)) || (rc = encode_cached(&bl, Blo, Kp, Np, Np, BK, true, H))) return rc; }
  }
  TcEpi e;
  e.C = p.C; e.ldc = p.ldc; e.M = p.M; e.N = p.N; e.K = p.K; e.alpha = p.alpha; e.bias = p.bias; e.act = p.act;
  e.mask_src = p.mask_src; e.ldm = p.ldm; e.mask_mode = p.mask_src ? p.mask_mode : 0; e.accumulate = p.accumulate;
  e.Chi = e.Clo = nullptr; e.ldp = 0; e.colsum = p.colsum_out;
  e.a_inv = (H && va.scale) ? va.scale + 1 : nullptr; e.b_inv = (H && vb.scale) ? vb.scale + 1 : nullptr;
  e.c_scale = nullptr; e.c_amax = nullptr; e.flag = nullptr;
  e.relu_bits = p.relu_bits_out; e.ldrb = p.ldrb; e.mask_bits = (e.mask_mode == 1) ? p.mask_bits : nullptr; e.ldmb = p.ldmb; e.skip_c = 0;
  // ---- output planes: a full write at the base of a registered buffer (re)declares its geometry; a partial write
  // keeps planes in sync only if they are currently valid with the same leading dimension; accumulation invalidates
  if (reg && !H) {
    if (PlaneBuf* x = reg->find(p.C)) {
      if (p.accumulate) x->valid = false;
      else if (p.C == x->base && (int64_t)p.M * pad_to(p.N, 4) <= x->plane_capacity && !(x->valid && x->ld == p.ldc && (x->rows > p.M || x->cols > p.N))) {
        x->ld = p.ldc; x->rows = p.M; x->cols = p.N; x->ldp = pad_to(p.N, 4); x->valid = true;
        e.Chi = x->hi; e.Clo = x->lo; e.ldp = x->ldp;
      } else if (x->valid && x->ld == p.ldc) {
        const int64_t off = p.C - x->base, r0 = off / x->ld, c0 = off - r0 * x->ld;
        if (r0 + p.M <= x->rows && c0 + p.N <= x->cols) { e.Chi = x->hi + r0 * x->ldp + c0; e.Clo = x->lo + r0 * x->ldp + c0; e.ldp = x->ldp; }
        else x->valid = false;
      } else x->valid = false;
    }
  } else if (reg && H) {
    // FP16 format.  A full write at the buffer base: the epilogue tracks max |C| at this GEMM's C site; if the site's scale is
    // already known (predicted from the previous call) it also writes the planes, else the first consumer splits with the exact
    // scale.  A tanh-bounded partial write into statically scaled planes (the style columns behind the normalised
    // observations) keeps them in sync.  Anything else leaves the buffer without planes.
    if (PlaneBuf* x = reg->find(p.C)) {
      if (x->fp32_stale && p.accumulate) { set_error("wgmma GEMM: accumulating into a planes-only tensor"); return ASE_ERR_INVALID; }
      x->fp32_stale = false;
      const bool full = !p.accumulate && p.C == x->base && (int64_t)p.M * pad_to(p.N, 8) <= 2 * x->plane_capacity && (int64_t)(p.M - 1) * p.ldc + p.N <= x->capacity &&
                        !(x->valid && x->is_static && x->ld == p.ldc && (x->rows > p.M || x->cols > p.N));
      if (full) {
        x->ld = p.ldc; x->rows = p.M; x->cols = p.N; x->ldp = pad_to(p.N, 8); x->is_static = false;
        reg->touched[site_c] = true; e.c_amax = reg->amax + site_c;
        if (reg->known[site_c]) {
          x->valid = true; x->amax_site = -1; x->scale_ptr = reg->scale + 2 * site_c;
          e.Chi = x->hi; e.Clo = x->lo; e.ldp = x->ldp; e.c_scale = x->scale_ptr; e.flag = reg->flag;
          if (p.c_planes_only) { e.skip_c = 1; x->fp32_stale = true; }
        } else { x->valid = false; x->amax_site = site_c; }
      } else if (!p.accumulate && x->valid && x->is_static && x->ld == p.ldc && p.act == 2 && !p.mask_src) {
        const int64_t off = p.C - x->base, r0 = off / x->ld, c0 = off - r0 * x->ld;
        if (r0 + p.M <= x->rows && c0 + p.N <= x->cols) { e.Chi = reg->plane(x, false, r0, c0); e.Clo = reg->plane(x, true, r0, c0); e.ldp = x->ldp; e.c_scale = x->scale_ptr; e.flag = reg->flag; }
        else x->drop();
      } else x->drop();
    }
  }
  e.kb_total = ceil_div(p.K, BK);
  e.debug = tc_debug();
  e.kb_per_split = ceil_div(e.kb_total, plan.splits);
  const int splits = ceil_div(e.kb_total, e.kb_per_split);
  const bool amn = H && p.a_trans, bmn = H && p.b_trans;
  // Launches whose every tile takes the fragment store phase (whole tiles in M and N, aligned operands, FP16 planes, BN = 128,
  // no accumulation) run the persistent kernel: the same tiles and arithmetic, one CTA per SM looping over them
  const bool persist = H && BN == 128 && !(e.debug & (256 | 1024)) && p.M % plan.bm == 0 && p.N % BN == 0 &&
                       epilogue_frag_ok(e, 0, 0, plan.bm, BN, H);
  if (persist) return plan.bm == 256 ? launch_tc_major<256, 128, true, true>(amn, bmn, ah, al, bh, bl, e, splits, st)
                                     : launch_tc_major<128, 128, true, true>(amn, bmn, ah, al, bh, bl, e, splits, st);
  if (H) {
    if (plan.bm == 256) return BN == 128 ? launch_tc_major<256, 128, true>(amn, bmn, ah, al, bh, bl, e, splits, st)
                                         : launch_tc_major<256, 64, true>(amn, bmn, ah, al, bh, bl, e, splits, st);
    return BN == 128 ? launch_tc_major<128, 128, true>(amn, bmn, ah, al, bh, bl, e, splits, st)
                     : launch_tc_major<128, 64, true>(amn, bmn, ah, al, bh, bl, e, splits, st);
  }
  if (plan.bm == 256) return BN == 128 ? launch_tc_major<256, 128, false>(amn, bmn, ah, al, bh, bl, e, splits, st)
                                       : launch_tc_major<256, 64, false>(amn, bmn, ah, al, bh, bl, e, splits, st);
  return BN == 128 ? launch_tc_major<128, 128, false>(amn, bmn, ah, al, bh, bl, e, splits, st)
                   : launch_tc_major<128, 64, false>(amn, bmn, ah, al, bh, bl, e, splits, st);
}

}  // namespace ase

extern "C" int ase_gemm_tc_plan(int M, int N, int K, int accumulate, int split_k, int backend, int* tile_m, int* tile_n, int* splits) {
  using namespace ase;
  if (M < 1 || N < 1 || K < 1 || (backend != 1 && backend != 2)) { set_error("ase_gemm_tc_plan: bad shape or backend"); return ASE_ERR_INVALID; }
  const TcPlan p = gemm_tc_plan(M, N, K, accumulate, split_k, NUM_SMS, backend == 2);
  if (tile_m) *tile_m = p.bm;
  if (tile_n) *tile_n = p.bn;
  if (splits) *splits = p.splits;
  return ASE_OK;
}

extern "C" int ase_gemm_tc_profile(int enable) {
  ase::g_prof.on = enable != 0;
  ase::g_prof.used = 0;
  ase::g_prof.flops = 0.0;
  return ASE_OK;
}

extern "C" int ase_gemm_tc_profile_read(double* total_ms, int64_t* launches, double* flops) {
  using namespace ase;
  double tot = 0.0;
  const size_t n = g_prof.used / 2;
  for (size_t i = 0; i < n; ++i) {
    float ms = 0.0f;
    ASE_CUDA_OK(cudaEventSynchronize(g_prof.ev[2 * i + 1]));
    ASE_CUDA_OK(cudaEventElapsedTime(&ms, g_prof.ev[2 * i], g_prof.ev[2 * i + 1]));
    tot += ms;
  }
  if (total_ms) *total_ms = tot;
  if (launches) *launches = (int64_t)n;
  if (flops) *flops = g_prof.flops;
  return ASE_OK;
}
