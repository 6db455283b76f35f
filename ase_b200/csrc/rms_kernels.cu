// RunningMeanStd (rl_games 1.1.4 algos_torch/running_mean_std.py): fp64 running moments, fp32 data.
// Column statistics are accumulated in fp64 (threads map to columns => coalesced row reads), merged with
// the parallel-Welford rule of the reference, and the normalise/clamp pass uses the UPDATED statistics
// exactly as the reference's train-mode forward does.  Up to 3 batches can be merged sequentially in one
// launch (the three AMP batches of calc_gradients, ase_agent.py:170-181).
#include "common.cuh"
#include "kernels.h"
#include "tc_common.cuh"

namespace ase {

constexpr int RMS_COLS_PER_BLOCK = 128;
constexpr int RMS_ROWS_PER_BLOCK = 64;

// partial[(batch*chunks + chunk)*cols + col] = (sum, sumsq) over the chunk's rows
__global__ void __launch_bounds__(RMS_COLS_PER_BLOCK)
rms_colstats_kernel(RmsBatchList bl, int cols, int chunks, double2* __restrict__ partial) {
  const int col = blockIdx.x * RMS_COLS_PER_BLOCK + threadIdx.x;
  const int chunk = blockIdx.y, batch = blockIdx.z;
  if (col >= cols) return;
  const float* x = bl.x[batch];
  const int64_t ld = bl.ld[batch];
  const int rows = bl.rows;
  const int r0 = chunk * RMS_ROWS_PER_BLOCK, r1 = min(rows, r0 + RMS_ROWS_PER_BLOCK);
  double s = 0.0, ss = 0.0;
#pragma unroll 4
  for (int r = r0; r < r1; ++r) {
    const double v = (double)x[(int64_t)r * ld + col];
    s += v; ss += v * v;
  }
  partial[((int64_t)batch * chunks + chunk) * cols + col] = make_double2(s, ss);
}

// Reduce the chunk partials, merge batch after batch, emit fp32 mean / std per batch.  Block = 32 columns x 8 chunk lanes: the
// chunk sums of a column are split over 8 threads (coalesced along the columns) and meet in shared memory; lane 0 does the merge.
__global__ void __launch_bounds__(256)
rms_finalize_kernel(const double2* __restrict__ partial, int cols, int chunks, int nbatch, int rows,
                    double* __restrict__ mean, double* __restrict__ var, const double* __restrict__ count,
                    float eps, float* __restrict__ meanf, float* __restrict__ stdf, int update) {
  __shared__ double ssum[8][33], ssq[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + tx;
  const bool ok = col < cols;
  double m = 0.0, v = 0.0, c = 0.0;
  if (ok && ty == 0) { m = mean[col]; v = var[col]; c = count[0]; }
  for (int b = 0; b < nbatch; ++b) {
    if (update) {
      double s = 0.0, ss = 0.0;
      if (ok) for (int k = ty; k < chunks; k += 8) {
        const double2 p = partial[((int64_t)b * chunks + k) * cols + col];
        s += p.x; ss += p.y;
      }
      ssum[ty][tx] = s; ssq[ty][tx] = ss;
      __syncthreads();
      if (ok && ty == 0) {
        s = 0.0; ss = 0.0;
#pragma unroll
        for (int k = 0; k < 8; ++k) { s += ssum[k][tx]; ss += ssq[k][tx]; }
        const double n = (double)rows;
        // the reference's batch moments are fp32 tensors (input.mean(0), input.var(0)): round like it does
        const double bm = (double)(float)(s / n);
        double bvar = (ss - s * s / n) / (n - 1.0);
        if (bvar < 0.0) bvar = 0.0;
        bvar = (double)(float)bvar;
        const double delta = bm - m, tot = c + n;
        const double m2 = v * c + bvar * n + delta * delta * c * n / tot;
        m = m + delta * n / tot;
        v = m2 / tot;
        c = tot;
      }
      __syncthreads();
    }
    if (ok && ty == 0) {
      meanf[b * cols + col] = (float)m;
      stdf[b * cols + col] = sqrtf((float)v + eps);
    }
  }
  if (update && ok && ty == 0) { mean[col] = m; var[col] = v; }
}

__global__ void rms_count_add_kernel(double* count, double inc) { count[0] += inc; }

// y = clamp((x-mean)/std, -5, 5) written to up to 3 destinations (unnorm: std*clamp(x,+-5)+mean).
// Threads map to columns (coalesced rows, the column's mean / std loaded once), blockIdx.y walks chunks of rows.
constexpr int NORM_ROWS_PER_BLOCK = 8;       // few rows per thread, all loads in flight at once: the pass is latency-bound otherwise
__global__ void __launch_bounds__(128)
rms_normalize_kernel(const float* __restrict__ x, int64_t ldx, int rows, int cols,
                     const float* __restrict__ meanf, const float* __restrict__ stdf, int unnorm, RmsDst dst) {
  const int c = blockIdx.x * 128 + threadIdx.x;
  if (c >= cols) return;
  const float mu = meanf[c], sd = stdf[c];
  const bool planes = dst.hi[0] || dst.hi[1] || dst.hi[2];
  const int r0 = blockIdx.y * NORM_ROWS_PER_BLOCK;
  float xv[NORM_ROWS_PER_BLOCK];
#pragma unroll
  for (int i = 0; i < NORM_ROWS_PER_BLOCK; ++i) xv[i] = (r0 + i < rows) ? x[(int64_t)(r0 + i) * ldx + c] : 0.0f;
#pragma unroll
  for (int i = 0; i < NORM_ROWS_PER_BLOCK; ++i) {
    const int r = r0 + i;
    if (r >= rows) break;
    const float v = xv[i];
    float y;
    if (unnorm) y = sd * fminf(fmaxf(v, -5.0f), 5.0f) + mu;
    else y = fminf(fmaxf((v - mu) / sd, -5.0f), 5.0f);
    float h = 0.0f, l = 0.0f;
    __half hh = __float2half_rn(0.0f), hl = hh;
    if (planes) {
      if (!dst.half) split_tf32(y, h, l);
      else split_f16(y * dst.pscale, hh, hl);
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      if (dst.y[d]) dst.y[d][(int64_t)r * dst.ld[d] + c] = y;
      if (dst.hi[d]) {
        const int64_t o = (int64_t)r * dst.ldp[d] + c;
        if (!dst.half) { ((float*)dst.hi[d])[o] = h; ((float*)dst.lo[d])[o] = l; }
        else { ((__half*)dst.hi[d])[o] = hh; ((__half*)dst.lo[d])[o] = hl; }
      }
    }
  }
}

// 4 columns x NORM_ROWS_PER_BLOCK rows per thread: 16-byte loads / fp32 stores and 8-byte half-plane stores (cols, every leading dimension a
// multiple of 4 and 16-byte aligned bases: the 1400-wide AMP observations; the 253-wide observations take the scalar kernel above).
// Same arithmetic per element as rms_normalize_kernel.
__global__ void __launch_bounds__(128)
rms_normalize_vec4_kernel(const float* __restrict__ x, int64_t ldx, int rows, int cols,
                          const float* __restrict__ meanf, const float* __restrict__ stdf, int unnorm, RmsDst dst) {
  const int c = (blockIdx.x * 128 + threadIdx.x) * 4;
  if (c >= cols) return;
  const float4 mu = *reinterpret_cast<const float4*>(meanf + c), sd = *reinterpret_cast<const float4*>(stdf + c);
  const bool planes = dst.hi[0] || dst.hi[1] || dst.hi[2];
  const int r0 = blockIdx.y * NORM_ROWS_PER_BLOCK;
  float4 xv[NORM_ROWS_PER_BLOCK];
#pragma unroll
  for (int i = 0; i < NORM_ROWS_PER_BLOCK; ++i)
    xv[i] = (r0 + i < rows) ? __ldcs(reinterpret_cast<const float4*>(x + (int64_t)(r0 + i) * ldx + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int i = 0; i < NORM_ROWS_PER_BLOCK; ++i) {
    const int r = r0 + i;
    if (r >= rows) break;
    const float v[4] = {xv[i].x, xv[i].y, xv[i].z, xv[i].w};
    const float m4[4] = {mu.x, mu.y, mu.z, mu.w}, s4[4] = {sd.x, sd.y, sd.z, sd.w};
    float y[4], h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (unnorm) y[j] = s4[j] * fminf(fmaxf(v[j], -5.0f), 5.0f) + m4[j];
      else y[j] = fminf(fmaxf((v[j] - m4[j]) / s4[j], -5.0f), 5.0f);
      h[j] = l[j] = 0.0f;
      if (planes && !dst.half) split_tf32(y[j], h[j], l[j]);
    }
    uint2 hv = make_uint2(0u, 0u), lv = hv;
    if (planes && dst.half) {
      split_f16x2(y[0] * dst.pscale, y[1] * dst.pscale, hv.x, lv.x);
      split_f16x2(y[2] * dst.pscale, y[3] * dst.pscale, hv.y, lv.y);
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      if (dst.y[d]) *reinterpret_cast<float4*>(dst.y[d] + (int64_t)r * dst.ld[d] + c) = make_float4(y[0], y[1], y[2], y[3]);
      if (dst.hi[d]) {
        const int64_t o = (int64_t)r * dst.ldp[d] + c;
        if (!dst.half) {
          *reinterpret_cast<float4*>((float*)dst.hi[d] + o) = make_float4(h[0], h[1], h[2], h[3]);
          *reinterpret_cast<float4*>((float*)dst.lo[d] + o) = make_float4(l[0], l[1], l[2], l[3]);
        } else {
          *reinterpret_cast<uint2*>((__half*)dst.hi[d] + o) = hv;
          *reinterpret_cast<uint2*>((__half*)dst.lo[d] + o) = lv;
        }
      }
    }
  }
}

// just copy columns (used to place latents next to the normalised observations)
__global__ void __launch_bounds__(256)
copy_cols_kernel(const float* __restrict__ x, int64_t ldx, int rows, int cols, float* __restrict__ y, int64_t ldy,
                 void* __restrict__ hi, void* __restrict__ lo, int64_t ldp, int half, float pscale, unsigned* __restrict__ flag) {
  const int64_t total = (int64_t)rows * cols;
  float m = 0.0f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / cols), c = (int)(i - (int64_t)r * cols);
    const float v = x[(int64_t)r * ldx + c];
    y[(int64_t)r * ldy + c] = v;
    if (hi) {
      const int64_t o = (int64_t)r * ldp + c;
      if (!half) { float h, l; split_tf32(v, h, l); ((float*)hi)[o] = h; ((float*)lo)[o] = l; }
      else { __half h, l; split_f16(v * pscale, h, l); ((__half*)hi)[o] = h; ((__half*)lo)[o] = l; m = fmaxf(m, fabsf(v)); }
    }
  }
  // the static plane scale assumes bounded inputs (unit latents): report instead of saturating silently
  if (hi && half) report_scale_miss(m, pscale, nullptr, flag);
}

int64_t rms_scratch_bytes(int cols, int rows, int nbatch) {
  const int chunks = ceil_div(rows, RMS_ROWS_PER_BLOCK);
  return align_up((int64_t)nbatch * chunks * cols * sizeof(double2), 256) + align_up((int64_t)2 * nbatch * cols * sizeof(float), 256);
}

// Merge `nbatch` batches sequentially into (mean,var,count); meanf/stdf[b] are the fp32 stats valid after batch b.
int rms_update_batches(const RmsBatchList& bl, int nbatch, int cols, double* mean, double* var, double* count, float eps,
                       int update, void* scratch, float** meanf_out, float** stdf_out, cudaStream_t st) {
  const int rows = bl.rows;
  const int chunks = ceil_div(rows, RMS_ROWS_PER_BLOCK);
  double2* partial = (double2*)scratch;
  float* meanf = (float*)((char*)scratch + align_up((int64_t)nbatch * chunks * cols * sizeof(double2), 256));
  float* stdf = meanf + (int64_t)nbatch * cols;
  if (update) {
    ASE_CHECK_ARG(rows >= 2, "RunningMeanStd update needs >= 2 rows (unbiased variance)");
    dim3 grid(ceil_div(cols, RMS_COLS_PER_BLOCK), chunks, nbatch);
    rms_colstats_kernel<<<grid, RMS_COLS_PER_BLOCK, 0, st>>>(bl, cols, chunks, partial);
    ASE_LAUNCH_OK();
  }
  rms_finalize_kernel<<<ceil_div(cols, 32), 256, 0, st>>>(partial, cols, chunks, nbatch, rows, mean, var, count, eps, meanf, stdf, update);
  ASE_LAUNCH_OK();
  if (update) {
    rms_count_add_kernel<<<1, 1, 0, st>>>(count, (double)rows * nbatch);
    ASE_LAUNCH_OK();
  }
  *meanf_out = meanf; *stdf_out = stdf;
  return ASE_OK;
}

int rms_normalize(const float* x, int64_t ldx, int rows, int cols, const float* meanf, const float* stdf, int unnorm,
                  const RmsDst& dst, cudaStream_t st) {
  if (rows <= 0 || cols <= 0) return ASE_OK;
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  bool vec = (cols % 4 == 0) && (ldx % 4 == 0) && al16(x) && al16(meanf) && al16(stdf);
  for (int d = 0; d < 3 && vec; ++d) {
    if (dst.y[d]) vec = vec && al16(dst.y[d]) && (dst.ld[d] % 4 == 0);
    if (dst.hi[d]) vec = vec && (dst.ldp[d] % 4 == 0) && (dst.half ? ((reinterpret_cast<uintptr_t>(dst.hi[d]) | reinterpret_cast<uintptr_t>(dst.lo[d])) & 7) == 0
                                                                  : (al16(dst.hi[d]) && al16(dst.lo[d])));
  }
  if (vec) {
    dim3 grid(ceil_div(cols / 4, 128), ceil_div(rows, NORM_ROWS_PER_BLOCK));
    rms_normalize_vec4_kernel<<<grid, 128, 0, st>>>(x, ldx, rows, cols, meanf, stdf, unnorm, dst);
    ASE_LAUNCH_OK();
    return ASE_OK;
  }
  dim3 grid(ceil_div(cols, 128), ceil_div(rows, NORM_ROWS_PER_BLOCK));
  rms_normalize_kernel<<<grid, 128, 0, st>>>(x, ldx, rows, cols, meanf, stdf, unnorm, dst);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

int copy_cols(const float* x, int64_t ldx, int rows, int cols, float* y, int64_t ldy, cudaStream_t st, void* hi, void* lo, int64_t ldp, int half,
              float pscale, unsigned* flag) {
  const int64_t total = (int64_t)rows * cols;
  const int blocks = (int)imin64((total + 255) / 256, NUM_SMS * 16);
  copy_cols_kernel<<<blocks, 256, 0, st>>>(x, ldx, rows, cols, y, ldy, hi, lo, ldp, half, pscale, flag);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

}  // namespace ase

using namespace ase;

extern "C" int64_t ase_rms_scratch_bytes(int rows, int cols) { return rms_scratch_bytes(cols, rows, 1); }

extern "C" int ase_rms_update(const float* x, int64_t ldx, int rows, int cols, double* mean, double* var, double* count,
                              float eps, float* y, int64_t ldy, void* scratch, void* stream) {
  ASE_CHECK_ARG(x && mean && var && count && scratch, "ase_rms_update: null pointer");
  RmsBatchList bl; bl.x[0] = x; bl.ld[0] = ldx; bl.rows = rows;
  float *meanf, *stdf;
  int rc = rms_update_batches(bl, 1, cols, mean, var, count, eps, 1, scratch, &meanf, &stdf, (cudaStream_t)stream);
  if (rc) return rc;
  if (y) {
    RmsDst d = {}; d.y[0] = y; d.ld[0] = ldy;
    return rms_normalize(x, ldx, rows, cols, meanf, stdf, 0, d, (cudaStream_t)stream);
  }
  return ASE_OK;
}

namespace ase {
// eval-mode normalisation straight from the fp64 stats (no scratch): used by rollout inference
__global__ void __launch_bounds__(256)
rms_apply_kernel(const float* __restrict__ x, int64_t ldx, int rows, int cols, const double* __restrict__ mean,
                 const double* __restrict__ var, float eps, int unnorm, float* __restrict__ y, int64_t ldy) {
  const int64_t total = (int64_t)rows * cols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / cols), c = (int)(i - (int64_t)r * cols);
    const float v = x[(int64_t)r * ldx + c];
    const float m = (float)mean[c], s = sqrtf((float)var[c] + eps);
    y[(int64_t)r * ldy + c] = unnorm ? (s * fminf(fmaxf(v, -5.0f), 5.0f) + m) : fminf(fmaxf((v - m) / s, -5.0f), 5.0f);
  }
}
int rms_apply(const float* x, int64_t ldx, int rows, int cols, const double* mean, const double* var, float eps, int unnorm,
              float* y, int64_t ldy, cudaStream_t st) {
  const int64_t total = (int64_t)rows * cols;
  if (total == 0) return ASE_OK;
  const int blocks = (int)imin64((total + 255) / 256, NUM_SMS * 16);
  rms_apply_kernel<<<blocks, 256, 0, st>>>(x, ldx, rows, cols, mean, var, eps, unnorm, y, ldy);
  ASE_LAUNCH_OK();
  return ASE_OK;
}
}  // namespace ase

extern "C" int ase_rms_apply(const float* x, int64_t ldx, int rows, int cols, const double* mean, const double* var,
                             float eps, int unnorm, float* y, int64_t ldy, void* stream) {
  ASE_CHECK_ARG(x && mean && var && y, "ase_rms_apply: null pointer");
  return rms_apply(x, ldx, rows, cols, mean, var, eps, unnorm, y, ldy, (cudaStream_t)stream);
}
