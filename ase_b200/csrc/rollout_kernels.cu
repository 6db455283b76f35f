// Rollout-side scans / reductions (HBM-bound): GAE, AMP/ASE rewards, advantage normalisation.
#include "common.cuh"
#include "kernels.h"
#include "philox.cuh"

namespace ase {

// learning/common_agent.py:437-449.  One thread per env, reverse scan over the horizon; [H,N] row-major so
// a warp reads 32 consecutive envs per step (coalesced).  Algorithmic bytes: (3*4 + 1 + 2*4) * H * N.
__global__ void __launch_bounds__(128)
gae_kernel(const uint8_t* __restrict__ dones, const float* __restrict__ values, const float* __restrict__ rewards,
           const float* __restrict__ next_values, int H, int N, float gamma, float tau,
           float* __restrict__ advs, float* __restrict__ returns) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= N) return;
  float last = 0.0f;
  for (int t = H - 1; t >= 0; --t) {
    const int64_t i = (int64_t)t * N + e;
    const float nd = 1.0f - (float)dones[i];
    const float v = values[i];
    const float delta = rewards[i] + gamma * next_values[i] - v;
    last = delta + gamma * tau * nd * last;
    advs[i] = last;
    if (returns) returns[i] = last + v;
  }
}

// amp_agent.py:570-577, ase_agent.py:404-411,469-472,484-490.  One warp per row (latent dot product).
__global__ void __launch_bounds__(256)
amp_rewards_kernel(const float* __restrict__ logits, const float* __restrict__ enc_pred, const float* __restrict__ z,
                   int zdim, int rows, float disc_scale, float enc_scale, const float* __restrict__ task_r,
                   float task_w, float disc_w, float enc_w, float* __restrict__ disc_r, float* __restrict__ enc_r,
                   float* __restrict__ combined) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= rows) return;
  float er = 0.0f;
  if (enc_pred) {
    float d = 0.0f;
    for (int j = lane; j < zdim; j += 32) d += enc_pred[(int64_t)row * zdim + j] * z[(int64_t)row * zdim + j];
    d = warp_sum(d);
    er = fmaxf(d, 0.0f) * enc_scale;      // clamp_min(-err, 0), err = -sum(enc*z)
  }
  if (lane == 0) {
    const float l = logits[row];
    const float prob = 1.0f / (1.0f + expf(-l));
    const float dr = -logf(fmaxf(1.0f - prob, 0.0001f)) * disc_scale;
    if (disc_r) disc_r[row] = dr;
    if (enc_r && enc_pred) enc_r[row] = er;
    if (combined) combined[row] = task_w * (task_r ? task_r[row] : 0.0f) + disc_w * dr + (enc_pred ? enc_w * er : 0.0f);
  }
}

// Gaussian sampling head (eval mode) + eps-greedy override; one warp per row.
__global__ void __launch_bounds__(256)
policy_sample_kernel(const float* __restrict__ mu, const float* __restrict__ logstd, const float* __restrict__ noise,
                     const float* __restrict__ rand_mask, int rows, int A, float* __restrict__ actions,
                     float* __restrict__ neglogp, float* __restrict__ sigma_out) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= rows) return;
  const bool det = rand_mask && rand_mask[row] == 0.0f;
  float s = 0.0f, sumlog = 0.0f;
  for (int j = lane; j < A; j += 32) {
    const float ls = logstd[j], sg = expf(ls), m = mu[(int64_t)row * A + j];
    const float a = m + sg * noise[(int64_t)row * A + j];
    const float t = (a - m) / sg;
    s += t * t; sumlog += ls;
    actions[(int64_t)row * A + j] = det ? m : a;
    if (sigma_out) sigma_out[(int64_t)row * A + j] = sg;
  }
  s = warp_sum(s); sumlog = warp_sum(sumlog);
  if (lane == 0 && neglogp) neglogp[row] = 0.5f * s + (float)(0.5 * 1.8378770664093453 * (double)A) + sumlog;
}

// stats[0..2] = sum(m), sum(v*m), sum((v*m)^2) ; unmasked: m = 1
__global__ void __launch_bounds__(256)
adv_stats_kernel(const float* __restrict__ ret, const float* __restrict__ val, const float* __restrict__ mask, int rows,
                 double* __restrict__ stats) {
  __shared__ double sm[32 * 3];
  double acc[3] = {0.0, 0.0, 0.0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += gridDim.x * blockDim.x) {
    const float a = ret[i] - val[i];
    const float m = mask ? mask[i] : 1.0f;
    const double vm = (double)(a * m);
    acc[0] += (double)m; acc[1] += vm; acc[2] += vm * vm;
  }
  block_sum<3>(acc, sm);
  if (threadIdx.x == 0) { atomicAdd(&stats[0], acc[0]); atomicAdd(&stats[1], acc[1]); atomicAdd(&stats[2], acc[2]); }
}

__global__ void __launch_bounds__(256)
adv_apply_kernel(const float* __restrict__ ret, const float* __restrict__ val, int rows, const double* __restrict__ stats,
                 float* __restrict__ advs) {
  // torch_ext.normalization_with_masks: var = (E[(vm)^2] - E[vm]^2) * n/(n-1)   (for mask == 1 this is the
  // unbiased variance that advantages.std() uses in common_agent.py:543)
  const double n = stats[0];
  const double mean = stats[1] / n;
  const double min_sqr = stats[2] / n - mean * mean;
  const double var = min_sqr * n / (n - 1.0);
  const float meanf = (float)mean, stdf = (float)sqrt(var > 0.0 ? var : 0.0);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += gridDim.x * blockDim.x)
    advs[i] = ((ret[i] - val[i]) - meanf) / (stdf + 1e-8f);
}

}  // namespace ase

using namespace ase;

extern "C" int ase_gae(const uint8_t* dones, const float* values, const float* rewards, const float* next_values,
                       int horizon, int num_envs, float gamma, float tau, float* advs, float* returns, void* stream) {
  ASE_CHECK_ARG(dones && values && rewards && next_values && advs, "ase_gae: null pointer");
  if (horizon <= 0 || num_envs <= 0) return ASE_OK;
  gae_kernel<<<ceil_div(num_envs, 128), 128, 0, (cudaStream_t)stream>>>(dones, values, rewards, next_values, horizon, num_envs,
                                                                         gamma, tau, advs, returns);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_amp_rewards(const float* disc_logits, const float* enc_pred, const float* latents, int latent_dim, int rows,
                               float disc_scale, float enc_scale, const float* task_rewards, float task_w, float disc_w,
                               float enc_w, float* disc_r, float* enc_r, float* combined, void* stream) {
  ASE_CHECK_ARG(disc_logits, "ase_amp_rewards: null logits");
  ASE_CHECK_ARG((enc_pred == nullptr) == (latents == nullptr), "ase_amp_rewards: enc_pred and latents go together");
  if (rows <= 0) return ASE_OK;
  amp_rewards_kernel<<<ceil_div((int64_t)rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      disc_logits, enc_pred, latents, latent_dim, rows, disc_scale, enc_scale, task_rewards, task_w, disc_w, enc_w, disc_r, enc_r,
      combined);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_adv_normalize(const float* returns, const float* values, const float* mask, int rows, float* advs,
                                 void* scratch, void* stream) {
  ASE_CHECK_ARG(returns && values && advs && scratch, "ase_adv_normalize: null pointer");
  if (rows <= 0) return ASE_OK;
  cudaStream_t st = (cudaStream_t)stream;
  ASE_CUDA_OK(cudaMemsetAsync(scratch, 0, 3 * sizeof(double), st));
  const int blocks = min(ceil_div(rows, 256), NUM_SMS * 4);
  adv_stats_kernel<<<blocks, 256, 0, st>>>(returns, values, mask, rows, (double*)scratch);
  ASE_LAUNCH_OK();
  adv_apply_kernel<<<blocks, 256, 0, st>>>(returns, values, rows, (const double*)scratch, advs);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_policy_sample(const float* mu, const float* logstd, const float* noise, const float* rand_mask, int rows,
                                 int act_dim, float* actions, float* neglogp, float* sigma_out, void* stream) {
  ASE_CHECK_ARG(mu && logstd && noise && actions, "ase_policy_sample: null pointer");
  if (rows <= 0) return ASE_OK;
  policy_sample_kernel<<<ceil_div((int64_t)rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(mu, logstd, noise, rand_mask, rows, act_dim,
                                                                                           actions, neglogp, sigma_out);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

// ------------------------------------------------------------------------------------------------------------
// Minibatch gather (learning/amp_datasets.py:14-27 AMPDataset._get_item + the demo / replay row fetches of
// amp_agent.py:194-202): dst_i[r, :] = src_i[idx_i[r], :] for up to ASE_GATHER_MAX tensors in ONE launch
// (the reference issues one advanced-indexing kernel per tensor, 13 per minibatch).  blockIdx.y = tensor.
// ------------------------------------------------------------------------------------------------------------
namespace ase {
__global__ void __launch_bounds__(256)
gather_rows_kernel(AseGatherBatch b) {
  const AseGatherItem it = b.item[blockIdx.y];
  const bool vec = ((it.cols & 3) == 0) && ((it.src_ld & 3) == 0) && ((it.dst_ld & 3) == 0) &&
                   ((reinterpret_cast<uintptr_t>(it.src) & 15) == 0) && ((reinterpret_cast<uintptr_t>(it.dst) & 15) == 0);
  if (vec) {
    const int c4n = it.cols >> 2;
    const int64_t total = (int64_t)it.rows * c4n;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
      const int r = (int)(i / c4n), c = (int)(i - (int64_t)r * c4n) * 4;
      const int64_t sr = it.idx ? it.idx[r] : r;
      *reinterpret_cast<float4*>(it.dst + (int64_t)r * it.dst_ld + c) = *reinterpret_cast<const float4*>(it.src + sr * it.src_ld + c);
    }
  } else {
    const int64_t total = (int64_t)it.rows * it.cols;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
      const int r = (int)(i / it.cols), c = (int)(i - (int64_t)r * it.cols);
      const int64_t sr = it.idx ? it.idx[r] : r;
      it.dst[(int64_t)r * it.dst_ld + c] = it.src[sr * it.src_ld + c];
    }
  }
}
}  // namespace ase

extern "C" int ase_gather_rows(const AseGatherBatch* batch, void* stream) {
  ASE_CHECK_ARG(batch && batch->count >= 0 && batch->count <= ASE_GATHER_MAX, "ase_gather_rows: bad batch");
  if (batch->count == 0) return ASE_OK;
  int64_t big = 0;
  for (int i = 0; i < batch->count; ++i) {
    const AseGatherItem& it = batch->item[i];
    ASE_CHECK_ARG(it.src && it.dst && it.rows >= 0 && it.cols > 0 && it.src_ld >= it.cols && it.dst_ld >= it.cols, "ase_gather_rows: item %d", i);
    big = ase::imax64(big, (int64_t)it.rows * it.cols);
  }
  if (big == 0) return ASE_OK;
  dim3 grid((unsigned)ase::imin64((big / 4 + 255) / 256 + 1, NUM_SMS * 4), (unsigned)batch->count);
  ase::gather_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(*batch);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

// ------------------------------------------------------------------------------------------------------------
// Rollout step without host round trips (SURVEY.md section 7.1 step 9; ase_agent.py:36-115,366-381).
// The reference draws its random numbers with eager torch calls and turns `dones` / `_latent_reset_steps <= progress_buf` into index
// lists with nonzero() -- a host sync per step.  Here the step is a fixed sequence of kernels driven by MASKS, with a counter-based
// generator (Philox4x32-10, Salmon et al. 2011) evaluated inside the kernels: element (row, column) of draw number `rng[1]` of stream
// `stream_id` is a pure function of (rng[0] = seed, stream_id, rng[1], row, column), so the sequence can be captured in a CUDA graph
// (ase_rollout_post_step advances rng[1] on the device).  Parity tests inject the draws instead (noise_in / mask_in / z_in / steps_in).
// The generator itself is in philox.cuh (shared with the episode resets of reset_kernels.cu).
// ------------------------------------------------------------------------------------------------------------
namespace ase {

// Gaussian head (eval mode) + eps-greedy override with in-kernel draws; one warp per row, lane = action dimension (A <= 128).
__global__ void __launch_bounds__(256)
policy_sample_rng_kernel(const float* __restrict__ mu, const float* __restrict__ logstd, const float* __restrict__ rand_probs, int rows, int A,
                         const uint64_t* __restrict__ rng, int sid, const float* __restrict__ noise_in, const float* __restrict__ mask_in,
                         float* __restrict__ actions, float* __restrict__ neglogp, float* __restrict__ sigma_out, float* __restrict__ mask_out) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= rows) return;
  float m = 1.0f;                                  // rand_action_mask: bernoulli(p) (amp_agent.py:164); 1 when there is no eps-greedy
  if (mask_in) m = mask_in[row];
  else if (rand_probs) m = (u01_open(philox_u4(rng, (uint32_t)sid + 1u, (uint32_t)row, 0xFFFFFFFFu).x) < rand_probs[row]) ? 1.0f : 0.0f;
  const bool det = m == 0.0f;
  float s = 0.0f, sumlog = 0.0f;
  for (int j0 = lane * 4; j0 < A; j0 += 128) {
    float4 z = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (!noise_in) z = philox_normal4(rng, (uint32_t)sid, (uint32_t)row, (uint32_t)(j0 >> 2));
    const float zz[4] = {z.x, z.y, z.z, z.w};
    for (int q = 0; q < 4 && j0 + q < A; ++q) {
      const int j = j0 + q;
      const float nz = noise_in ? noise_in[(int64_t)row * A + j] : zz[q];
      const float ls = logstd[j], sg = expf(ls), mm = mu[(int64_t)row * A + j];
      const float a = mm + sg * nz;
      const float t = (a - mm) / sg;
      s += t * t; sumlog += ls;
      actions[(int64_t)row * A + j] = det ? mm : a;
      if (sigma_out) sigma_out[(int64_t)row * A + j] = sg;
    }
  }
  s = warp_sum(s); sumlog = warp_sum(sumlog);
  if (lane == 0) {
    if (neglogp) neglogp[row] = 0.5f * s + (float)(0.5 * 1.8378770664093453 * (double)A) + sumlog;
    if (mask_out) mask_out[row] = m;
  }
}

// ase_agent.py:366-381 _update_latents + :329-364 env_reset's latent part, mask driven.  One warp per env.
//   done_mask[e] != 0 : fresh latent, reset_steps[e]  = randint(min, max)      (_reset_latents + _reset_latent_step_count)
//   else if reset_steps[e] <= progress[e] : fresh latent, reset_steps[e] += randint(min, max)   (_update_latents)
// latent = normalize(randn(Z)) (ase_network_builder.py:221-225; F.normalize eps 1e-12)
__global__ void __launch_bounds__(256)
latent_update_kernel(float* __restrict__ latents, int Z, int32_t* __restrict__ reset_steps, const int64_t* __restrict__ progress,
                     const uint8_t* __restrict__ done_mask, int n, int smin, int smax, const uint64_t* __restrict__ rng, int sid,
                     const float* __restrict__ z_in, const int32_t* __restrict__ steps_in) {
  const int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (e >= n) return;
  const bool reset = done_mask && done_mask[e] != 0;
  const int32_t cur = reset_steps[e];
  const bool update = !reset && ((int64_t)cur <= progress[e]);
  if (!reset && !update) return;                   // warp-uniform
  warp_write_latent(latents + (int64_t)e * Z, Z, rng, (uint32_t)sid, (uint32_t)e, z_in ? z_in + (int64_t)e * Z : nullptr);
  if (lane == 0) {
    int32_t r;
    if (steps_in) r = steps_in[e];
    else r = smin + (int32_t)(philox_u4(rng, (uint32_t)sid + 1u, (uint32_t)e, 0xFFFFFFFEu).x % (uint32_t)max(1, smax - smin));   // torch.randint(low, high): [low, high)
    reset_steps[e] = reset ? r : cur + r;
  }
}

// after env.step (ase_agent.py:66-92): next_values = unnorm(v) * (1 - terminated); episode statistics; advances the RNG call counter.
__global__ void __launch_bounds__(256)
rollout_post_step_kernel(const float* __restrict__ rewards, const uint8_t* __restrict__ dones, const uint8_t* __restrict__ terminate,
                         const float* __restrict__ v_next, const double* __restrict__ vmean, const double* __restrict__ vvar, float eps, int n,
                         float* __restrict__ next_values, float* __restrict__ cur_r, float* __restrict__ cur_l, float* __restrict__ meter,
                         uint64_t* __restrict__ rng) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  float dr = 0.0f, dl = 0.0f, dc = 0.0f;
  if (e < n) {
    if (next_values) {
      const float m = (float)vmean[0], s = sqrtf((float)vvar[0] + eps);
      const float v = s * fminf(fmaxf(v_next[e], -5.0f), 5.0f) + m;
      next_values[e] = v * (1.0f - (float)(terminate[e] != 0));
    }
    const float r = cur_r[e] + rewards[e], l = cur_l[e] + 1.0f;
    const bool d = dones[e] != 0;
    if (d) { dr = r; dl = l; dc = 1.0f; }            // game_rewards / game_lengths .update(current_*[done_indices])
    cur_r[e] = d ? 0.0f : r; cur_l[e] = d ? 0.0f : l;
  }
  dr = warp_sum(dr); dl = warp_sum(dl); dc = warp_sum(dc);
  if ((threadIdx.x & 31) == 0 && dc > 0.0f && meter) { atomicAdd(meter + 0, dr); atomicAdd(meter + 1, dl); atomicAdd(meter + 2, dc); }
  if (rng && e == 0) rng[1] += 1;                   // every draw of this step has been taken (stream order)
}

// env/tasks/humanoid.py:645-670 compute_humanoid_reset: one warp per env over the bodies.
__global__ void __launch_bounds__(256)
humanoid_reset_kernel(const int64_t* __restrict__ progress, const float* __restrict__ contact, int64_t contact_env_stride, int64_t contact_body_stride,
                      const float* __restrict__ body_state, int64_t env_stride, int64_t body_stride, int J, const uint8_t* __restrict__ is_contact_body,
                      const float* __restrict__ term_heights, float max_episode_length, int early_term, int n,
                      uint8_t* __restrict__ reset_out, uint8_t* __restrict__ terminate_out) {
  const int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (e >= n) return;
  int fc = 0, fh = 0;
  if (early_term) {
    for (int b = lane; b < J; b += 32) {
      if (is_contact_body[b]) continue;              // masked_contact_buf[:, contact_body_ids, :] = 0 ; fall_height[:, contact_body_ids] = False
      const float* c = contact + (int64_t)e * contact_env_stride + (int64_t)b * contact_body_stride;
      fc |= (fabsf(c[0]) > 0.1f) || (fabsf(c[1]) > 0.1f) || (fabsf(c[2]) > 0.1f);
      fh |= body_state[(int64_t)e * env_stride + (int64_t)b * body_stride + 2] < term_heights[b];
    }
  }
  fc = __any_sync(0xffffffffu, fc); fh = __any_sync(0xffffffffu, fh);
  if (lane == 0) {
    const int64_t p = progress[e];
    const int term = (early_term && fc && fh && p > 1) ? 1 : 0;
    terminate_out[e] = (uint8_t)term;
    reset_out[e] = (uint8_t)(((float)p >= max_episode_length - 1.0f) ? 1 : term);
  }
}

// env/tasks/humanoid_strike.py:254-295 compute_humanoid_reset: the base rule plus "the target was hit while a body other than the strike bodies
// touches something".  nonstrike_body_force aliases masked_contact_buf, but fall_contact is computed before the strike bodies are zeroed.
__global__ void __launch_bounds__(256)
strike_reset_kernel(const int64_t* __restrict__ progress, const float* __restrict__ contact, int64_t contact_env_stride, int64_t contact_body_stride,
                    const float* __restrict__ body_state, int64_t env_stride, int64_t body_stride, int J, const uint8_t* __restrict__ is_contact_body,
                    const uint8_t* __restrict__ is_strike_body, const float* __restrict__ term_heights, const float* __restrict__ tar_contact,
                    int64_t tar_contact_stride, float max_episode_length, int early_term, int n, uint8_t* __restrict__ reset_out,
                    uint8_t* __restrict__ terminate_out) {
  const int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (e >= n) return;
  int fc = 0, fh = 0, ns = 0;
  if (early_term) {
    for (int b = lane; b < J; b += 32) {
      if (is_contact_body[b]) continue;
      const float* c = contact + (int64_t)e * contact_env_stride + (int64_t)b * contact_body_stride;
      fc |= (fabsf(c[0]) > 0.1f) || (fabsf(c[1]) > 0.1f) || (fabsf(c[2]) > 0.1f);
      fh |= body_state[(int64_t)e * env_stride + (int64_t)b * body_stride + 2] < term_heights[b];
      if (!is_strike_body[b]) ns |= (fabsf(c[0]) > 1.0f) || (fabsf(c[1]) > 1.0f) || (fabsf(c[2]) > 1.0f);
    }
  }
  fc = __any_sync(0xffffffffu, fc); fh = __any_sync(0xffffffffu, fh); ns = __any_sync(0xffffffffu, ns);
  if (lane == 0) {
    const int64_t p = progress[e];
    int term = 0;
    if (early_term) {
      const float* tc = tar_contact + (int64_t)e * tar_contact_stride;
      const bool tar_has_contact = (fabsf(tc[0]) > 1.0f) || (fabsf(tc[1]) > 1.0f);      // x and y only
      term = ((fc && fh) || (tar_has_contact && ns)) && p > 1;
    }
    terminate_out[e] = (uint8_t)term;
    reset_out[e] = (uint8_t)(((float)p >= max_episode_length - 1.0f) ? 1 : term);
  }
}

// _update_task / _reset_task of humanoid_{heading,location,reach}.py and _reset_target of humanoid_strike.py, mask driven.  One thread per env.
// Update mode (mask NULL): envs with progress >= change_steps resample.  Reset mode: envs with a non-zero mask resample.  Uniform k of an env is
// its k-th draw in the reference's order (torch.rand calls, or the columns of torch.rand([n, c])); the randint of change_steps is [min, max).
__global__ void __launch_bounds__(128)
task_resample_kernel(AseTaskParams p, const float* __restrict__ root, int64_t rs, const int64_t* __restrict__ progress, const uint8_t* __restrict__ mask,
                     int n, float* __restrict__ tar, int64_t ts, float* __restrict__ tar_speed, float* __restrict__ face, int64_t* __restrict__ change_steps,
                     const uint64_t* __restrict__ rng, int sid, const float* __restrict__ u_in, const int64_t* __restrict__ steps_in) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const bool go = mask ? mask[e] != 0 : progress[e] >= change_steps[e];
  if (!go) return;
  float u[4];
  if (u_in) {
    for (int q = 0; q < 4; ++q) u[q] = u_in[(int64_t)e * 4 + q];
  } else {
    const uint4 r = philox_u4(rng, (uint32_t)sid, (uint32_t)e, 0u);
    u[0] = u01_open(r.x); u[1] = u01_open(r.y); u[2] = u01_open(r.z); u[3] = u01_open(r.w);
  }
  const float kTwoPi = 6.28318530717958647692f, kPi = 3.14159265358979323846f;
  const float* r = root + (int64_t)e * rs;
  float* t = tar + (int64_t)e * ts;
  // __f*_rn: the reference rounds each product and sum separately (no fused multiply-add)
  switch (p.kind) {
    case ASE_TASK_HEADING: {                      // humanoid_heading.py:154-174
      float th = 0.0f, thf = 0.0f;
      int k = 0;
      if (p.rand_heading) { th = __fsub_rn(__fmul_rn(kTwoPi, u[0]), kPi); thf = __fsub_rn(__fmul_rn(kTwoPi, u[1]), kPi); k = 2; }
      tar_speed[e] = __fadd_rn(__fmul_rn(p.speed_max - p.speed_min, u[k]), p.speed_min);
      t[0] = cosf(th); t[1] = sinf(th);
      face[2 * e] = cosf(thf); face[2 * e + 1] = sinf(thf);
      break;
    }
    case ASE_TASK_LOCATION:                       // humanoid_location.py:115-125: root xy + dist_max * (2u - 1)
      t[0] = __fadd_rn(r[0], __fmul_rn(p.dist_max, __fsub_rn(2.0f * u[0], 1.0f)));
      t[1] = __fadd_rn(r[1], __fmul_rn(p.dist_max, __fsub_rn(2.0f * u[1], 1.0f)));
      break;
    case ASE_TASK_REACH:                          // humanoid_reach.py:119-130: absolute xy, height in [min, max)
      t[0] = __fmul_rn(p.dist_max, __fsub_rn(2.0f * u[0], 1.0f));
      t[1] = __fmul_rn(p.dist_max, __fsub_rn(2.0f * u[1], 1.0f));
      t[2] = __fadd_rn(__fmul_rn(p.height_max - p.height_min, u[2]), p.height_min);
      break;
    default: {                                    // ASE_TASK_STRIKE, humanoid_strike.py:108-128
      const float dmax = u[0] < p.near_prob ? p.near_dist : p.dist_max;
      const float dist = __fadd_rn(__fmul_rn(dmax - p.dist_min, u[1]), p.dist_min);
      const float th = __fmul_rn(kTwoPi, u[2]);
      t[0] = __fadd_rn(__fmul_rn(dist, cosf(th)), r[0]);
      t[1] = __fadd_rn(__fmul_rn(dist, sinf(th)), r[1]);
      t[2] = p.target_height;
      const Quat q = quat_from_angle_axis(__fmul_rn(kTwoPi, u[3]), {0.0f, 0.0f, 1.0f});
      t[3] = q.x; t[4] = q.y; t[5] = q.z; t[6] = q.w;
      for (int c = 7; c < 13; ++c) t[c] = 0.0f;
      return;                                     // the strike target has no change schedule
    }
  }
  int64_t steps;
  if (steps_in) steps = steps_in[e];
  else steps = p.change_steps_min + (int64_t)(philox_u4(rng, (uint32_t)sid + 1u, (uint32_t)e, 0xFFFFFFFEu).x %
                                              (uint32_t)max(1, p.change_steps_max - p.change_steps_min));
  change_steps[e] = progress[e] + steps;
}

}  // namespace ase

extern "C" int ase_policy_sample_rng(const float* mu, const float* logstd, const float* rand_probs, int rows, int act_dim, const uint64_t* rng, int stream_id,
                                     const float* noise_in, const float* mask_in, float* actions, float* neglogp, float* sigma_out, float* mask_out,
                                     void* stream) {
  ASE_CHECK_ARG(mu && logstd && actions && (rng || noise_in), "ase_policy_sample_rng: null pointer");
  ASE_CHECK_ARG(noise_in || mask_in || !rand_probs || rng, "ase_policy_sample_rng: rng state required");
  if (rows <= 0) return ASE_OK;
  ase::policy_sample_rng_kernel<<<ase::ceil_div((int64_t)rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(mu, logstd, rand_probs, rows, act_dim, rng, stream_id, noise_in,
                                                                                                        mask_in, actions, neglogp, sigma_out, mask_out);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_latent_update(float* latents, int latent_dim, int32_t* reset_steps, const int64_t* progress, const uint8_t* done_mask, int num_envs,
                                 int steps_min, int steps_max, const uint64_t* rng, int stream_id, const float* z_in, const int32_t* steps_in, void* stream) {
  ASE_CHECK_ARG(latents && reset_steps && progress && latent_dim > 0 && latent_dim <= 128, "ase_latent_update: bad argument");
  ASE_CHECK_ARG((rng || (z_in && steps_in)), "ase_latent_update: rng state or injected draws required");
  if (num_envs <= 0) return ASE_OK;
  ase::latent_update_kernel<<<ase::ceil_div((int64_t)num_envs * 32, 256), 256, 0, (cudaStream_t)stream>>>(latents, latent_dim, reset_steps, progress, done_mask, num_envs,
                                                                                                        steps_min, steps_max, rng, stream_id, z_in, steps_in);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_rollout_post_step(const float* rewards, const uint8_t* dones, const uint8_t* terminate, const float* v_next_normed, const double* val_mean,
                                     const double* val_var, float eps, int num_envs, float* next_values, float* cur_rewards, float* cur_lengths, float* meter,
                                     uint64_t* rng, void* stream) {
  ASE_CHECK_ARG(rewards && dones && cur_rewards && cur_lengths, "ase_rollout_post_step: null pointer");
  ASE_CHECK_ARG(!next_values || (terminate && v_next_normed && val_mean && val_var), "ase_rollout_post_step: value pointers");
  if (num_envs <= 0) return ASE_OK;
  ase::rollout_post_step_kernel<<<ase::ceil_div(num_envs, 256), 256, 0, (cudaStream_t)stream>>>(rewards, dones, terminate, v_next_normed, val_mean, val_var, eps, num_envs,
                                                                                             next_values, cur_rewards, cur_lengths, meter, rng);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_humanoid_reset(const int64_t* progress, const float* contact, int64_t contact_env_stride, int64_t contact_body_stride, const float* body_state,
                                  int64_t env_stride, int64_t body_stride, int num_bodies, const uint8_t* is_contact_body, const float* termination_heights,
                                  float max_episode_length, int enable_early_termination, int num_envs, uint8_t* reset_out, uint8_t* terminate_out, void* stream) {
  ASE_CHECK_ARG(progress && reset_out && terminate_out && num_bodies > 0, "ase_humanoid_reset: null pointer");
  ASE_CHECK_ARG(!enable_early_termination || (contact && body_state && is_contact_body && termination_heights), "ase_humanoid_reset: early termination inputs");
  if (num_envs <= 0) return ASE_OK;
  ase::humanoid_reset_kernel<<<ase::ceil_div((int64_t)num_envs * 32, 256), 256, 0, (cudaStream_t)stream>>>(progress, contact, contact_env_stride, contact_body_stride, body_state,
                                                                                                         env_stride, body_stride, num_bodies, is_contact_body, termination_heights,
                                                                                                         max_episode_length, enable_early_termination, num_envs, reset_out, terminate_out);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_strike_reset(const int64_t* progress, const float* contact, int64_t contact_env_stride, int64_t contact_body_stride, const float* body_state,
                                int64_t env_stride, int64_t body_stride, int num_bodies, const uint8_t* is_contact_body, const uint8_t* is_strike_body,
                                const float* termination_heights, const float* tar_contact, int64_t tar_contact_stride, float max_episode_length,
                                int enable_early_termination, int num_envs, uint8_t* reset_out, uint8_t* terminate_out, void* stream) {
  ASE_CHECK_ARG(progress && reset_out && terminate_out && num_bodies > 0, "ase_strike_reset: null pointer");
  ASE_CHECK_ARG(!enable_early_termination || (contact && body_state && is_contact_body && is_strike_body && termination_heights && tar_contact),
                "ase_strike_reset: early termination inputs");
  if (num_envs <= 0) return ASE_OK;
  ase::strike_reset_kernel<<<ase::ceil_div((int64_t)num_envs * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      progress, contact, contact_env_stride, contact_body_stride, body_state, env_stride, body_stride, num_bodies, is_contact_body, is_strike_body,
      termination_heights, tar_contact, tar_contact_stride, max_episode_length, enable_early_termination, num_envs, reset_out, terminate_out);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_task_resample(const AseTaskParams* p, const float* root_states, int64_t root_stride, const int64_t* progress, const uint8_t* reset_mask,
                                 int num_envs, float* tar, int64_t tar_stride, float* tar_speed, float* tar_face_dir, int64_t* change_steps,
                                 const uint64_t* rng, int stream_id, const float* u_in, const int64_t* steps_in, void* stream) {
  ASE_CHECK_ARG(p && tar && (progress || (p && p->kind == ASE_TASK_STRIKE)), "ase_task_resample: null pointer");
  ASE_CHECK_ARG(p->kind >= ASE_TASK_HEADING && p->kind <= ASE_TASK_STRIKE, "ase_task_resample: unknown task kind %d", p->kind);
  ASE_CHECK_ARG(p->kind != ASE_TASK_STRIKE || reset_mask, "ase_task_resample: the strike target is only resampled on reset (reset_mask required)");
  ASE_CHECK_ARG(p->kind == ASE_TASK_STRIKE || change_steps, "ase_task_resample: change_steps required");
  ASE_CHECK_ARG(p->kind != ASE_TASK_HEADING || (tar_speed && tar_face_dir), "ase_task_resample: heading needs tar_speed and tar_face_dir");
  ASE_CHECK_ARG(p->kind == ASE_TASK_REACH || p->kind == ASE_TASK_HEADING || root_states, "ase_task_resample: root_states required");
  ASE_CHECK_ARG(p->kind == ASE_TASK_STRIKE || p->change_steps_max > p->change_steps_min, "ase_task_resample: empty change-steps range");
  ASE_CHECK_ARG(rng || (u_in && (steps_in || p->kind == ASE_TASK_STRIKE)), "ase_task_resample: rng state or injected draws required");
  if (num_envs <= 0) return ASE_OK;
  ase::task_resample_kernel<<<ase::ceil_div(num_envs, 128), 128, 0, (cudaStream_t)stream>>>(*p, root_states, root_stride, progress, reset_mask, num_envs, tar,
                                                                                          tar_stride, tar_speed, tar_face_dir, change_steps, rng, stream_id,
                                                                                          u_in, steps_in);
  ASE_LAUNCH_OK();
  return ASE_OK;
}
