// Evaluation players (learning/common_player.py, amp_players.py, ase_players.py, hrl_players.py) without host round trips: the latent writes,
// the action head and the episode bookkeeping of CommonPlayer.run are mask driven, so a window of player steps is a fixed sequence of launches.
#include "common.cuh"
#include "kernels.h"
#include "philox.cuh"

namespace ase {

// ase_players.py:61-80 env_reset(done) -> _reset_latents(done_ids), and :82-94 _update_latents (resample_all).  One warp per env.
__global__ void __launch_bounds__(256)
player_latents_kernel(float* __restrict__ latents, int Z, const uint8_t* __restrict__ done_mask, int resample_all, int n,
                      const uint64_t* __restrict__ rng, int sid, const float* __restrict__ z_in) {
  const int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (e >= n) return;
  if (!resample_all && !(done_mask && done_mask[e] != 0)) return;     // warp-uniform
  warp_write_latent(latents + (int64_t)e * Z, Z, rng, (uint32_t)sid, (uint32_t)e, z_in ? z_in + (int64_t)e * Z : nullptr);
}

// ase_players.py:54-59 / hrl_players.py:53-60,247-249: a = mu (deterministic) or mu + exp(logstd) * eps (Normal.sample), clamp to [-1, 1],
// then rl_games rescale_actions(low, high, a) = a * (high - low) / 2 + (high + low) / 2.  unit_out = normalize(clamped a) (the HRL LLC's
// latent, F.normalize eps 1e-12).  __f*_rn: the reference rounds each product and sum separately.  One warp per row, A <= 128.
__global__ void __launch_bounds__(256)
player_act_kernel(const float* __restrict__ mu, const float* __restrict__ logstd, int rows, int A, const float* __restrict__ low,
                  const float* __restrict__ high, const uint64_t* __restrict__ rng, int sid, const float* __restrict__ noise_in,
                  float* __restrict__ actions, float* __restrict__ unit_out) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= rows) return;
  float a[4] = {0.0f, 0.0f, 0.0f, 0.0f};
  float ss = 0.0f;
  for (int j0 = lane * 4; j0 < A; j0 += 128) {
    float4 z = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (logstd && !noise_in) z = philox_normal4(rng, (uint32_t)sid, (uint32_t)row, (uint32_t)(j0 >> 2));
    const float zz[4] = {z.x, z.y, z.z, z.w};
    for (int q = 0; q < 4 && j0 + q < A; ++q) {
      const int j = j0 + q;
      float v = mu[(int64_t)row * A + j];
      if (logstd) v = __fadd_rn(__fmul_rn(noise_in ? noise_in[(int64_t)row * A + j] : zz[q], expf(logstd[j])), v);
      v = fminf(fmaxf(v, -1.0f), 1.0f);
      a[q] = v;
      ss += v * v;
      if (actions) {
        float o = v;
        if (low) o = __fadd_rn(__fmul_rn(v, (high[j] - low[j]) / 2.0f), (high[j] + low[j]) / 2.0f);
        actions[(int64_t)row * A + j] = o;
      }
    }
  }
  if (!unit_out) return;                            // row-uniform
  ss = warp_sum(ss);
  const float den = fmaxf(sqrtf(ss), 1e-12f);
  for (int j0 = lane * 4; j0 < A; j0 += 128)
    for (int q = 0; q < 4 && j0 + q < A; ++q) unit_out[(int64_t)row * A + j0 + q] = a[q] / den;
}

// common_player.py:73-117 after env.step, hrl_players.py:174-191 for the sub-steps.  See ase_player_post_step in include/ase_b200.h.
__global__ void __launch_bounds__(256)
player_post_step_kernel(const float* __restrict__ rewards, const uint8_t* __restrict__ dones, int n, int sub_step, int llc_steps,
                        float* __restrict__ sub_rewards, float* __restrict__ sub_dones, float* __restrict__ cr, float* __restrict__ steps,
                        uint8_t* __restrict__ done_out, int64_t n_games, AsePlayerStatus* __restrict__ status, double* __restrict__ record,
                        double* __restrict__ partials, uint64_t* __restrict__ rng) {
  __shared__ double sm[32 * 3];
  __shared__ bool last;
  if (*(volatile int32_t*)&status->stopped) return;          // sticky: every block of every later launch leaves the accumulators alone
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const bool final_sub = sub_step == llc_steps - 1;
  double acc[3] = {0.0, 0.0, 0.0};                            // finished envs: sum of cr, sum of steps, count
  if (e < n) {
    float r = rewards[e];
    bool d = dones[e] != 0;
    if (llc_steps > 1) {                                      // rewards = 0.0 + r_0 + ... ; done_count = 0.0 + d_0 + ...
      const float sr = (sub_step == 0 ? 0.0f : sub_rewards[e]) + r, sd = (sub_step == 0 ? 0.0f : sub_dones[e]) + (d ? 1.0f : 0.0f);
      sub_rewards[e] = sr; sub_dones[e] = sd;
      r = sr / (float)llc_steps;
      d = sd > 0.0f;
    }
    if (final_sub) {
      const float c = cr[e] + r, s = steps[e] + 1.0f;
      if (d) { acc[0] = (double)c; acc[1] = (double)s; acc[2] = 1.0; }
      cr[e] = d ? 0.0f : c; steps[e] = d ? 0.0f : s;
      done_out[e] = d ? 1 : 0;
    }
  }
  if (!final_sub) return;                                     // grid-uniform
  block_sum<3>(acc, sm);
  if (threadIdx.x == 0) {
    for (int i = 0; i < 3; ++i) partials[blockIdx.x * 3 + i] = acc[i];
    __threadfence();
    last = atomicAdd(&status->ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  double t[3] = {0.0, 0.0, 0.0};
  for (unsigned b = 0; b < gridDim.x; ++b)                    // in block order: the totals do not depend on which block finished last
    for (int i = 0; i < 3; ++i) t[i] += ((volatile double*)partials)[b * 3 + i];
  const int64_t count = (int64_t)t[2];
  record[0] = t[2]; record[1] = t[0]; record[2] = t[1];
  status->reward_sum += t[0];
  status->steps_sum += t[1];
  status->games_played += count;
  if (status->games_played >= n_games) status->stopped = 1;   // the step that reaches n_games counts in full
  status->ticket = 0;
  if (rng) rng[1] += 1;                                       // every draw of this player step has been taken (stream order)
}

}  // namespace ase

extern "C" int ase_player_latents(float* latents, int latent_dim, const uint8_t* done_mask, int resample_all, int num_envs, const uint64_t* rng,
                                  int stream_id, const float* z_in, void* stream) {
  ASE_CHECK_ARG(latents && latent_dim > 0 && latent_dim <= 128, "ase_player_latents: bad argument");
  ASE_CHECK_ARG(resample_all || done_mask, "ase_player_latents: done_mask required unless resample_all");
  ASE_CHECK_ARG(rng || z_in, "ase_player_latents: rng state or injected latents required");
  if (num_envs <= 0) return ASE_OK;
  ase::player_latents_kernel<<<ase::ceil_div((int64_t)num_envs * 32, 256), 256, 0, (cudaStream_t)stream>>>(latents, latent_dim, done_mask, resample_all,
                                                                                                         num_envs, rng, stream_id, z_in);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_player_act(const float* mu, const float* logstd, int rows, int act_dim, const float* low, const float* high, const uint64_t* rng,
                              int stream_id, const float* noise_in, float* actions, float* unit_out, void* stream) {
  ASE_CHECK_ARG(mu && (actions || unit_out) && act_dim > 0 && act_dim <= 128, "ase_player_act: bad argument");
  ASE_CHECK_ARG(!logstd || rng || noise_in, "ase_player_act: stochastic mode needs rng state or injected noise");
  ASE_CHECK_ARG((low == nullptr) == (high == nullptr), "ase_player_act: low and high go together");
  if (rows <= 0) return ASE_OK;
  ase::player_act_kernel<<<ase::ceil_div((int64_t)rows * 32, 256), 256, 0, (cudaStream_t)stream>>>(mu, logstd, rows, act_dim, low, high, rng, stream_id,
                                                                                                 noise_in, actions, unit_out);
  ASE_LAUNCH_OK();
  return ASE_OK;
}

extern "C" int ase_player_scratch_bytes(int num_envs) { return ase::ceil_div(num_envs > 0 ? num_envs : 1, 256) * 3 * (int)sizeof(double); }

extern "C" int ase_player_post_step(const float* rewards, const uint8_t* dones, int num_envs, int sub_step, int llc_steps, float* sub_rewards,
                                    float* sub_dones, float* cr, float* steps, uint8_t* done_out, int64_t n_games, AsePlayerStatus* status,
                                    double* record, void* scratch, uint64_t* rng, void* stream) {
  ASE_CHECK_ARG(rewards && dones && cr && steps && done_out && status && record && scratch, "ase_player_post_step: null pointer");
  ASE_CHECK_ARG(llc_steps >= 1 && sub_step >= 0 && sub_step < llc_steps, "ase_player_post_step: sub_step %d of %d", sub_step, llc_steps);
  ASE_CHECK_ARG(llc_steps == 1 || (sub_rewards && sub_dones), "ase_player_post_step: sub-step accumulators required");
  if (num_envs <= 0) return ASE_OK;
  ase::player_post_step_kernel<<<ase::ceil_div(num_envs, 256), 256, 0, (cudaStream_t)stream>>>(rewards, dones, num_envs, sub_step, llc_steps, sub_rewards,
                                                                                              sub_dones, cr, steps, done_out, n_games, status, record,
                                                                                              (double*)scratch, rng);
  ASE_LAUNCH_OK();
  return ASE_OK;
}
