"""Torch restatement of the reference's HRL rollout (learning/hrl_agent.py:45-82 env_step, :95-163 play_steps, :231-249 the LLC action and
discriminator reward; common_agent.py:309-351 prepare_dataset) over the scripted env of tests/golden/rollout_hrl.pt, built from
ase_oracle's network functions.  Runs in fp32 (the reference's arithmetic) or fp64 (an exact yardstick for the device rollout)."""
import torch
import torch.nn.functional as F

import ase_oracle as O


def _norm(x, st, dtype, eps=1e-5):
    """rl_games RunningMeanStd in eval mode: fp64 statistics cast to the compute type."""
    m, v = st['running_mean'].to(dtype), st['running_var'].to(dtype)
    return torch.clamp((x.to(dtype) - m) / torch.sqrt(v + eps), -5.0, 5.0)


def _unnorm(x, st, dtype, eps=1e-5):
    m, v = st['running_mean'].to(dtype), st['running_var'].to(dtype)
    return torch.sqrt(v + eps) * torch.clamp(x, -5.0, 5.0) + m


def rollout(fx, hlc_params, llc_params, hlc_sigma, dtype=torch.float32, noise=None):
    """fx: the fixture with its regenerated script (golden_util.load('rollout_hrl.pt')); noise: the HLC's standard-normal draws [H, N, 64]
    (default: the recorded ones).  -> dict of the experience-buffer tensors, llc_actions [K, N, 31], returns [N * H, 1], the dataset's
    advantages and the value normaliser after prepare_dataset."""
    N, H, L = fx['N'], fx['H'], fx['llc_steps']
    task = fx['obs_t'].shape[-1] - 253
    Ph = {k: v.to(dtype) for k, v in hlc_params.items()}
    Pl = {k: v.to(dtype) for k, v in llc_params.items()}
    hrms, lrms = fx['hlc_rms'], fx['llc_rms']
    noise = torch.stack(fx['rec']['normal']) if noise is None else noise
    logstd = torch.full((Ph['mu.weight'].shape[0],), float(hlc_sigma), dtype=dtype)
    cfg, dscale = fx['cfg'], fx['llc_disc_reward_scale']
    obs_t, reset_obs_t, amp_t = fx['obs_t'].to(dtype), fx['reset_obs_t'].to(dtype), fx['amp_t'].to(dtype)
    rew_t, dones_t, term_t = fx['rew_t'].to(dtype), fx['dones_t'], fx['term_t']
    z = lambda *s: torch.zeros(H, N, *s, dtype=dtype)
    eb = dict(obses=z(obs_t.shape[-1]), actions=z(logstd.numel()), mus=z(logstd.numel()), sigmas=z(logstd.numel()), neglogpacs=z(), values=z(1),
              rewards=z(1), disc_rewards=z(1), next_values=z(1), dones=torch.zeros(H, N, dtype=torch.uint8))
    llc_actions = torch.zeros(H * L, N, 31, dtype=dtype)
    cur = reset_obs_t[0].clone()                 # train()'s initial env_reset(None)
    done = torch.zeros(N, dtype=torch.bool)      # play_steps starts with done_indices = []
    for n in range(H):
        cur[done] = reset_obs_t[n][done]         # env_reset(done_indices); the env has taken n * L sub-steps
        eb['obses'][n] = cur
        on = _norm(cur, hrms['running_mean_std'], dtype)
        mu = O.eval_actor(Ph, on, mu_tanh=True)
        sigma = torch.exp(logstd).expand_as(mu)
        a = mu + sigma * noise[n].to(dtype)
        eb['actions'][n], eb['mus'][n], eb['sigmas'][n] = a, mu, sigma
        eb['neglogpacs'][n] = O.neglogp(a, mu, logstd)
        eb['values'][n] = _unnorm(O.eval_critic(Ph, on), hrms['reward_mean_std'], dtype)
        # env_step: the frozen LLC runs L sub-steps on the clamped, normalised HLC action
        latent = F.normalize(torch.clamp(a, -1.0, 1.0), dim=-1)
        obs, r, dr = cur, 0.0, 0.0
        dc = torch.zeros(N, dtype=dtype); tc = torch.zeros(N, dtype=dtype)
        for s in range(L):
            k = n * L + s
            lo = _norm(obs[..., :obs.shape[-1] - task], lrms['running_mean_std'], dtype)
            llc_actions[k] = torch.clamp(O.eval_actor(Pl, lo, latent), -1.0, 1.0)
            obs = obs_t[k + 1].clone()
            r = r + rew_t[k]
            dc = dc + dones_t[k].to(dtype); tc = tc + term_t[k].to(dtype)
            logit = O.eval_disc(Pl, _norm(amp_t[k], lrms['amp_input_mean_std'], dtype))
            prob = 1 / (1 + torch.exp(-logit))
            dr = dr + (-torch.log(torch.maximum(1 - prob, torch.tensor(0.0001, dtype=dtype))) * dscale)
        eb['rewards'][n] = (r / L).unsqueeze(-1)
        eb['disc_rewards'][n] = dr / L
        done = dc > 0
        eb['dones'][n] = done.to(torch.uint8)
        cur = obs
        nv = _unnorm(O.eval_critic(Ph, _norm(cur, hrms['running_mean_std'], dtype)), hrms['reward_mean_std'], dtype)
        eb['next_values'][n] = nv * (1.0 - (tc > 0).to(dtype)).unsqueeze(-1)
    comb = cfg['task_reward_w'] * eb['rewards'] + cfg['disc_reward_w'] * eb['disc_rewards']
    adv = O.discount_values(eb['dones'].to(dtype), eb['values'], comb, eb['next_values'], cfg['gamma'], cfg['tau'])
    returns = O.swap_and_flatten01(adv + eb['values'])
    values = O.swap_and_flatten01(eb['values'])
    advantages = O.calc_advs(returns, values)
    vr = O.RMS(1)
    vr.mean, vr.var, vr.count = (hrms['reward_mean_std'][k].clone() for k in ('running_mean', 'running_var', 'count'))
    vr.update(values); vr.update(returns)       # prepare_dataset: value_mean_std in train mode on values, then returns
    return dict(eb=eb, llc_actions=llc_actions, returns=returns, advantages=advantages,
                value_rms_after={'running_mean': vr.mean, 'running_var': vr.var, 'count': vr.count})
