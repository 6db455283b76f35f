"""ms per evaluation-player step at 4096 envs on SyntheticHumanoidEnv: ASEPlayer, and HRLPlayer with llc_steps = 5 over a frozen full-size
LLC.  Each is timed two ways on the same GPU, alternating over several repetitions:
  device : ase_b200.player (mask-driven kernels, the status read once per window of player.WINDOW steps);
  eager  : the reference's player formulas in eager torch around the same network calls -- index lists from done.nonzero(), torch.randn
           latents and Normal noise, clamp / rescale_actions / F.normalize, and two .item() reads of the finished episodes' sums per step
           (common_player.py:65-117, ase_players.py:33-94, hrl_players.py:36-251).
Prints the card name and its power limit, then one JSON line.  Usage: python tools/bench_player.py [--envs 4096 --steps 64 --reps 5]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ase_b200 import configs                          # noqa: E402
from ase_b200 import player as PL                     # noqa: E402
from ase_b200.learner import Learner                  # noqa: E402
from ase_b200.synthetic_env import SyntheticHumanoidEnv   # noqa: E402


def _device_steps(pl, obs, k):
    for i in range(k):
        slot = i % pl._window
        if slot == 0:
            pl._records.zero_()
        obs = pl.env_reset()
        obs = pl._step(obs, slot)
        if slot == pl._window - 1:
            pl._read_window(pl._window)
    return obs


def _eager_steps(pl, obs, k, hrl):
    """The reference's per-step host logic: nonzero() index lists and .item() sums (host syncs), eager torch draws."""
    n, dev = pl.num_envs, pl.device
    cr = torch.zeros(n, device=dev); steps = torch.zeros(n, device=dev)
    done_indices = torch.empty(0, dtype=torch.long, device=dev)
    low, high = pl.actions_low, pl.actions_high
    for _ in range(k):
        obs = pl.env.reset(done_indices)
        if not hrl:
            lat = pl._ase_latents
            lat[done_indices] = torch.nn.functional.normalize(torch.randn(len(done_indices), lat.shape[1], device=dev), dim=-1)
            mu, _ = pl.model.eval_actor_critic(obs, lat, want_value=False)
            a = torch.distributions.Normal(mu, torch.exp(pl.model.sigma)).sample()
            act = torch.clamp(a, -1.0, 1.0) * ((high - low) / 2.0) + (high + low) / 2.0
            obs, r, done, _ = pl.env.step(act)
        else:
            mu, _ = pl.model.eval_actor_critic(obs, None, want_value=False)
            a = torch.clamp(torch.distributions.Normal(mu, torch.exp(pl.model.sigma)).sample(), -1.0, 1.0)
            z = torch.nn.functional.normalize(a, dim=-1)
            rewards, done_count = 0.0, 0.0
            for _t in range(pl._llc_steps):
                lmu, _ = pl._llc.eval_actor_critic(obs[..., :obs.shape[-1] - pl._task_size], z, want_value=False)
                obs, rr, dd, _ = pl.env.step(torch.clamp(lmu, -1.0, 1.0) * ((high - low) / 2.0) + (high + low) / 2.0)
                rewards = rewards + rr
                done_count = done_count + dd.float()
            r, done = rewards / pl._llc_steps, (done_count > 0).float()
        cr += r; steps += 1
        done_indices = done.nonzero(as_tuple=False)[:, 0]
        if len(done_indices) > 0:
            cr[done_indices].sum().item(); steps[done_indices].sum().item()
            cr = cr * (1.0 - done.float()); steps = steps * (1.0 - done.float())
    return obs


def _time(fn, k):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn(k)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--envs', type=int, default=4096)
    ap.add_argument('--steps', type=int, default=64)
    ap.add_argument('--reps', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_player needs a GPU"
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    print('gpu:', q or torch.cuda.get_device_name(0))
    np.random.seed(0)
    out = {'envs': args.envs, 'steps': args.steps, 'reps': args.reps, 'gpu': q}
    for name in ('ase', 'hrl'):
        env = SyntheticHumanoidEnv(args.envs, device='cuda', seed=1, done_prob=1.0 / 300.0, demo_pool=512, task='location' if name == 'hrl' else None)
        player_cfg = {'games_num': 10 ** 9, 'determenistic': False}
        if name == 'ase':
            pl = PL.ASEPlayer(configs.make('ase', vec_env=env, device='cuda:0', player=player_cfg))
        else:         # a full-size LLC in the reference initialisation, saved in the rl_games layout
            llc = Learner('ase', env.num_humanoid_obs, env.NUM_DOFS, 2, amp_dim=env.num_amp_obs, latent_dim=64, amp_batch=2, device='cuda')
            llc.init_reference(seed=1)
            ckpt = os.path.join(tempfile.mkdtemp(), 'llc.pth')
            torch.save(dict(llc.get_stats_weights(), model=llc.state_dict()), ckpt)
            del llc
            pl = PL.HRLPlayer(configs.make('hrl', vec_env=env, device='cuda:0', player=player_cfg, llc_steps=5, llc_checkpoint=ckpt))
        pl._n_games = 10 ** 12
        pl._calls = {'noise': 0, 'z': 0}
        pl._stat.zero_()
        if name == 'ase':
            pl._begin_run()
        obs = pl.env_reset(full=True)
        st = {'obs': obs}

        def dev(k):
            st['obs'] = _device_steps(pl, st['obs'], k)

        def eager(k):
            st['obs'] = _eager_steps(pl, st['obs'], k, name == 'hrl')
        dev(pl._window); eager(8)                        # warm-up: modules, FP16 plane scales, allocator
        d, e = [], []
        for _ in range(args.reps):
            d.append(_time(dev, args.steps)); e.append(_time(eager, args.steps))
        out[name] = {'device_ms_per_step': float(np.median(d)), 'eager_ms_per_step': float(np.median(e)), 'device_all': d, 'eager_all': e}
        print(name, 'device %.3f ms/step, eager %.3f ms/step' % (out[name]['device_ms_per_step'], out[name]['eager_ms_per_step']))
        del pl, env
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
