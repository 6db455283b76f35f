"""Cost of the device episode resets of HumanoidAMP / HumanoidAMPGetup at 4096 envs -- a report, not a gate.  Prints JSON lines with
  - reset_ms: CUDA-event time per sim step of the three reset launches (ase_amp_state_init, ase_amp_history_init, ase_recovery_step) with
    the getup constants, at the synthetic env's done rate (1/300) and with every env resetting;
  - eager_reset_ms: the same work in the reference's order on the same GPU tensors (bernoulli -> env_ids[mask] -> len() > 0, multinomial,
    index-list writes; get_motion_state and the AMP frames through the motion-library kernels), which syncs with the host several times;
  - ms_per_epoch of ASEAgent on SyntheticHumanoidEnv(state_init='Hybrid', getup=True) and on the default env (rollout graph captured);
and the GPU name and power limit the numbers were taken on.
    python tools/bench_getup_reset.py [--envs 4096] [--epochs 5] [--warmup 3] [--reps 200]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from ase_b200 import configs, ops  # noqa: E402
from ase_b200.agent import ASEAgent  # noqa: E402
from ase_b200.synthetic_env import SyntheticHumanoidEnv  # noqa: E402


def _gpu():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[torch.cuda.current_device()] if r.returncode == 0 else torch.cuda.get_device_name()


def _events(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn(); torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def _device_reset(env, mask):
    def run():
        env._init_state(mask)
        ops.amp_history_init(env._motion_lib, env._reset_kind, env._reset_motion_id, env._reset_motion_time, env._amp_obs_buf, env.dt)
        ops.recovery_step(env._recovery_counter, env.reset_buf, env._terminate_buf)
        env._reset_rng[1:].add_(1)
    return run


def _eager_reset(env, mask):
    """humanoid_amp_getup.py:78-129 + humanoid_amp.py:141-236 in their order, with index lists."""
    P, D, ml, dev = env._state_init_params, env.NUM_DOFS, env._motion_lib, env.device
    root, dpos, dvel, amp = env._body[:, 0], env._dof[:, :D], env._dof[:, D:], env._amp_obs_buf

    def run():
        env_ids = mask.nonzero().flatten()
        if len(env_ids) == 0:
            return
        rec = torch.bernoulli(torch.full((len(env_ids),), P['recovery_prob'], device=dev)) == 1.0
        rec = rec & (env._terminate_buf[env_ids] == 1)
        env._recovery_counter[env_ids[rec]] = P['recovery_steps']
        nonrec = env_ids[~rec]
        fall = torch.bernoulli(torch.full((len(nonrec),), P['fall_prob'], device=dev)) == 1.0
        fall_ids = nonrec[fall]
        if len(fall_ids) > 0:
            r = torch.randint_like(fall_ids, 0, env._fall_root.shape[0])
            root[fall_ids] = env._fall_root[r]; dpos[fall_ids] = env._fall_dof_pos[r]; dvel[fall_ids] = env._fall_dof_vel[r]
            env._recovery_counter[fall_ids] = P['recovery_steps']
        nonfall = nonrec[~fall]
        ref_ids = nonfall[:0]
        if len(nonfall) > 0:
            h = torch.bernoulli(torch.full((len(nonfall),), P['hybrid_prob'], device=dev)) == 1.0
            ref_ids, def_ids = nonfall[h], nonfall[~h]
            if len(ref_ids) > 0:
                ids = torch.multinomial(ml._motion_weights, len(ref_ids), replacement=True)
                t = torch.rand(len(ref_ids), device=dev) * ml._motion_lengths[ids]
                rp, rr, dp, rv, rw, dv, _ = ml.get_motion_state(ids, t)
                root[ref_ids] = torch.cat([rp, rr, rv, rw], dim=-1); dpos[ref_ids] = dp; dvel[ref_ids] = dv
            if len(def_ids) > 0:
                root[def_ids] = env._init_root[def_ids]; dpos[def_ids] = env._init_dof_pos[def_ids]; dvel[def_ids] = env._init_dof_vel[def_ids]
            env._recovery_counter[nonfall] = 0
        env.task.progress_buf[env_ids] = 0; env.reset_buf[env_ids] = 0; env._terminate_buf[env_ids] = 0
        df = torch.cat([def_ids, fall_ids]) if len(nonfall) > 0 else fall_ids
        if len(df) > 0:
            amp[df, 1:] = amp[df, 0:1]
        if len(ref_ids) > 0:
            tk = (t.unsqueeze(-1) + (-env.dt * torch.arange(1, env.AMP_STEPS, device=dev))).reshape(-1)
            amp[ref_ids, 1:] = ml.build_amp_obs_demo(ids.repeat_interleave(env.AMP_STEPS - 1), tk, env.dt, 1).view(len(ref_ids), env.AMP_STEPS - 1, -1)
        c = torch.clamp_min(env._recovery_counter - 1, 0)
        env._recovery_counter.copy_(c)
        on = c > 0
        env.reset_buf[on] = 0; env._terminate_buf[on] = 0
    return run


def _epoch_ms(env, a):
    cfg = configs.make('ase', device='cuda:0', vec_env=env, num_actors=a.envs, print_stats=False, seed=0, gemm_backend=2)
    ag = ASEAgent('bench', cfg)
    ag.init_tensors(); ag.obs = ag.env_reset(); ag._init_train()
    for _ in range(a.warmup):
        ag.update_epoch(); ag.train_epoch()
    ms = _events(lambda: (ag.update_epoch(), ag.train_epoch()), a.epochs)
    return ms, ag._rollout_graph is not None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--envs', type=int, default=4096)
    ap.add_argument('--epochs', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reps', type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_getup_reset: no CUDA device (this measures the GPU; there is nothing to report without one)')
    gpu = _gpu()
    torch.manual_seed(0)
    env = SyntheticHumanoidEnv(a.envs, device='cuda', seed=0, state_init='Hybrid', getup=True)
    env.reset()
    for label, p in (('done_rate', env.done_prob), ('full_reset', 1.0)):
        mask = (torch.rand(a.envs, device='cuda') < p).to(torch.uint8)
        env._terminate_buf.copy_(mask)
        rec = dict(case=label, envs=a.envs, reset_envs=int(mask.sum()), reset_ms=round(_events(_device_reset(env, mask), a.reps), 5),
                   eager_reset_ms=round(_events(_eager_reset(env, mask), a.reps), 5), gpu=gpu)
        print(json.dumps(rec), flush=True)
    del env
    for label, kw in (('getup_hybrid', dict(state_init='Hybrid', getup=True)), ('default', {})):
        torch.manual_seed(0)
        env = SyntheticHumanoidEnv(a.envs, device='cuda', seed=0, **kw)
        ms, captured = _epoch_ms(env, a)
        print(json.dumps(dict(case='ase_epoch', env=label, envs=a.envs, ms_per_epoch=round(ms, 3), rollout_graph=captured, gpu=gpu)), flush=True)
        del env
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
