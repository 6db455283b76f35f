"""Cost of the four HRL tasks (heading, location, reach, strike) on the synthetic env at 4096 envs -- a report, not a gate.
For each SyntheticHumanoidEnv(task=...) it prints one JSON line with
  - ms_per_epoch: CUDA-event time of HRLAgent epochs (rollout replayed from its CUDA graph + update), full-size LLC and HLC;
  - task_step_ms: CUDA-event time of one sim step's task work on the device (update-mode resampling + task obs + task reward kernels);
  - oracle_task_step_ms: the same step done the reference's way with the oracle formulas, run eagerly on the same GPU tensors
    (nonzero() index list, torch.rand / randint draws, jit-style tensor expressions);
and the GPU name and power limit the numbers were taken on.
    python tools/bench_hrl_tasks.py [--envs 4096] [--epochs 5] [--warmup 3] [--reps 200] [--out results.jsonl]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import torch  # noqa: E402

import ase_oracle as O  # noqa: E402
import hrl_tasks_oracle as T  # noqa: E402
from ase_b200 import configs, ops  # noqa: E402
from ase_b200.agent import HRLAgent  # noqa: E402
from ase_b200.synthetic_env import SyntheticHumanoidEnv  # noqa: E402

TASKS = ['heading', 'location', 'reach', 'strike']


def _gpu():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[torch.cuda.current_device()] if r.returncode == 0 else torch.cuda.get_device_name()


def _events(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn(); torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def _task_step(env):
    """One sim step's task work as SyntheticHumanoidEnv.step does it (strike has no update-mode resampling)."""
    def run():
        if env.task_name != 'strike':
            env._resample_task(None)
        env._compute_task_obs()
        env._compute_task_reward()
        env._task_rng[1:].add_(1)
    return run


def _oracle_step(env):
    """The reference's pre_physics_step / post_physics_step task work with the oracle's formulas on the env's GPU tensors."""
    t, P = env.task_name, ops.TASK_PARAMS[env.task_name]
    root, prog = env._body[:, 0], env.task.progress_buf
    dev = root.device

    def run():
        if t != 'strike':
            ids = (prog >= env._tar_change_steps).nonzero(as_tuple=False).flatten()
            if len(ids) > 0:                                                  # host sync, as in _update_task
                u = torch.rand(len(ids), 4, device=dev)
                steps = torch.randint(P['change_steps_min'], P['change_steps_max'], (len(ids),), device=dev)
                new = T.task_resample(t, P, u, steps, root[ids], prog[ids])
                env._tar_change_steps[ids] = new['change_steps']
                if t == 'heading':
                    env._tar_dir[ids], env._tar_speed[ids], env._tar_face_dir[ids] = new['tar_dir'], new['tar_speed'], new['tar_face_dir']
                else:
                    env._tar_pos[ids] = new['tar_pos']
        if t == 'heading':
            O.compute_heading_observations(root, env._tar_dir, env._tar_speed, env._tar_face_dir)
            O.compute_heading_reward(root[:, 0:3], env._prev_root_pos, root[:, 3:7], env._tar_dir, env._tar_speed, env._tar_face_dir, env.dt)
        elif t == 'location':
            T.compute_location_observations(root, env._tar_pos)
            T.compute_location_reward(root[:, 0:3], env._prev_root_pos, root[:, 3:7], env._tar_pos, 1.0, env.dt)
        elif t == 'reach':
            T.compute_reach_observations(root, env._tar_pos)
            T.compute_reach_reward(env._body[:, ops.REACH_BODY_SWORD_SHIELD, 0:3], env._tar_pos)
        else:
            T.compute_strike_observations(root, env._tar_states)
            T.compute_strike_reward(env._tar_states[:, 0:3], env._tar_states[:, 3:7], root, env._prev_root_pos, env.dt)
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--envs', type=int, default=4096)
    ap.add_argument('--epochs', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reps', type=int, default=200)
    ap.add_argument('--tasks', default=','.join(TASKS))
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_hrl_tasks: no CUDA device (this measures the GPU; there is nothing to report without one)')
    gpu = _gpu()
    lines = []
    for task in a.tasks.split(','):
        torch.manual_seed(0)
        env = SyntheticHumanoidEnv(a.envs, device='cuda', seed=0, task=task)
        cfg = configs.make('hrl', device='cuda:0', vec_env=env, num_actors=a.envs, print_stats=False, seed=0, gemm_backend=2)
        ag = HRLAgent('bench', cfg)
        ag.init_tensors(); ag.obs = ag.env_reset(); ag._init_train()
        for _ in range(a.warmup):
            ag.update_epoch(); ag.train_epoch()
        captured = ag._rollout_graph is not None
        ms_epoch = _events(lambda: (ag.update_epoch(), ag.train_epoch()), a.epochs)
        rec = dict(task=task, envs=a.envs, obs_dim=ag.obs_shape[0], rollout_graph=captured, ms_per_epoch=round(ms_epoch, 3),
                   task_step_ms=round(_events(_task_step(env), a.reps), 5), oracle_task_step_ms=round(_events(_oracle_step(env), a.reps), 5),
                   gpu=gpu)
        print(json.dumps(rec), flush=True)
        lines.append(rec)
        del ag, env
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.writelines(json.dumps(r) + '\n' for r in lines)


if __name__ == '__main__':
    main()
