"""Stand-in for the Isaac Gym vec-env (run.py:100-145 RLGPUEnv over HumanoidAMP) for benchmarks and tests:
Isaac Gym is bypassed with synthetic rigid-body-state tensors of the named shape (BASELINE.json north_star),
everything downstream of the simulator -- compute_humanoid_observations_max, the 10-frame AMP observation
history, resets -- runs through the CUDA kernels exactly as post_physics_step would
(env/tasks/humanoid.py:430-440, env/tasks/humanoid_amp.py:50-59).

`state_source`:
  'device' : a pool of pre-generated states resident in HBM (bench `value`)
  'host'   : states arrive from PINNED HOST memory every step (bench `e2e`; H2D copy inside the step)

`task` (HumanoidHeading / HumanoidLocation / HumanoidReach / HumanoidStrike, env/tasks/humanoid_<task>.py): the task observation is
appended behind the humanoid features, the task reward replaces the zero reward, and targets are resampled on the device the way
_update_task / _reset_task / _reset_target do, with in-kernel Philox draws (no host sync, CUDA-graph capturable).  `heading_task=True` is
the older heading stand-in with FIXED targets (no resampling) and stays as it was."""
import numpy as np
import torch

from . import ops


class _Box:
    def __init__(self, low, high):
        self.low = np.asarray(low, dtype=np.float32); self.high = np.asarray(high, dtype=np.float32); self.shape = self.low.shape


class _Task:
    def __init__(self, n, device, task_obs_size=0):
        self.num_envs = n
        self.progress_buf = torch.zeros(n, dtype=torch.long, device=device)
        self.viewer = None
        self._task_obs_size = task_obs_size

    def get_task_obs_size(self):
        return self._task_obs_size


class SyntheticHumanoidEnv:
    NUM_BODIES, NUM_DOFS, AMP_STEPS, AMP_STEP_DIM = 17, 31, 10, 140

    def __init__(self, num_envs, device='cuda', seed=0, pool=8, state_source='device', done_prob=1.0 / 300.0,
                 local_root_obs=True, root_height_obs=True, demo_pool=8192, heading_task=False, dt=1.0 / 30.0, demo_source='motion_lib',
                 task=None):
        if task is not None and heading_task:
            raise ValueError("heading_task=True (fixed targets) and task=... (resampled targets) exclude each other")
        if task is not None and task not in ops.TASK_OBS_SIZE:
            raise ValueError(f"task must be one of {sorted(ops.TASK_OBS_SIZE)}, got {task!r}")
        self.device = torch.device(device)
        self.task_name = task
        self.num_envs = num_envs
        self.local_root_obs, self.root_height_obs = local_root_obs, root_height_obs
        self.state_source = state_source
        self.done_prob = done_prob
        self.heading_task, self.dt = heading_task, dt
        task_obs = 5 if heading_task else (ops.TASK_OBS_SIZE[task] if task else 0)      # HumanoidHeading: 5 task-obs floats
        self.task = _Task(num_envs, self.device, task_obs)
        self.env = self                      # agents reach vec_env.env.task / vec_env.env.fetch_amp_obs_demo
        self.num_humanoid_obs = 1 + 16 * 3 + 17 * 6 + 17 * 3 + 17 * 3
        self.num_obs = self.num_humanoid_obs + task_obs
        self.num_amp_obs = self.AMP_STEPS * self.AMP_STEP_DIM
        self.observation_space = _Box(-np.inf * np.ones(self.num_obs), np.inf * np.ones(self.num_obs))
        self.amp_observation_space = _Box(-np.inf * np.ones(self.num_amp_obs), np.inf * np.ones(self.num_amp_obs))
        self.action_space = _Box(-np.ones(self.NUM_DOFS), np.ones(self.NUM_DOFS))
        g = torch.Generator().manual_seed(seed)
        self._gen = torch.Generator(device=self.device).manual_seed(seed + 1) if self.device.type == 'cuda' else g
        n, J, D = num_envs, self.NUM_BODIES, self.NUM_DOFS
        pos = torch.randn(pool, n, J, 3, generator=g); pos[:, :, 0, 2] = 0.5 + 0.7 * torch.rand(pool, n, generator=g)
        rot = torch.nn.functional.normalize(torch.randn(pool, n, J, 4, generator=g), dim=-1)
        vel = torch.randn(pool, n, J, 3, generator=g); ang = torch.randn(pool, n, J, 3, generator=g)
        body = torch.cat([pos, rot, vel, ang], dim=-1).contiguous()                 # [pool, N, J, 13]
        dof = torch.cat([torch.rand(pool, n, D, generator=g) * 2 - 1, torch.randn(pool, n, D, generator=g) * 2], dim=-1).contiguous()
        self.h2d_bytes_per_step = 0
        if state_source == 'host':
            self._body_pool = body.pin_memory(); self._dof_pool = dof.pin_memory()
            self.h2d_bytes_per_step = body[0].numel() * 4 + dof[0].numel() * 4
        else:
            self._body_pool = body.to(self.device); self._dof_pool = dof.to(self.device)
        self._pool = pool
        self._t = 0
        self._body = torch.empty(n, J, 13, device=self.device)      # what gym.acquire_rigid_body_state_tensor would expose
        self._dof = torch.empty(n, 2 * D, device=self.device)
        self.obs_buf = torch.zeros(n, self.num_obs, device=self.device)
        self._amp_obs_buf = torch.zeros(n, self.AMP_STEPS, self.AMP_STEP_DIM, device=self.device)
        self.rew_buf = torch.zeros(n, device=self.device)
        self.reset_buf = torch.zeros(n, dtype=torch.uint8, device=self.device)
        self._terminate_buf = torch.zeros(n, dtype=torch.uint8, device=self.device)
        self._done_bool = torch.zeros(n, dtype=torch.bool, device=self.device); self._term_bool = torch.zeros(n, dtype=torch.bool, device=self.device)
        self.extras = {}
        # demo AMP observations.  'motion_lib': synthetic clips in MotionLib's table format, sampled and turned into 10-frame AMP
        # observations by the ase_amp_obs_demo kernel every fetch (what HumanoidAMP.fetch_amp_obs_demo does, humanoid_amp.py:64-83);
        # 'pool': a fixed pool of rows built once by the AMP-obs kernel.
        self.demo_source = demo_source
        if demo_source == 'motion_lib':
            self._motion_lib = self._synthetic_motion_lib(g)
        dn = demo_pool
        dpos = torch.randn(dn, J, 3, generator=g); dpos[:, 0, 2] = 0.8 + 0.1 * torch.rand(dn, generator=g)
        drot = torch.nn.functional.normalize(torch.randn(dn, J, 4, generator=g) * 0.3 + torch.tensor([0., 0., 0., 1.]), dim=-1)
        dbody = torch.cat([dpos, drot, 0.5 * torch.randn(dn, J, 3, generator=g), 0.5 * torch.randn(dn, J, 3, generator=g)], dim=-1).to(self.device)
        ddof_p = (torch.rand(dn, D, generator=g) - 0.5).to(self.device); ddof_v = torch.randn(dn, D, generator=g).to(self.device)
        self._demo_pool = torch.zeros(dn, self.AMP_STEPS, self.AMP_STEP_DIM, device=self.device)
        for _ in range(self.AMP_STEPS):
            ops.build_amp_observations(dbody, ddof_p, ddof_v, self._demo_pool, local_root_obs, root_height_obs, shift_history=True)
            dbody = dbody + 0.01 * torch.randn(dbody.shape, device=self.device, generator=self._gen)
            dbody[:, :, 3:7] = torch.nn.functional.normalize(dbody[:, :, 3:7], dim=-1)
        self._demo_pool = self._demo_pool.view(dn, -1)
        if heading_task:     # humanoid_heading.py:60-76 target direction / speed / facing direction per env
            th = torch.rand(num_envs, generator=g) * 6.2831853; fh = torch.rand(num_envs, generator=g) * 6.2831853
            self._tar_dir = torch.stack([torch.cos(th), torch.sin(th)], dim=-1).to(self.device)
            self._tar_face_dir = torch.stack([torch.cos(fh), torch.sin(fh)], dim=-1).to(self.device)
            self._tar_speed = (1.0 + 4.0 * torch.rand(num_envs, generator=g)).to(self.device)
            self._prev_root_pos = torch.zeros(num_envs, 3, device=self.device)
        if task is not None:
            self._init_task(seed)
        self._load_state()
        if heading_task or task is not None:
            self._prev_root_pos.copy_(self._body[:, 0, 0:3])
        if task is not None:      # every env starts with a sampled target (HumanoidAMPTask._reset_envs -> _reset_task at the first reset)
            self._resample_task(self._all_envs)
        self._compute_observations(shift=False)
        self._amp_obs_buf[:, 1:] = self._amp_obs_buf[:, 0:1]

    # ---- what RLGPUEnv exposes (run.py:100-145) -------------------------------------------------------
    def get_env_info(self):
        return {'action_space': self.action_space, 'observation_space': self.observation_space,
                'amp_observation_space': self.amp_observation_space}

    def _synthetic_motion_lib(self, g, clips=24):
        """Smooth random clips (1.3 - 6 s at 30 fps, upright root) in the flat per-frame layout of utils/motion_lib.py:65-89."""
        from .motion_lib import MotionLib
        J, D = self.NUM_BODIES, self.NUM_DOFS
        nf = torch.randint(40, 180, (clips,), generator=g)
        F = int(nf.sum())
        def smooth(shape_tail, scale):
            return torch.randn(F, *shape_tail, generator=g).cumsum(0) * scale
        gts = torch.randn(1, J, 3, generator=g) + smooth((J, 3), 0.01)
        gts[:, 0, 2] = 0.9 + 0.05 * torch.randn(F, generator=g)
        yaw = smooth((), 0.05)
        tilt = 0.1 * torch.randn(F, 2, generator=g)
        grs = torch.nn.functional.normalize(torch.randn(1, J, 4, generator=g) + smooth((J, 4), 0.03), dim=-1)
        grs[:, 0] = torch.nn.functional.normalize(torch.stack([tilt[:, 0], tilt[:, 1], torch.sin(yaw / 2), torch.cos(yaw / 2)], dim=-1), dim=-1)
        lrs = torch.nn.functional.normalize(torch.tensor([0., 0., 0., 1.]) + smooth((J, 4), 0.03), dim=-1)
        grvs, gravs, dvs = torch.randn(F, 3, generator=g), torch.randn(F, 3, generator=g), torch.randn(F, D, generator=g)
        return MotionLib(gts, grs, lrs, grvs, gravs, dvs, (nf - 1).float() / 30.0, nf, torch.full((clips,), 1.0 / 30.0), device=self.device)

    def fetch_amp_obs_demo(self, num_samples):
        if self.demo_source == 'motion_lib':
            return self._motion_lib.fetch_amp_obs_demo(num_samples, self.dt, self.AMP_STEPS, self.local_root_obs, self.root_height_obs)
        idx = torch.randint(0, self._demo_pool.shape[0], (num_samples,), device=self.device, generator=self._gen)
        return self._demo_pool[idx]

    def _load_state(self):
        i = self._t % self._pool
        self._body.copy_(self._body_pool[i], non_blocking=True)
        self._dof.copy_(self._dof_pool[i], non_blocking=True)
        self._t += 1

    def _compute_observations(self, shift, env_ids=None, env_mask=None, fill_history=False):
        D = self.NUM_DOFS
        ops.compute_humanoid_observations_max(self._body, self.local_root_obs, self.root_height_obs, out=self.obs_buf, env_ids=env_ids,
                                              env_mask=env_mask)
        if self.heading_task:      # humanoid_amp_task.py:51-64: task obs appended behind the humanoid features
            ops.compute_heading_observations(self._body[:, 0], self._tar_dir, self._tar_speed, self._tar_face_dir, out=self.obs_buf,
                                             col0=self.num_humanoid_obs)
        elif self.task_name is not None:
            self._compute_task_obs()
        ops.build_amp_observations(self._body, self._dof[:, :D], self._dof[:, D:], self._amp_obs_buf, self.local_root_obs,
                                   self.root_height_obs, shift_history=shift, env_ids=env_ids, env_mask=env_mask, fill_history=fill_history)

    def step(self, actions):
        """base_task.py:119-137: pre_physics_step (prev_root_pos; _update_task), physics (bypassed: next synthetic state), then
        post_physics_step."""
        if self.heading_task or self.task_name is not None:
            self._prev_root_pos.copy_(self._body[:, 0, 0:3])
        if self.task_name is not None and self.task_name != 'strike':
            self._resample_task(None)                       # _update_task: envs with progress >= change_steps
        self._load_state()
        self.task.progress_buf += 1
        self._compute_observations(shift=True)
        if self.heading_task:
            self.rew_buf = ops.compute_heading_reward(self._body[:, 0, 0:3], self._prev_root_pos, self._body[:, 0, 3:7], self._tar_dir,
                                                      self._tar_speed, self._tar_face_dir, self.dt)
        elif self.task_name is not None:
            self._compute_task_reward()
            self._task_rng[1:].add_(1)                      # every task draw of this step has been taken (a launch of its own)
        # (the default CUDA generator: it is CUDA-graph safe, a private torch.Generator is not)
        r = torch.rand(self.num_envs, device=self.device) if self.device.type == 'cuda' else torch.rand(self.num_envs, generator=self._gen)
        torch.lt(r, self.done_prob, out=self._done_bool); torch.lt(r, 0.5 * self.done_prob, out=self._term_bool)
        self.reset_buf.copy_(self._done_bool); self._terminate_buf.copy_(self._term_bool)        # terminate is a subset of dones
        self.extras['terminate'] = self._terminate_buf
        self.extras['amp_obs'] = self._amp_obs_buf.view(self.num_envs, -1)
        return self.obs_buf, self.rew_buf, self.reset_buf, self.extras

    def reset(self, env_ids=None):
        """vec_task_wrappers.py:24-26 -> task.reset(env_ids): obs + AMP history re-initialised for those envs
        (humanoid_amp.py:146-166,206-218 default-state path: history := current frame).  env_ids None resets EVERY env
        (humanoid.py:125-128), an empty list none."""
        if env_ids is None:
            env_ids = torch.arange(self.num_envs, device=self.device)
        if len(env_ids) > 0:
            ids = env_ids.to(torch.int32)
            self.task.progress_buf[env_ids] = 0
            mask = None
            if self.task_name is not None:
                mask = torch.zeros(self.num_envs, dtype=torch.uint8, device=self.device); mask[env_ids] = 1
            if self.task_name == 'strike':
                self._resample_task(mask)
            self._compute_observations(shift=False, env_ids=ids)
            self._amp_obs_buf[env_ids, 1:] = self._amp_obs_buf[env_ids, 0:1]
            if self.task_name is not None and self.task_name != 'strike':
                self._resample_task(mask)
        return self.obs_buf

    def reset_done(self, mask):
        """The same reset driven by a uint8 [N] mask on the device: no index list, no host sync (the agents use it when the env offers it)."""
        self.task.progress_buf.masked_fill_(mask.bool(), 0)
        if self.task_name == 'strike':            # _reset_target runs inside _reset_actors, before the observation is built
            self._resample_task(mask)
        self._compute_observations(shift=False, env_mask=mask, fill_history=True)
        if self.task_name is not None and self.task_name != 'strike':
            self._resample_task(mask)             # HumanoidAMPTask._reset_envs: _reset_task after the observation (it carries the old target)
        return self.obs_buf

    # ---- the location / reach / strike tasks and device-side resampling for all four (task=...) ------------------------------------
    def _init_task(self, seed):
        n, dev = self.num_envs, self.device
        self._prev_root_pos = torch.zeros(n, 3, device=dev)
        self._tar_change_steps = torch.zeros(n, dtype=torch.int64, device=dev)
        self._all_envs = torch.ones(n, dtype=torch.uint8, device=dev)
        self._task_rng = torch.tensor([seed * 7919 + 104729, 0], dtype=torch.int64, device=dev)     # {seed, step counter} of the Philox stream
        t = self.task_name
        if t == 'heading':
            self._tar_dir = torch.zeros(n, 2, device=dev); self._tar_dir[:, 0] = 1.0
            self._tar_face_dir = self._tar_dir.clone()
            self._tar_speed = torch.ones(n, device=dev)
        elif t == 'location':
            self._tar_pos = torch.zeros(n, 2, device=dev)
        elif t == 'reach':
            self._tar_pos = torch.zeros(n, 3, device=dev)
        else:
            self._tar_states = torch.zeros(n, 13, device=dev)

    def _resample_task(self, mask):
        """mask None: update mode (_update_task); a uint8 [N] mask: reset mode for the flagged envs.  Update and reset draw from different
        Philox streams, so a step's two calls never share draws."""
        t = self.task_name
        tar = {'heading': getattr(self, '_tar_dir', None), 'strike': getattr(self, '_tar_states', None)}.get(t, getattr(self, '_tar_pos', None))
        ops.task_resample(t, tar, self.task.progress_buf, root_states=self._body[:, 0], reset_mask=mask,
                          tar_speed=getattr(self, '_tar_speed', None) if t == 'heading' else None,
                          tar_face_dir=getattr(self, '_tar_face_dir', None) if t == 'heading' else None,
                          change_steps=None if t == 'strike' else self._tar_change_steps, rng=self._task_rng, stream_id=0 if mask is None else 2)

    def _compute_task_obs(self):
        root, col0, t = self._body[:, 0], self.num_humanoid_obs, self.task_name
        if t == 'heading':
            ops.compute_heading_observations(root, self._tar_dir, self._tar_speed, self._tar_face_dir, out=self.obs_buf, col0=col0)
        elif t == 'location':
            ops.compute_location_observations(root, self._tar_pos, out=self.obs_buf, col0=col0)
        elif t == 'reach':
            ops.compute_reach_observations(root, self._tar_pos, out=self.obs_buf, col0=col0)
        else:
            ops.compute_strike_observations(root, self._tar_states, out=self.obs_buf, col0=col0)

    def _compute_task_reward(self):
        root, t = self._body[:, 0], self.task_name
        if t == 'heading':
            self.rew_buf = ops.compute_heading_reward(root[:, 0:3], self._prev_root_pos, root[:, 3:7], self._tar_dir, self._tar_speed,
                                                      self._tar_face_dir, self.dt)
        elif t == 'location':
            ops.compute_location_reward(root, self._prev_root_pos, self._tar_pos, 1.0, self.dt, out=self.rew_buf)      # tarSpeed: 1.0
        elif t == 'reach':
            ops.compute_reach_reward(self._body, self._tar_pos, out=self.rew_buf)
        else:
            ops.compute_strike_reward(self._tar_states, root, self._prev_root_pos, self.dt, out=self.rew_buf)

    def on_graph_replay(self, steps):
        """A captured rollout was replayed: advance the host-side step counter the capture baked in (the pool index pattern repeats
        every `pool` steps, so a rollout of a multiple of `pool` steps replays identically)."""
        assert steps % self._pool == 0, "CUDA-graph rollouts need horizon_length to be a multiple of the synthetic state pool"
        self._t += steps
