"""Device-side mirror of utils/motion_lib.py MotionLib for the training hot path: the flat per-frame tables live in
HBM, `get_motion_state` and `build_amp_obs_demo` (env/tasks/humanoid_amp.py:64-101) are single kernel launches.
Clip sampling (`sample_motions`, `sample_time`, motion_lib.py:99-118) is torch RNG plumbing.
Loading .npy clips through poselib (motion_lib.py:174-238) stays in the reference; `from_reference` adopts its tensors."""
import ctypes as C

import torch

from . import lib as L
from .lib import lib, check
from .ops import _p, _stream, DOF_OFFSETS_SWORD_SHIELD, KEY_BODY_IDS_SWORD_SHIELD

DOF_BODY_IDS_SWORD_SHIELD = [1, 2, 3, 4, 5, 7, 8, 11, 12, 13, 14, 15, 16]      # env/tasks/humanoid.py:191


class MotionLib:
    def __init__(self, gts, grs, lrs, grvs, gravs, dvs, motion_lengths, motion_num_frames, motion_dt, motion_weights=None,
                 dof_body_ids=DOF_BODY_IDS_SWORD_SHIELD, dof_offsets=DOF_OFFSETS_SWORD_SHIELD, key_body_ids=KEY_BODY_IDS_SWORD_SHIELD,
                 device='cuda'):
        dev = torch.device(device)
        f = lambda t: t.to(dev, torch.float32).contiguous()
        self.gts, self.grs, self.lrs, self.grvs, self.gravs, self.dvs = f(gts), f(grs), f(lrs), f(grvs), f(gravs), f(dvs)
        self._motion_lengths, self._motion_dt = f(motion_lengths), f(motion_dt)
        self._motion_num_frames = motion_num_frames.to(dev, torch.int32).contiguous()
        shifted = self._motion_num_frames.roll(1).clone(); shifted[0] = 0
        self.length_starts = shifted.cumsum(0).to(torch.int32).contiguous()
        w = torch.ones(len(motion_lengths)) if motion_weights is None else motion_weights
        self._motion_weights = (w / w.sum()).to(dev, torch.float32)
        # inverse-CDF table of the device resets (ase_amp_state_init): fp32 cumsum of the normalised weights, computed in fp64, last entry 1
        w64 = w.to(torch.float64)
        cdf = (w64 / w64.sum()).cumsum(0)
        cdf[-1] = 1.0
        self._motion_cdf = cdf.to(dev, torch.float32).contiguous()
        self.device = dev
        self._num_bodies, self._num_dof = self.gts.shape[1], dof_offsets[-1]
        self._nj, self._nk = len(dof_body_ids), len(key_body_ids)
        self._c_body = (C.c_int32 * self._nj)(*dof_body_ids)
        self._c_off = (C.c_int32 * (self._nj + 1))(*dof_offsets)
        self._c_key = (C.c_int32 * self._nk)(*key_body_ids)
        self._step_dim = 13 + 6 * self._nj + self._num_dof + 3 * self._nk

    @classmethod
    def from_reference(cls, ref_motion_lib, device='cuda'):
        """Adopt the tensors of an already-loaded reference MotionLib (utils/motion_lib.py:65-89)."""
        m = ref_motion_lib
        return cls(m.gts, m.grs, m.lrs, m.grvs, m.gravs, m.dvs, m._motion_lengths, m._motion_num_frames, m._motion_dt, m._motion_weights,
                   m._dof_body_ids, m._dof_offsets, m._key_body_ids.tolist(), device)

    def _params(self):
        return L.MotionLibParams(_p(self.gts), _p(self.grs), _p(self.lrs), _p(self.grvs), _p(self.gravs), _p(self.dvs), _p(self._motion_lengths),
                                 _p(self._motion_num_frames), _p(self._motion_dt), _p(self.length_starts), self._num_bodies, self._num_dof,
                                 self._nj, self._c_body, self._c_off, self._nk, self._c_key)

    def num_motions(self):
        return self._motion_lengths.shape[0]

    def sample_motions(self, n):
        return torch.multinomial(self._motion_weights, num_samples=n, replacement=True)

    def sample_time(self, motion_ids, truncate_time=None):
        phase = torch.rand(motion_ids.shape, device=self.device)
        motion_len = self._motion_lengths[motion_ids]
        if truncate_time is not None:
            motion_len = motion_len - truncate_time
        return phase * motion_len

    def get_motion_state(self, motion_ids, motion_times):
        n = motion_ids.shape[0]
        ids = motion_ids.to(self.device, torch.int32).contiguous(); t = motion_times.to(self.device, torch.float32).contiguous()
        e = lambda *s: torch.empty(*s, device=self.device, dtype=torch.float32)
        out = (e(n, 3), e(n, 4), torch.zeros(n, self._num_dof, device=self.device), e(n, 3), e(n, 3), e(n, self._num_dof), e(n, self._nk, 3))
        p = self._params()
        check(lib.ase_motion_state(C.byref(p), _p(ids), _p(t), n, *[_p(x) for x in out], _stream()), 'ase_motion_state')
        return out

    def build_amp_obs_demo(self, motion_ids, motion_times0, sim_dt, num_steps, local_root_obs=True, root_height_obs=True):
        n = motion_ids.shape[0]
        ids = motion_ids.to(self.device, torch.int32).contiguous(); t = motion_times0.to(self.device, torch.float32).contiguous()
        out = torch.empty(n, num_steps * self._step_dim, device=self.device, dtype=torch.float32)
        p = self._params()
        check(lib.ase_amp_obs_demo(C.byref(p), _p(ids), _p(t), n, float(sim_dt), num_steps, int(bool(local_root_obs)), int(bool(root_height_obs)),
                                   _p(out), _stream()), 'ase_amp_obs_demo')
        return out

    def fetch_amp_obs_demo(self, num_samples, sim_dt, num_steps, local_root_obs=True, root_height_obs=True):
        """env/tasks/humanoid_amp.py:64-83."""
        ids = self.sample_motions(num_samples)
        trunc = sim_dt * (num_steps - 1)
        t0 = self.sample_time(ids, truncate_time=trunc) + trunc
        return self.build_amp_obs_demo(ids, t0, sim_dt, num_steps, local_root_obs, root_height_obs)
