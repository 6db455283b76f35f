"""TEST INFRASTRUCTURE ONLY -- torch (CPU) restatement of the episode-reset kernels of ase_b200/csrc/reset_kernels.cu:
  state_init     ase_amp_state_init   (HumanoidAMP / HumanoidAMPGetup._reset_actors + the zeroing of _reset_env_tensors)
  history_init   ase_amp_history_init (HumanoidAMP._init_amp_obs + the getup override)
  recovery_step  ase_recovery_step    (HumanoidAMPGetup._update_recovery_count + its _compute_reset)
and of their Philox draws (philox_draws), on top of ase_oracle's motion library and oracle/philox_oracle.py.

Draws of env e from {seed, call}, stream sid (include/ase_b200.h):
    stream sid,     group 0, words x, y, z, w: recovery, fall and hybrid Bernoulli uniforms (u < p) and the phase
    stream sid,     group 1, word x: the clip-id uniform; clip id = the first m with u < cdf[m]
    stream sid + 1, group 0xFFFFFFFE, word x: the fall-bank row x % max(1, F)
every uniform through u_open = min(u_closed, 1 - 2^-24).  cdf is the fp32 cumsum of the normalised clip weights computed in fp64, last entry 1."""
import numpy as np
import torch

import ase_oracle as O
import philox_oracle as PX

NONE, DEFAULT, REF, FALL, RECOVERY = 0, 1, 2, 3, 4
STATE_INIT = {'Default': 0, 'Start': 1, 'Random': 2, 'Hybrid': 3}


def amp_before(n, steps=10, step_dim=140):
    """The AMP buffer the fixture's resets start from: every entry of slot s of env e is e + s / 16 (distinct per row and slot, and rebuilt
    here rather than stored)."""
    return (torch.arange(n).view(n, 1, 1) + torch.arange(steps).view(1, steps, 1) / 16.0).expand(n, steps, step_dim).float().contiguous()


def obs_before(n, dim=253):
    """The observation buffer the fixture's resets start from: row e holds -1 - e."""
    return (-1.0 - torch.arange(n).float()).view(n, 1).expand(n, dim).contiguous()


def fixture_buffers(fx, name):
    """The reference's obs [N, 253] and AMP [N, S, 140] buffers after reset `name` of tests/golden/getup_reset.pt, rebuilt from what the fixture
    stores: the obs and AMP slot 0 of the reset envs and slots 1..S-1 of the reference-init envs.  Default and fall envs repeat slot 0, the
    other rows and slots keep obs_before / amp_before (oracle/gen_golden_getup.py checks all of this against the reference's buffers)."""
    rec = fx['modes'][name]
    m, kind = rec['mask'].bool(), rec['kind']
    n = m.shape[0]
    obs = obs_before(n)
    obs[m] = fx['obs'][m[fx['inputs']['mask'].bool()]]
    amp = amp_before(n)
    amp[m, 0] = rec['after']['amp0']
    df = (kind == DEFAULT) | (kind == FALL)
    amp[df, 1:] = amp[df, 0:1]
    amp[kind == REF, 1:] = rec['after']['amp_ref']
    return obs, amp


def motion_cdf(weights):
    w = torch.as_tensor(weights, dtype=torch.float64)
    c = (w / w.sum()).cumsum(0)
    c[-1] = 1.0
    return c.to(torch.float32)


def philox_draws(seed, call, sid, n, cdf, num_fall, p):
    """-> per-env draw outcomes {recovery, fall, hybrid (uint8), motion_id (int32), phase (fp32), fall_row (int32)} as the kernel takes them."""
    x, y, z, w = PX.words(seed, call, sid, np.arange(n), 0)
    uc = PX.u01_open(PX.words(seed, call, sid, np.arange(n), 1)[0])
    cdf = np.asarray(cdf, np.float32)
    ids = np.searchsorted(cdf, uc, side='right')                  # first m with u < cdf[m]
    row = PX.words(seed, call, int(sid) + 1, np.arange(n), PX.GROUP_RANDINT)[0] % np.uint64(max(1, int(num_fall)))
    f32 = np.float32
    return dict(recovery=torch.from_numpy((PX.u01_open(x) < f32(p['recovery_prob'])).astype(np.uint8)),
                fall=torch.from_numpy((PX.u01_open(y) < f32(p['fall_prob'])).astype(np.uint8)),
                hybrid=torch.from_numpy((PX.u01_open(z) < f32(p['hybrid_prob'])).astype(np.uint8)),
                motion_id=torch.from_numpy(ids.astype(np.int32)), phase=torch.from_numpy(PX.u01_open(w).astype(np.float32)),
                fall_row=torch.from_numpy(row.astype(np.int32)))


def init_kinds(mask, terminate, draws, state_init):
    """The init kind of every env (NONE where the mask is 0), in the reference's order: recovery, fall, then by state_init."""
    m = torch.as_tensor(mask).bool()
    rec = (draws['recovery'] != 0) & (torch.as_tensor(terminate) != 0)
    fall = ~rec & (draws['fall'] != 0)
    si = STATE_INIT[state_init]
    ref = ~rec & ~fall & (torch.ones_like(m) if si in (1, 2) else ((draws['hybrid'] != 0) if si == 3 else torch.zeros_like(m)))
    kind = torch.full(m.shape, DEFAULT, dtype=torch.uint8)
    kind[ref] = REF; kind[fall] = FALL; kind[rec] = RECOVERY
    kind[~m] = NONE
    return kind


def state_init(mt, st, mask, draws, p):
    """st: dict of root [N,13], dof_pos / dof_vel [N,D], counter [N] int32 or None, progress, reset, terminate, init_* and fall_* banks.
    Returns a new dict with the kernel's outputs (kind, motion_id, motion_time included)."""
    out = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in st.items()}
    kind = init_kinds(mask, st['terminate'], draws, p['state_init'])
    n = kind.shape[0]
    ids, times = torch.zeros(n, dtype=torch.int32), torch.zeros(n, dtype=torch.float32)
    d = kind == DEFAULT
    out['root'][d], out['dof_pos'][d], out['dof_vel'][d] = st['init_root'][d], st['init_dof_pos'][d], st['init_dof_vel'][d]
    f = kind == FALL
    r = draws['fall_row'][f].long()
    if f.any():
        out['root'][f], out['dof_pos'][f], out['dof_vel'][f] = st['fall_root'][r], st['fall_dof_pos'][r], st['fall_dof_vel'][r]
    ref = kind == REF
    if ref.any():
        mid = draws['motion_id'][ref].long()
        t = torch.zeros(mid.shape[0]) if p['state_init'] == 'Start' else draws['phase'][ref] * mt.lengths[mid]
        rp, rr, dp, rv, rw, dv, _ = O.get_motion_state(mt, mid, t)
        out['root'][ref] = torch.cat([rp, rr, rv, rw], dim=-1)
        out['dof_pos'][ref], out['dof_vel'][ref] = dp, dv
        ids[ref], times[ref] = mid.to(torch.int32), t
    if out.get('counter') is not None:
        c = out['counter']
        c[(kind == RECOVERY) | f] = int(p['recovery_steps'])
        c[d | ref] = 0
    flagged = kind != NONE
    out['progress'][flagged] = 0; out['reset'][flagged] = 0; out['terminate'][flagged] = 0
    out.update(kind=kind, motion_id=ids, motion_time=times)
    return out


def history_init(mt, amp_buf, kind, motion_id, motion_time, dt):
    """amp_buf [N, S, F] after slot 0 was rebuilt -> a new buffer: DEFAULT / FALL repeat slot 0, REF get the clip at time + fp32(-dt * k)."""
    out = amp_buf.clone()
    S = out.shape[1]
    df = (kind == DEFAULT) | (kind == FALL)
    out[df, 1:] = out[df, 0:1]
    ref = kind == REF
    if ref.any():
        k = torch.arange(1, S)
        t = (motion_time[ref].unsqueeze(-1) + (-dt * k).to(torch.float32)).reshape(-1)
        ids = motion_id[ref].long().unsqueeze(-1).expand(-1, S - 1).reshape(-1)
        rp, rr, dp, rv, rw, dv, kp = O.get_motion_state(mt, ids, t)
        obs = O.build_amp_observations(rp, rr, rv, rw, dp, dv, kp, True, True, O.DOF_OFFSETS_SWORD_SHIELD)
        out[ref, 1:] = obs.reshape(int(ref.sum()), S - 1, -1)
    return out


def recovery_step(counter, reset, terminate):
    c = torch.clamp_min(counter - 1, 0)
    on = c > 0
    r, t = reset.clone(), terminate.clone()
    r[on] = 0; t[on] = 0
    return c.to(counter.dtype), r, t
