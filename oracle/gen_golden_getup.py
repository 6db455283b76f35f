"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/getup_reset.pt by executing the UNMODIFIED reference episode-reset methods of
HumanoidAMP and HumanoidAMPGetup (env/tasks/humanoid_amp.py, humanoid_amp_getup.py), called unbound on a stand-in `self` (an instance made
without __init__, as oracle/gen_golden_hrl_tasks.py does): the synthetic-table reference MotionLib of gen_golden.gen_motion_lib with
non-uniform clip weights, Isaac Gym's tensor layouts (_root_states [2N, 13] with two actors per env, _dof_state [N * D, 2]), a no-op gym for
_reset_env_tensors and a stubbed _refresh_sim_tensors.  torch.bernoulli / multinomial / rand / randint_like are wrapped so every draw is
recorded and mapped back to its env row.
Usage: python oracle/gen_golden_getup.py"""
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_harness as rh          # noqa: E402
import ase_oracle as O            # noqa: E402
import getup_oracle as GO         # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), 'tests', 'golden')
N, J, D, S, STEP = 24, 17, 31, 10, 140
DT = 1.0 / 30.0
WEIGHTS = [4.0, 1.0, 2.0, 3.0]
MODES = {'default': ('Default', False), 'start': ('Start', False), 'random': ('Random', False), 'hybrid': ('Hybrid', False),
         'hybrid_getup': ('Hybrid', True)}


class _Draws:
    def __init__(self):
        self.log = {'bernoulli': [], 'multinomial': [], 'rand': [], 'randint_like': []}

    def __enter__(self):
        self._orig = {k: getattr(torch, k) for k in self.log}
        for k in self.log:
            def wrap(*a, _k=k, **kw):
                x = self._orig[_k](*a, **kw); self.log[_k].append(x.clone()); return x
            setattr(torch, k, wrap)
        return self

    def __exit__(self, *exc):
        for k, f in self._orig.items():
            setattr(torch, k, f)


def _ref_motion_lib():
    from utils.motion_lib import MotionLib
    mt = O.synthetic_motion_tables(seed=7)
    ml = MotionLib.__new__(MotionLib)
    ml._dof_body_ids = O.DOF_BODY_IDS_SWORD_SHIELD; ml._dof_offsets = O.DOF_OFFSETS_SWORD_SHIELD; ml._num_dof = 31
    ml._key_body_ids = torch.tensor(O.KEY_BODY_IDS_SWORD_SHIELD); ml._device = 'cpu'
    ml.gts, ml.grs, ml.lrs, ml.grvs, ml.gravs, ml.dvs = mt.gts, mt.grs, mt.lrs, mt.grvs, mt.gravs, mt.dvs
    ml._motion_lengths, ml._motion_num_frames, ml._motion_dt, ml.length_starts = mt.lengths, mt.num_frames, mt.dts, mt.length_starts
    w = torch.tensor(WEIGHTS)
    ml._motion_weights = w / w.sum()

    class _M: num_joints = 17
    ml._motions = [_M()]
    return ml, mt


def _inputs(g):
    """The env state before the reset (shared by every mode)."""
    body = torch.randn(N, J, 13, generator=g)
    body[..., 3:7] = torch.nn.functional.normalize(body[..., 3:7], dim=-1)
    body[:, 0, 2] = 0.3 + 0.8 * torch.rand(N, generator=g)
    return dict(
        body=body, root=torch.randn(N, 2, 13, generator=g), dof=torch.randn(N * D, 2, generator=g),
        init_root=torch.cat([torch.zeros(N, 2), torch.full((N, 1), 0.9), torch.tensor([[0., 0., 0., 1.]]).repeat(N, 1), torch.zeros(N, 6)], -1),
        init_dof_pos=0.1 * torch.randn(N, D, generator=g), init_dof_vel=torch.zeros(N, D),
        fall_root=torch.randn(N, 13, generator=g), fall_dof_pos=torch.randn(N, D, generator=g), fall_dof_vel=torch.zeros(N, D),
        progress=torch.randint(0, 300, (N,), generator=g), reset=(torch.rand(N, generator=g) < 0.5).long(),
        terminate=(torch.rand(N, generator=g) < 0.7).long(), counter=torch.randint(0, 3, (N,), generator=g).to(torch.int32),
        mask=(torch.rand(N, generator=g) < 0.75).to(torch.uint8))


def _stand_in(cls, ml, x, state_init, getup):
    from env.tasks.humanoid_amp import HumanoidAMP
    st = object.__new__(cls)
    st.device, st.num_envs, st.dt = 'cpu', N, DT
    st._state_init = HumanoidAMP.StateInit[state_init]
    st._hybrid_init_prob, st._num_amp_obs_steps = 0.5, S
    st._reset_default_env_ids, st._reset_ref_env_ids = [], []
    st._motion_lib = ml
    st._local_root_obs, st._root_height_obs = True, True
    st._dof_obs_size, st._dof_offsets = 78, O.DOF_OFFSETS_SWORD_SHIELD
    st._key_body_ids = torch.tensor(O.KEY_BODY_IDS_SWORD_SHIELD)
    st._root_states = x['root'].clone().view(2 * N, 13)
    st._humanoid_root_states = st._root_states.view(N, 2, 13)[..., 0, :]
    st._humanoid_actor_ids = 2 * torch.arange(N, dtype=torch.int32)
    st._dof_state = x['dof'].clone()
    st._dof_pos = st._dof_state.view(N, D, 2)[..., 0]
    st._dof_vel = st._dof_state.view(N, D, 2)[..., 1]
    st._initial_humanoid_root_states = x['init_root'].clone()
    st._initial_dof_pos, st._initial_dof_vel = x['init_dof_pos'].clone(), x['init_dof_vel'].clone()
    rbs = x['body'].clone()
    st._rigid_body_pos, st._rigid_body_rot, st._rigid_body_vel, st._rigid_body_ang_vel = rbs[..., 0:3], rbs[..., 3:7], rbs[..., 7:10], rbs[..., 10:13]
    st._amp_obs_buf = GO.amp_before(N, S, STEP)
    st._curr_amp_obs_buf, st._hist_amp_obs_buf = st._amp_obs_buf[:, 0], st._amp_obs_buf[:, 1:]
    st.obs_buf = GO.obs_before(N)
    st.progress_buf, st.reset_buf, st._terminate_buf = x['progress'].clone(), x['reset'].clone(), x['terminate'].clone()
    st.gym = types.SimpleNamespace(**{k: (lambda *a, **kw: None) for k in ('set_actor_root_state_tensor_indexed', 'set_dof_state_tensor_indexed',
                                                                          'set_dof_position_target_tensor_indexed')})
    st.sim = None
    st._refresh_sim_tensors = lambda: None
    if getup:
        st._recovery_episode_prob, st._recovery_steps, st._fall_init_prob = 0.2, 60, 0.1
        st._reset_fall_env_ids = []
        st._recovery_counter = x['counter'].clone()
        st._fall_root_states, st._fall_dof_pos, st._fall_dof_vel = x['fall_root'].clone(), x['fall_dof_pos'].clone(), x['fall_dof_vel'].clone()
    return st


def _per_env_draws(log, env_ids, terminate, state_init, getup):
    """Map the recorded draws back to env rows (the order of humanoid_amp_getup.py:78-103 and humanoid_amp.py:141-201)."""
    z8 = lambda: torch.zeros(N, dtype=torch.uint8)
    d = dict(recovery=z8(), fall=z8(), hybrid=z8(), motion_id=torch.zeros(N, dtype=torch.int32), phase=torch.zeros(N),
             fall_row=torch.zeros(N, dtype=torch.int32))
    bern = list(log['bernoulli'])
    nonfall = env_ids
    if getup:
        rec = bern.pop(0) == 1.0
        d['recovery'][env_ids] = rec.to(torch.uint8)
        nonrec = env_ids[~(rec & (terminate[env_ids] == 1))]
        fall = bern.pop(0) == 1.0
        d['fall'][nonrec] = fall.to(torch.uint8)
        fall_ids = nonrec[fall]
        if len(fall_ids) > 0:
            d['fall_row'][fall_ids] = log['randint_like'][0].to(torch.int32)
        nonfall = nonrec[~fall]
    ref_ids = nonfall
    if state_init == 'Default':
        ref_ids = nonfall[:0]
    elif state_init == 'Hybrid' and len(nonfall) > 0:
        h = bern.pop(0) == 1.0
        d['hybrid'][nonfall] = h.to(torch.uint8)
        ref_ids = nonfall[h]
    assert not bern
    if len(ref_ids) > 0:
        d['motion_id'][ref_ids] = log['multinomial'][0].to(torch.int32)
        if log['rand']:
            d['phase'][ref_ids] = log['rand'][0]
    return d


def _mode_mask(name, mask):
    """Start and Random reset every sixth env, plain Hybrid every third (each reference-init env stores nine AMP frames; this keeps the
    fixture small); Default and the getup case reset all flagged envs."""
    every = {'start': 6, 'random': 6, 'hybrid': 3}.get(name, 1)
    return mask & (torch.arange(N) % every == 0).to(torch.uint8)


def gen_getup_reset():
    """Every mode resets the same env state; the AMP and observation buffers start from GO.amp_before / GO.obs_before.  Stored per mode:
    the draws per env, the init kinds, the env state after, AMP slot 0 of the reset envs and slots 1..S-1 of the reference-init envs (the
    generator checks that the other rows and slots are what the kernels promise: copies of slot 0, or untouched)."""
    humanoid, _, _ = rh.import_env_fns()
    from env.tasks.humanoid_amp import HumanoidAMP
    from env.tasks.humanoid_amp_getup import HumanoidAMPGetup
    ml, mt = _ref_motion_lib()
    g = torch.Generator().manual_seed(29)
    x = _inputs(g)
    b = x['body']
    obs_all = humanoid.compute_humanoid_observations_max(b[..., 0:3], b[..., 3:7], b[..., 7:10], b[..., 10:13], True, True)
    amp0, obs0 = GO.amp_before(N, S, STEP), GO.obs_before(N)
    out = dict(n=N, dt=DT, weights=torch.tensor(WEIGHTS), motion_seed=7, inputs=x, obs=obs_all[x['mask'].bool()], modes={})
    for name, (si, getup) in MODES.items():
        mask = _mode_mask(name, x['mask'])
        m = mask.bool()
        env_ids = mask.nonzero().flatten()
        for attempt in range(50):              # the getup case must show every init kind
            torch.manual_seed(1000 + 100 * len(out['modes']) + attempt)
            st = _stand_in(HumanoidAMPGetup if getup else HumanoidAMP, ml, x, si, getup)
            with _Draws() as dr:
                (HumanoidAMPGetup if getup else HumanoidAMP)._reset_envs(st, env_ids)
            draws = _per_env_draws(dr.log, env_ids, x['terminate'], si, getup)
            kind = GO.init_kinds(mask, x['terminate'] if getup else torch.zeros(N), draws, si)
            kinds = {int(k): int((kind == k).sum()) for k in range(5)}
            if not getup or all(kinds[k] > 0 for k in range(5)):
                break
        assert not getup or all(kinds[k] > 0 for k in range(5)), kinds
        print(name, 'kinds', kinds)
        ref, rv = kind == GO.REF, kind == GO.RECOVERY
        df = (kind == GO.DEFAULT) | (kind == GO.FALL)
        amp, obs = st._amp_obs_buf, st.obs_buf
        assert torch.equal(obs[~m], obs0[~m]) and torch.equal(obs[m], obs_all[m])
        assert torch.equal(amp[~m], amp0[~m]) and torch.equal(amp[rv, 1:], amp0[rv, 1:])
        assert torch.equal(amp[df, 1:], amp[df, 0:1].expand(-1, S - 1, -1))
        after = dict(root=st._humanoid_root_states.clone(), dof_pos=st._dof_pos.clone(), dof_vel=st._dof_vel.clone(),
                     counter=st._recovery_counter.clone() if getup else None, progress=st.progress_buf.clone(),
                     reset=st.reset_buf.to(torch.uint8), terminate=st._terminate_buf.to(torch.uint8),
                     amp0=amp[m, 0].clone(), amp_ref=amp[ref, 1:].clone())
        times = torch.zeros(N)
        if ref.any() and si != 'Start':
            times[ref] = draws['phase'][ref] * mt.lengths[draws['motion_id'][ref].long()]
        out['modes'][name] = dict(state_init=si, getup=getup, mask=mask, draws=draws, kind=kind, motion_time=times, after=after)
        neg = (times[ref].unsqueeze(-1) + (-DT * torch.arange(1, S)).float()) < 0
        out['modes'][name]['negative_times'] = int(neg.sum())
    # history times before the clip start (negative blend): always with Start, and with a drawn phase too
    assert out['modes']['start']['negative_times'] > 0
    assert any(out['modes'][k]['negative_times'] > 0 for k in ('random', 'hybrid', 'hybrid_getup'))
    used = torch.cat([r['draws']['motion_id'][r['kind'] == GO.REF] for r in out['modes'].values()])
    assert bool((used == 3).any())                                     # the two-frame clip is used
    out['recovery_seq'] = _recovery_sequence(g)
    torch.save(out, os.path.join(OUT, 'getup_reset.pt'))
    print('getup_reset.pt ok', os.path.getsize(os.path.join(OUT, 'getup_reset.pt')), 'bytes')


def _recovery_sequence(g, n=32, steps=6):
    """-> {counter_in, base_reset, base_terminate, counter, reset, terminate} [steps, n]: pre_physics_step's _update_recovery_count, then
    progress += 1 and the getup _compute_reset, `steps` times (humanoid_amp_getup.py:36-40,
    131-142, humanoid.py:430-436).  Env 0 recovers past max_episode_length - 1 and must not reset; env 1 counts 1 -> 0."""
    humanoid, _, _ = rh.import_env_fns()
    from env.tasks.humanoid_amp_getup import HumanoidAMPGetup
    st = object.__new__(HumanoidAMPGetup)
    st.max_episode_length, st._enable_early_termination = 300.0, True
    st._contact_body_ids = torch.tensor([13, 16])
    st._termination_heights = torch.full((J,), 0.15)
    st.progress_buf = torch.randint(0, 300, (n,), generator=g)
    st.progress_buf[0] = 297
    st._recovery_counter = torch.randint(0, 5, (n,), generator=g).to(torch.int32)
    st._recovery_counter[0], st._recovery_counter[1], st._recovery_counter[2] = 60, 2, 0
    st.reset_buf = torch.zeros(n, dtype=torch.long); st._terminate_buf = torch.zeros(n, dtype=torch.long)
    seq = []
    for _ in range(steps):
        c_in = st._recovery_counter.clone()
        HumanoidAMPGetup._update_recovery_count(st)
        st.progress_buf += 1
        contact = torch.randn(n, J, 3, generator=g) * 0.08
        contact[torch.rand(n, J, generator=g) < 0.1] *= 30.0
        pos = torch.randn(n, J, 3, generator=g); pos[..., 2] = 0.1 + torch.rand(n, J, generator=g)
        st._contact_forces, st._rigid_body_pos = contact, pos
        base_r, base_t = humanoid.compute_humanoid_reset(st.reset_buf, st.progress_buf, contact, st._contact_body_ids, pos, 300.0, True,
                                                         st._termination_heights)
        HumanoidAMPGetup._compute_reset(st)
        seq.append(dict(counter_in=c_in, base_reset=base_r.to(torch.uint8), base_terminate=base_t.to(torch.uint8),
                        counter=st._recovery_counter.clone(), reset=st.reset_buf.to(torch.uint8), terminate=st._terminate_buf.to(torch.uint8)))
    assert any(int(s['base_reset'][0]) == 1 and int(s['reset'][0]) == 0 for s in seq)        # timeout suppressed while recovering
    assert any(int(s['counter_in'][1]) == 1 and int(s['counter'][1]) == 0 for s in seq)
    assert any(bool(((s['base_reset'] == 1) & (s['reset'] == 0)).any()) for s in seq)
    return {k: torch.stack([s[k] for s in seq]) for k in seq[0]}              # [steps, n] each


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    gen_getup_reset()
