"""TEST INFRASTRUCTURE ONLY.  Generates the HRL-task fixtures by executing the UNMODIFIED reference (the checkout named by
ASE_REFERENCE_ROOT, through oracle/shims), as oracle/gen_golden.py does for the rest of tests/golden:
  tests/golden/task_{heading,location,reach,strike}.pt   (gen_hrl_tasks)
  tests/golden/checkpoint_layout_hlc_tasks.json          (gen_hlc_checkpoint_layouts)
Usage: python oracle/gen_golden_hrl_tasks.py [gen_hrl_tasks] [gen_hlc_checkpoint_layouts]"""
import json
import math
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_harness as rh          # noqa: E402
import ase_oracle as O            # noqa: E402
import hrl_tasks_oracle as T      # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), 'tests', 'golden')


def _upright_roots(n, g, actors=1):
    """Root states [n, actors, 13] whose rotation is a yaw times a tilt of at most ~0.3 rad (mostly-upright heading: a root whose x axis is
    vertical makes the heading angle ill-conditioned for any fp32 implementation)."""
    s = torch.randn(n, actors, 13, generator=g)
    yaw = (torch.rand(n, actors, generator=g) * 2 - 1) * math.pi
    tilt = torch.nn.functional.normalize(torch.cat([0.15 * torch.randn(n, actors, 3, generator=g), torch.ones(n, actors, 1)], dim=-1), dim=-1)
    qy = torch.stack([torch.zeros_like(yaw), torch.zeros_like(yaw), torch.sin(yaw / 2), torch.cos(yaw / 2)], dim=-1)
    s[..., 3:7] = torch.nn.functional.normalize(O.quat_mul(qy, tilt), dim=-1)
    return s


class _Draws:
    """torch.rand / torch.randint wrapped so a reference method's draws are recorded in call order."""
    def __init__(self):
        self.rand, self.randint = [], []

    def __enter__(self):
        self._r, self._ri = torch.rand, torch.randint
        def rand(*a, **k):
            x = self._r(*a, **k); self.rand.append(x.clone()); return x
        def randint(*a, **k):
            x = self._ri(*a, **k); self.randint.append(x.clone()); return x
        torch.rand, torch.randint = rand, randint
        return self

    def __exit__(self, *exc):
        torch.rand, torch.randint = self._r, self._ri

    def per_env(self):
        """-> (u [n,4]: column k = each env's k-th uniform, steps [n] or None)"""
        cols = [c for x in self.rand for c in (x.unsqueeze(-1) if x.dim() == 1 else x).unbind(-1)]
        u = torch.stack(cols + [torch.zeros_like(cols[0])] * (4 - len(cols)), dim=-1)
        return u, (self.randint[0] if self.randint else None)


def gen_hrl_tasks():
    """The location / reach / strike tasks (env/tasks/humanoid_{location,reach,strike}.py): their jit observation, reward and strike-reset
    functions on seeded inputs with edge rows, and the target resampling methods of all four HRL tasks (_update_task / _reset_task /
    strike _reset_target) called unbound on a stand-in `self`, with their torch.rand / torch.randint draws recorded: each draw, the env rows it
    went to, the target state before and after.  -> tests/golden/task_{heading,location,reach,strike}.pt"""
    import types
    rh.import_env_fns()
    from env.tasks import humanoid_heading, humanoid_location, humanoid_reach, humanoid_strike
    g = torch.Generator().manual_seed(61)
    n, dt = 64, 1.0 / 30.0

    def resample_records(cls, task, make_self, targets, update=True):
        """update mode (progress vs change_steps) and reset mode (a subset, progress already 0) on a fresh stand-in each."""
        recs = {}
        for mode in (('update', 'reset') if update else ('reset',)):
            torch.manual_seed(100 + len(recs) + 7 * len(task))
            st = make_self()
            if mode == 'update':
                st.progress_buf = torch.randint(0, 300, (n,), generator=g)
                cs = st.progress_buf + torch.randint(-40, 40, (n,), generator=g)
                cs[:3] = st.progress_buf[:3] + torch.tensor([0, 1, -1])             # due exactly at the boundary / one step early / late
                getattr(st, targets['change_steps']).copy_(cs)
            else:
                st.progress_buf = torch.randint(0, 300, (n,), generator=g)
            ids = (getattr(st, targets['change_steps']) <= st.progress_buf).nonzero().flatten() if mode == 'update' else \
                torch.nonzero(torch.rand(n, generator=g) < 0.4).flatten()
            if mode == 'reset':
                st.progress_buf[ids] = 0                                            # _reset_env_tensors ran first
            before = {k: getattr(st, a).clone() for k, a in targets.items()}
            progress = st.progress_buf.clone()
            with _Draws() as d:
                if mode == 'update':
                    cls._update_task(st)
                elif task == 'strike':
                    cls._reset_target(st, ids)
                else:
                    cls._reset_task(st, ids)
            u, steps = d.per_env()
            recs[mode] = dict(env_ids=ids, progress=progress, u=u, steps=steps, before=before,
                              after={k: getattr(st, a).clone() for k, a in targets.items()})
        return recs

    def stand_in(cls, **attrs):
        st = types.SimpleNamespace(device='cpu', num_envs=n, **attrs)
        st._reset_task = lambda ids: cls._reset_task(st, ids)
        return st

    # ---- heading: resampling only (its obs / reward are in heading.pt)
    H = humanoid_heading.HumanoidHeading
    hp = dict(T.HRL_TASK_PARAMS['heading'])
    recs = resample_records(H, 'heading', lambda: stand_in(
        H, _enable_rand_heading=True, _tar_speed_min=hp['speed_min'], _tar_speed_max=hp['speed_max'],
        _heading_change_steps_min=hp['change_steps_min'], _heading_change_steps_max=hp['change_steps_max'],
        _tar_speed=torch.ones(n), _tar_dir=torch.tensor([[1.0, 0.0]]).repeat(n, 1), _tar_facing_dir=torch.tensor([[1.0, 0.0]]).repeat(n, 1),
        _heading_change_steps=torch.zeros(n, dtype=torch.int64)),
        dict(tar_dir='_tar_dir', tar_speed='_tar_speed', tar_face_dir='_tar_facing_dir', change_steps='_heading_change_steps'))
    torch.save(dict(params=hp, resample=recs), os.path.join(OUT, 'task_heading.pt'))

    # ---- location
    root = _upright_roots(n, g)[:, 0]
    prev = root[:, 0:3] - 0.05 * torch.randn(n, 3, generator=g)
    tar = root[:, 0:2] + 3.0 * torch.randn(n, 2, generator=g)
    tar[0] = root[0, 0:2]                                                       # target exactly at the root: zero tar_dir
    root[1, 0:2] = torch.tensor([1.0, 2.0]); tar[1] = torch.tensor([1.5, 2.5])   # pos_err == 0.5 exactly: outside dist_mask
    root[2, 0:2] = torch.tensor([1.0, 2.0]); tar[2] = torch.tensor([1.5, 2.4999])
    prev[3] = root[3, 0:3]                                                      # standing still: tar_dir_speed == 0 -> speed_mask
    lp = dict(T.HRL_TASK_PARAMS['location'])
    out = dict(root=root, prev=prev, tar_pos=tar, tar_speed=1.0, dt=dt, params=lp,
               obs=humanoid_location.compute_location_observations(root, tar),
               reward=humanoid_location.compute_location_reward(root[:, 0:3], prev, root[:, 3:7], tar, 1.0, dt))
    Lc = humanoid_location.HumanoidLocation
    out['resample'] = resample_records(Lc, 'location', lambda: stand_in(
        Lc, _humanoid_root_states=root, _tar_dist_max=lp['dist_max'], _tar_change_steps_min=lp['change_steps_min'],
        _tar_change_steps_max=lp['change_steps_max'], _tar_pos=torch.zeros(n, 2), _tar_change_steps=torch.zeros(n, dtype=torch.int64)),
        dict(tar_pos='_tar_pos', change_steps='_tar_change_steps'))
    torch.save(out, os.path.join(OUT, 'task_location.pt'))

    # ---- reach (reach body = sword, body 6 of the [N, 17, 13] rigid-body state)
    body = _upright_roots(n, g, actors=17)
    root = body[:, 0]
    tar = body[:, 6, 0:3] + 0.4 * torch.randn(n, 3, generator=g)
    tar[0] = body[0, 6, 0:3]                                                    # on the sword: reward 1
    rp = dict(T.HRL_TASK_PARAMS['reach'])
    out = dict(body=body, tar_pos=tar, reach_body=6, params=rp, obs=humanoid_reach.compute_location_observations(root, tar),
               reward=humanoid_reach.compute_reach_reward(body[:, 6, 0:3], root[:, 3:7], tar, 1.0, dt))
    Rc = humanoid_reach.HumanoidReach
    out['resample'] = resample_records(Rc, 'reach', lambda: stand_in(
        Rc, _tar_dist_max=rp['dist_max'], _tar_height_min=rp['height_min'], _tar_height_max=rp['height_max'],
        _tar_change_steps_min=rp['change_steps_min'], _tar_change_steps_max=rp['change_steps_max'],
        _tar_pos=torch.zeros(n, 3), _tar_change_steps=torch.zeros(n, dtype=torch.int64)),
        dict(tar_pos='_tar_pos', change_steps='_tar_change_steps'))
    torch.save(out, os.path.join(OUT, 'task_reach.pt'))

    # ---- strike: humanoid and target are actors 0 and 1 of _root_states [N, 2, 13] (row stride 26)
    rs = _upright_roots(n, g, actors=2)
    rs[:, 1, 3:7] = torch.nn.functional.normalize(torch.randn(n, 4, generator=g), dim=-1)
    up_ang = torch.tensor([0.0, 0.3, math.acos(0.2) - 1e-3, math.acos(0.2) + 1e-3, 1.5, math.pi / 2])      # around the success threshold
    ax = torch.nn.functional.normalize(torch.randn(len(up_ang), 3, generator=g) * torch.tensor([1.0, 1.0, 0.0]), dim=-1)
    rs[4:4 + len(up_ang), 1, 3:7] = O.quat_from_angle_axis(up_ang, ax)
    rs[0, 1, 0:2] = rs[0, 0, 0:2]                                              # target straight above the root: zero tar_dir
    prev = rs[:, 0, 0:3] - 0.05 * torch.randn(n, 3, generator=g)
    sp = dict(T.HRL_TASK_PARAMS['strike'])
    out = dict(root_states=rs, prev=prev, dt=dt, params=sp,
               obs=humanoid_strike.compute_strike_observations(rs[:, 0], rs[:, 1]),
               reward=humanoid_strike.compute_strike_reward(rs[:, 1, 0:3], rs[:, 1, 3:7], rs[:, 0], prev, torch.zeros(n, 3), dt, 1.5))
    # strike termination
    N, J = 96, 17
    contact = torch.randn(N, J + 1, 3, generator=g) * 0.08                       # body J = the target's slot of the net-contact tensor
    contact[:, :J][torch.rand(N, J, generator=g) < 0.08] *= 30.0
    contact[:, J, 0:2] *= torch.where(torch.rand(N, 1, generator=g) < 0.5, 30.0, 1.0)
    pos = torch.randn(N, J, 3, generator=g); pos[..., 2] = 0.2 + torch.rand(N, J, generator=g) * 0.6
    heights = torch.full((J,), 0.15); heights[0] = 0.3
    progress = torch.randint(3, 310, (N,), generator=g)
    progress[:3] = torch.tensor([0, 1, 2])
    cids, sids = torch.tensor([13, 16]), torch.tensor(T.STRIKE_BODY_IDS_SWORD_SHIELD)
    contact[:11] = 0.0; pos[:11, :, 2] = 1.0                                     # the edge rows below: nothing else touches or is low
    hit = torch.tensor([40.0, 0.0, 0.0])
    for i in range(3):                                                       # progress 0 / 1 / 2 with a target hit and a non-strike contact
        contact[i, J] = hit; contact[i, 2] = torch.tensor([0.0, 5.0, 0.0])
    contact[3, J] = torch.tensor([1.0, -1.0, 0.0]); contact[3, 2] = torch.tensor([3.0, 0.0, 0.0])       # target force exactly at 1.0
    contact[4, J] = hit; contact[4, 2] = torch.tensor([0.0, 0.0, 1.0])                                  # non-strike force exactly at 1.0
    contact[5, J] = hit; contact[5, 6] = torch.tensor([9.0, 0.0, 0.0])                                  # only a strike body touches
    contact[6, J] = torch.tensor([0.0, 0.0, 50.0]); contact[6, 2] = torch.tensor([5.0, 0.0, 0.0])        # target force with only z
    contact[7, 3] = torch.tensor([0.1, 0.0, 0.0]); pos[7, 3, 2] = 0.0                                   # fall contact exactly at 0.1
    contact[8, 5] = torch.tensor([0.5, 0.0, 0.0]); pos[8, 5, 2] = 0.0; contact[8, J] = hit               # strike body low with force 0.5
    contact[9, J] = hit; contact[9, 13] = torch.tensor([9.0, 0.0, 0.0])                                 # only a contact body (foot) touches
    contact[10, 3] = torch.tensor([0.0, 0.5, 0.0]); pos[10, 3, 2] = 0.0                                 # fallen (contact + low body)
    progress[3:11] = 50
    progress[11:14] = torch.tensor([298, 299, 300])                           # the episode-length reset
    rst = dict(contact=contact[:, :J].contiguous(), tar_contact=contact[:, J].contiguous(), pos=pos, heights=heights, progress=progress,
               contact_body_ids=cids, strike_body_ids=sids, max_episode_length=300.0)
    for et in (True, False):
        r, t = humanoid_strike.compute_humanoid_reset(torch.zeros(N, dtype=torch.long), progress, contact[:, :J], cids, pos, contact[:, J], sids,
                                                      300.0, et, heights)
        rst[f'reset_{int(et)}'], rst[f'term_{int(et)}'] = r, t
    out['reset'] = rst
    Sc = humanoid_strike.HumanoidStrike

    def strike_self():
        rs2 = rs.clone()
        return stand_in(Sc, _humanoid_root_states=rs2[:, 0], _target_states=rs2[:, 1], _tar_dist_min=sp['dist_min'], _tar_dist_max=sp['dist_max'],
                        _near_dist=sp['near_dist'], _near_prob=sp['near_prob'])
    out['resample'] = resample_records(Sc, 'strike', strike_self, dict(tar_states='_target_states'), update=False)
    torch.save(out, os.path.join(OUT, 'task_strike.pt'))
    print('task_{heading,location,reach,strike}.pt ok', {k: int(v['term_1'].sum()) for k, v in [('strike', rst)]})


def gen_hlc_checkpoint_layouts():
    """Layout (keys, shapes, dtypes, optimizer state indices, hyper-parameter keys -- NO weights) of the location, reach and strike HLC
    checkpoints the reference ships (ase/data/models/ase_hlc_<task>_reallusion_sword_shield.pth), in the format of
    tests/golden/checkpoint_layout.json (oracle/gen_golden.py gen_checkpoint_layout)."""
    out = {}
    for task in ('location', 'reach', 'strike'):
        name = f'ase_hlc_{task}_reallusion_sword_shield'
        w = torch.load(os.path.join(rh.REF_ROOT, 'ase/data/models', name + '.pth'), map_location='cpu', weights_only=False)
        lay = {}
        for k, v in w.items():
            if k == 'optimizer':
                lay[k] = {'state': {str(i): {kk: (list(vv.shape), str(vv.dtype)) if torch.is_tensor(vv) else type(vv).__name__ for kk, vv in st.items()}
                                    for i, st in v['state'].items()},
                          'param_groups': [{kk: (type(vv).__name__ if kk != 'params' else list(vv)) for kk, vv in pg.items()} for pg in v['param_groups']]}
            elif isinstance(v, dict):
                lay[k] = {kk: (list(vv.shape), str(vv.dtype)) for kk, vv in v.items()}
            else:
                lay[k] = type(v).__name__
        out[name] = lay
    with open(os.path.join(OUT, 'checkpoint_layout_hlc_tasks.json'), 'w') as f:
        json.dump(out, f, indent=0, sort_keys=False)
    print('checkpoint_layout_hlc_tasks.json ok', {k: len(v['model']) for k, v in out.items()})


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    for name in (sys.argv[1:] or ['gen_hrl_tasks', 'gen_hlc_checkpoint_layouts']):
        globals()[name]()
