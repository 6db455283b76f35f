"""GPU tests of the device episode resets (ase_amp_state_init, ase_amp_history_init, ase_recovery_step): the kernels fed the reference's
recorded draws against its own resets (tests/golden/getup_reset.pt), reference-init history slots against ase_amp_obs_demo bit for bit,
untouched rows, the in-kernel Philox draws against oracle/getup_oracle.py, Isaac Gym's layouts against contiguous ones, the recovery
counter over the reference's multi-step sequence, and an ASE agent on SyntheticHumanoidEnv(state_init='Hybrid', getup=True)."""
import numpy as np
import pytest
import torch

import ase_oracle as O
import getup_oracle as GO
import golden_util as G

pytestmark = pytest.mark.gpu

D, S = 31, 10
MODES = ['default', 'start', 'random', 'hybrid', 'hybrid_getup']
# Worst error against the reference's fp32 CPU results, relative to max(1, |value|), measured on an H100 80GB HBM3 (700 W power limit):
# root 6.6e-7, dof_pos 9.2e-6 (acos / atan2 of the joint rotations), dof_vel 0, obs 8.9e-7, AMP rows 3.8e-5 (extrapolated blends of the
# history slots).  The bounds are about 4x those.
TOL = {'state': 4e-5, 'obs': 4e-6, 'amp': 1.5e-4}


def _motion_lib(fx):
    from ase_b200.motion_lib import MotionLib
    mt = O.synthetic_motion_tables(seed=fx['motion_seed'])
    return MotionLib(mt.gts, mt.grs, mt.lrs, mt.grvs, mt.gravs, mt.dvs, mt.lengths, mt.num_frames, mt.dts, motion_weights=fx['weights']), mt


def _run(fx, name, layout='gym', rng=None):
    """One reset of the fixture's inputs on the device (injected draws unless rng is given) -> dict of results on the CPU."""
    from ase_b200 import ops
    x, rec = fx['inputs'], fx['modes'][name]
    ml, _ = _motion_lib(fx)
    c = lambda t: t.clone().cuda()
    n = x['mask'].shape[0]
    if layout == 'gym':
        root_buf = c(x['root']); root = root_buf[:, 0]
        dof_buf = c(x['dof']).view(n, D, 2); dpos, dvel = dof_buf[..., 0], dof_buf[..., 1]
    else:
        root = c(x['root'][:, 0]).contiguous()
        dpos, dvel = c(x['dof'].view(n, D, 2)[..., 0]).contiguous(), c(x['dof'].view(n, D, 2)[..., 1]).contiguous()
    getup = rec['getup']
    prog, reset = c(x['progress']), c(x['reset']).to(torch.uint8)
    term = c(x['terminate']).to(torch.uint8)
    counter = c(x['counter']) if getup else None
    kind = torch.full((n,), 77, dtype=torch.uint8, device='cuda')
    mid = torch.full((n,), -1, dtype=torch.int32, device='cuda'); mtime = torch.zeros(n, device='cuda')
    d = {k: v.cuda() for k, v in rec['draws'].items()}
    params = dict(ops.STATE_INIT_PARAMS['getup' if getup else 'amp'], state_init=rec['state_init'])
    inj = {} if rng is not None else dict(recovery_in=d['recovery'] if getup else None, fall_in=d['fall'] if getup else None,
                                          hybrid_in=d['hybrid'], motion_id_in=d['motion_id'], phase_in=d['phase'],
                                          fall_row_in=d['fall_row'] if getup else None)
    mask = c(rec['mask'])
    ops.amp_state_init(ml, mask, root, dpos, dvel, prog, reset, term, kind, mid, mtime, init_root_states=c(x['init_root']),
                       init_dof_pos=c(x['init_dof_pos']), init_dof_vel=c(x['init_dof_vel']), fall_root_states=c(x['fall_root']),
                       fall_dof_pos=c(x['fall_dof_pos']), fall_dof_vel=c(x['fall_dof_vel']), recovery_counter=counter, rng=rng, **params, **inj)
    body = c(x['body'])
    obs, amp = GO.obs_before(n).cuda(), GO.amp_before(n, S).cuda()
    ops.compute_humanoid_observations_max(body, True, True, out=obs, env_mask=mask)
    ops.build_amp_observations(body, dpos, dvel, amp, True, True, shift_history=False, env_mask=mask)
    ops.amp_history_init(ml, kind, mid, mtime, amp, fx['dt'])
    torch.cuda.synchronize()
    out = dict(root=root, dof_pos=dpos, dof_vel=dvel, progress=prog, reset=reset, terminate=term, counter=counter, kind=kind,
               motion_id=mid, motion_time=mtime, obs=obs, amp=amp)
    return {k: (None if v is None else v.cpu()) for k, v in out.items()}


def _rel(got, want):
    return float(((got.double() - want.double()).abs() / want.double().abs().clamp_min(1.0)).max()) if got.numel() else 0.0


@pytest.mark.parametrize('name', MODES)
def test_injected_draws_match_reference(name):
    fx = G.load('getup_reset.pt')
    rec, want, x = fx['modes'][name], fx['modes'][name]['after'], fx['inputs']
    got = _run(fx, name)
    m = rec['mask'].bool()
    want_obs, want_amp = GO.fixture_buffers(fx, name)
    assert torch.equal(got['kind'][m], rec['kind'][m]) and torch.all(got['kind'][~m] == 0)
    for k in ('progress', 'reset', 'terminate') + (('counter',) if rec['getup'] else ()):
        assert torch.equal(got[k].to(want[k].dtype), want[k]), (name, k)
    ref = rec['kind'] == GO.REF
    assert torch.equal(got['motion_id'][ref], rec['draws']['motion_id'][ref])
    assert torch.equal(got['motion_time'][ref], rec['motion_time'][ref])
    errs = {k: _rel(got[k], want[k]) for k in ('root', 'dof_pos', 'dof_vel')}
    errs['obs'] = _rel(got['obs'][m], want_obs[m]); errs['amp'] = _rel(got['amp'][m], want_amp[m])
    print(f"\n{name} worst relative error vs reference: {errs}")
    for k, e in errs.items():
        assert e <= TOL['state' if k in ('root', 'dof_pos', 'dof_vel') else k], (name, k, e)
    # untouched rows: unflagged envs everywhere, recovery envs' state and history slots 1..S-1
    amp0, obs0 = GO.amp_before(m.shape[0], S), GO.obs_before(m.shape[0])
    assert torch.equal(got['root'][~m], x['root'][~m, 0]) and torch.equal(got['amp'][~m], amp0[~m]) and torch.equal(got['obs'][~m], obs0[~m])
    dof = x['dof'].view(-1, D, 2)
    assert torch.equal(got['dof_pos'][~m], dof[~m, :, 0]) and torch.equal(got['dof_vel'][~m], dof[~m, :, 1])
    rv = rec['kind'] == GO.RECOVERY
    assert torch.equal(got['root'][rv], x['root'][rv, 0]) and torch.equal(got['dof_pos'][rv], dof[rv, :, 0])
    assert torch.equal(got['amp'][rv, 1:], amp0[rv, 1:])
    if name == 'hybrid_getup':
        assert int(rv.sum()) > 0


@pytest.mark.parametrize('name', ['start', 'random', 'hybrid_getup'])
def test_reference_history_is_amp_obs_demo_bitwise(name):
    fx = G.load('getup_reset.pt')
    got = _run(fx, name)
    ml, _ = _motion_lib(fx)
    ref = got['kind'] == GO.REF
    ids, t = got['motion_id'][ref], got['motion_time'][ref]
    k = torch.arange(1, S)
    tk = t.unsqueeze(-1) + (-fx['dt'] * k).to(torch.float32)
    assert bool((tk < 0).any())                                               # negative times: extrapolated blends
    demo = ml.build_amp_obs_demo(ids.repeat_interleave(S - 1).cuda(), tk.reshape(-1).cuda(), fx['dt'], 1).cpu()
    assert torch.equal(got['amp'][ref, 1:].reshape(-1, demo.shape[1]), demo)


@pytest.mark.parametrize('name', MODES)
def test_gym_layout_equals_contiguous_layout(name):
    fx = G.load('getup_reset.pt')
    a, b = _run(fx, name, 'gym'), _run(fx, name, 'contiguous')
    for k in a:
        if a[k] is not None:
            assert torch.equal(a[k], b[k]), (name, k)


@pytest.mark.parametrize('seed,call', [(12345, 0), (2 ** 33 + 7, 2 ** 32 + 3), (-5, 2 ** 40)])
def test_philox_draws_match_oracle(seed, call):
    from ase_b200 import ops
    fx = G.load('getup_reset.pt')
    ml, mt = _motion_lib(fx)
    n, F = 4096, 64
    g = torch.Generator().manual_seed(3)
    term = (torch.rand(n, generator=g) < 0.5).to(torch.uint8)
    mask = (torch.rand(n, generator=g) < 0.9).to(torch.uint8)
    root = torch.zeros(n, 13, device='cuda'); dpos = torch.zeros(n, D, device='cuda'); dvel = torch.zeros(n, D, device='cuda')
    fall_root = torch.randn(F, 13, generator=g)
    kind = torch.zeros(n, dtype=torch.uint8, device='cuda'); mid = torch.zeros(n, dtype=torch.int32, device='cuda'); mtime = torch.zeros(n, device='cuda')
    rng = torch.tensor([seed, call], dtype=torch.int64, device='cuda')
    p = dict(ops.STATE_INIT_PARAMS['getup'])
    z = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype, device='cuda')
    args = (ml, mask.cuda(), root, dpos, dvel, z(n, dtype=torch.int64), z(n, dtype=torch.uint8), term.cuda(), kind, mid, mtime)
    kw = dict(init_root_states=z(n, 13), init_dof_pos=z(n, D), init_dof_vel=z(n, D), fall_root_states=fall_root.cuda(), fall_dof_pos=z(F, D),
              fall_dof_vel=z(F, D), recovery_counter=z(n, dtype=torch.int32), rng=rng, stream_id=4, **p)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')             # the reset takes no host round trip
    try:
        ops.amp_state_init(*args, **kw)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    d = GO.philox_draws(seed, call, 4, n, ml._motion_cdf.cpu(), F, p)
    want = GO.init_kinds(mask, term, d, 'Hybrid')
    assert torch.equal(kind.cpu(), want)
    ref, fl = want == GO.REF, want == GO.FALL
    assert torch.equal(mid.cpu()[ref], d['motion_id'][ref])
    assert torch.equal(mtime.cpu()[ref], d['phase'][ref] * mt.lengths[d['motion_id'][ref].long()])
    assert torch.equal(root.cpu()[fl], fall_root[d['fall_row'][fl].long()])
    assert int(ref.sum()) > 0 and int(fl.sum()) > 0 and int((want == GO.RECOVERY).sum()) > 0


def test_recovery_step_sequence():
    from ase_b200 import ops
    q = G.load('getup_reset.pt')['recovery_seq']
    for i in range(q['counter'].shape[0]):
        c, r, t = q['counter_in'][i].cuda(), q['base_reset'][i].cuda(), q['base_terminate'][i].cuda()
        ops.recovery_step(c, r, t)
        assert torch.equal(c.cpu(), q['counter'][i]) and torch.equal(r.cpu(), q['reset'][i]) and torch.equal(t.cpu(), q['terminate'][i])


def _getup_env(n=64, seed=5, done_prob=0.05):
    from ase_b200.synthetic_env import SyntheticHumanoidEnv
    return SyntheticHumanoidEnv(n, device='cuda', seed=seed, done_prob=done_prob, demo_pool=256, state_init='Hybrid', getup=True)


def test_synthetic_env_resets_suppress_dones_and_replay_in_a_graph():
    """Steps of SyntheticHumanoidEnv(state_init='Hybrid', getup=True): dones are 0 wherever the counter is positive after the step, reference
    envs carry their clip's frames in slots 1..S-1, every kind occurs; a captured reset equals an eager one from the same state."""
    env = _getup_env(n=2048, done_prob=0.2)
    env.reset()
    seen = set()
    for _ in range(30):
        _, _, dones, infos = env.step(torch.zeros(env.num_envs, D, device='cuda'))
        cnt = env._recovery_counter
        assert not bool(((cnt > 0) & (dones != 0)).any()) and not bool(((cnt > 0) & (infos['terminate'] != 0)).any())
        mask = dones.clone()
        env.reset_done(mask)
        kinds = env._reset_kind
        seen |= set(torch.unique(kinds).cpu().tolist())
        ref = kinds == GO.REF
        if bool(ref.any()):
            ids, t = env._reset_motion_id[ref], env._reset_motion_time[ref]
            k = torch.arange(1, S, device='cuda')
            tk = (t.unsqueeze(-1) + (-env.dt * k).to(torch.float32)).reshape(-1)
            demo = env._motion_lib.build_amp_obs_demo(ids.repeat_interleave(S - 1), tk, env.dt, 1)
            assert torch.equal(env._amp_obs_buf[ref, 1:].reshape(-1, demo.shape[1]), demo)
    assert seen == {0, 1, 2, 3, 4}, seen
    a, b = _getup_env(seed=9), _getup_env(seed=9)
    for e in (a, b):
        e.reset(); e._terminate_buf.fill_(1)
    mask = (torch.arange(64, device='cuda') % 3 != 0).to(torch.uint8)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        a.reset_done(mask)
        a._reset_rng[1:].add_(1)
    graph.replay()
    b.reset_done(mask); b._reset_rng[1:].add_(1)
    torch.cuda.synchronize()
    for k in ('obs_buf', '_amp_obs_buf', '_recovery_counter', '_reset_kind', '_body', '_dof', '_reset_rng'):
        assert torch.equal(getattr(a, k), getattr(b, k)), k


def test_ase_agent_trains_on_getup_env(capfd):
    """ASEAgent epochs on the getup env with the rollout captured in a CUDA graph; a replayed rollout never waits on the device."""
    from ase_b200 import configs
    from ase_b200.agent import ASEAgent
    torch.manual_seed(0)
    n, h = 64, 8
    env = _getup_env(n)
    cfg = configs.make('ase', device='cuda:0', vec_env=env, num_actors=n, horizon_length=h, minibatch_size=128, amp_minibatch_size=32,
                       mini_epochs=2, amp_obs_demo_buffer_size=2048, amp_replay_buffer_size=2048, amp_batch_size=64, print_stats=False)
    cfg['net_params']['mlp']['units'] = [128, 96, 64]
    cfg['net_params']['disc']['units'] = [128, 96, 64]
    ag = ASEAgent('t', cfg)
    ag.init_tensors(); ag.obs = ag.env_reset(); ag._init_train()
    for _ in range(4):                                   # the rollout graph is captured at the third epoch
        ag.update_epoch(); info = ag.train_epoch()
        for k, v in info.items():
            assert torch.isfinite(v).all(), k
    assert ag._rollout_graph is not None
    assert 'capture' not in capfd.readouterr().err
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        with torch.no_grad():
            ag.set_eval()
            ag._play_steps_device()
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert int(env._reset_rng[1]) == 5 * h             # one reset-draw step per sim step, graph replays included
