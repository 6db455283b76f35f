"""GPU tests of the location / reach / strike tasks and the device-side target resampling of all four HRL tasks: the kernels against the
reference's own outputs (tests/golden/task_*.pt), the resampling kernel fed the reference's recorded draws and with its own Philox draws,
HRLAgent epochs on SyntheticHumanoidEnv(task=...) with the rollout captured in a CUDA graph, the shipped HLC checkpoint layouts, and the
HLC learner at the three new input widths against the fp64 oracle."""
import pytest
import torch

import ase_oracle as O
import golden_util as G

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-4, 1e-5          # as test_heading_task_kernels_golden
TASKS = ['heading', 'location', 'reach', 'strike']
OBS = {'heading': 258, 'location': 255, 'reach': 256, 'strike': 268}


def _strided(rows, actors=2, slot=0):
    """rows [N, 13] as actor `slot` of a [N, actors, 13] buffer: a view with row stride 13 * actors."""
    buf = torch.full((rows.shape[0], actors, 13), float('nan'), device='cuda')
    buf[:, slot] = rows.cuda()
    return buf, buf[:, slot]


def _obs_into_wide_buffer(fn, size, n):
    """fn(out, col0) writes task obs at col0 = 253 of a 253 + size wide buffer: the task columns equal a plain call, the others stay."""
    buf = torch.full((n, 253 + size), 7.0, device='cuda')
    fn(buf, 253)
    assert torch.equal(buf[:, :253], torch.full((n, 253), 7.0, device='cuda'))
    return buf[:, 253:]


def test_location_kernels_golden():
    from ase_b200 import ops
    fx = G.load('task_location.pt')
    _, root = _strided(fx['root'])
    tar, prev = fx['tar_pos'].cuda(), fx['prev'].cuda()
    obs = ops.compute_location_observations(root, tar)
    assert torch.allclose(obs.cpu(), fx['obs'], rtol=RTOL, atol=ATOL)
    wide = _obs_into_wide_buffer(lambda out, c0: ops.compute_location_observations(root, tar, out=out, col0=c0), 2, root.shape[0])
    assert torch.equal(wide, obs)
    rew = ops.compute_location_reward(root, prev, tar, fx['tar_speed'], fx['dt'])
    assert torch.allclose(rew.cpu(), fx['reward'], rtol=RTOL, atol=ATOL)
    assert float(rew[0]) == pytest.approx(float(fx['reward'][0]))        # target exactly at the root: zero direction, not NaN


def test_reach_kernels_golden():
    from ase_b200 import ops
    fx = G.load('task_reach.pt')
    body = fx['body'].cuda()
    tar = fx['tar_pos'].cuda()
    big = torch.zeros(body.shape[0], 19, 13, device='cuda'); big[:, :17] = body      # a strided view of a wider rigid-body tensor
    obs = ops.compute_reach_observations(big[:, 0], tar)
    assert torch.allclose(obs.cpu(), fx['obs'], rtol=RTOL, atol=ATOL)
    wide = _obs_into_wide_buffer(lambda out, c0: ops.compute_reach_observations(big[:, 0], tar, out=out, col0=c0), 3, body.shape[0])
    assert torch.equal(wide, obs)
    rew = ops.compute_reach_reward(big[:, :17], tar, reach_body=fx['reach_body'])
    assert torch.allclose(rew.cpu(), fx['reward'], rtol=RTOL, atol=ATOL)


def test_strike_kernels_golden():
    from ase_b200 import ops
    fx = G.load('task_strike.pt')
    rs = fx['root_states'].cuda()                 # [N, 2, 13]: humanoid and target, row stride 26
    root, tar = rs[:, 0], rs[:, 1]
    assert root.stride(0) == 26 and tar.stride(0) == 26
    obs = ops.compute_strike_observations(root, tar)
    assert torch.allclose(obs.cpu(), fx['obs'], rtol=RTOL, atol=ATOL)
    wide = _obs_into_wide_buffer(lambda out, c0: ops.compute_strike_observations(root, tar, out=out, col0=c0), 15, root.shape[0])
    assert torch.equal(wide, obs)
    rew = ops.compute_strike_reward(tar, root, fx['prev'].cuda(), fx['dt'])
    assert torch.allclose(rew.cpu(), fx['reward'], rtol=RTOL, atol=ATOL)


def test_strike_reset_kernel_golden():
    from ase_b200 import ops
    r = G.load('task_strike.pt')['reset']
    N, J, _ = r['contact'].shape
    net = torch.zeros(N, J + 1, 3, device='cuda')                 # the net-contact tensor: the target is body J of each env
    net[:, :J] = r['contact'].cuda(); net[:, J] = r['tar_contact'].cuda()
    body = torch.zeros(N, J, 13, device='cuda'); body[..., 0:3] = r['pos'].cuda()
    is_contact = torch.zeros(J, dtype=torch.uint8, device='cuda'); is_contact[r['contact_body_ids']] = 1
    is_strike = torch.zeros(J, dtype=torch.uint8, device='cuda'); is_strike[r['strike_body_ids']] = 1
    for et in (True, False):
        reset, term = ops.compute_strike_reset(r['progress'].cuda(), net[:, :J], is_contact, is_strike, body, net[:, J], r['max_episode_length'], et,
                                               r['heights'].cuda())
        assert torch.equal(reset.cpu().long(), r[f'reset_{int(et)}']) and torch.equal(term.cpu().long(), r[f'term_{int(et)}']), et


def _resample_state(task, fx, rec):
    """-> (kwargs of ops.task_resample for the fixture's state 'before', {name: device tensor} of the targets)"""
    b = {k: v.clone().cuda() for k, v in rec['before'].items()}
    kw = dict(progress=rec['progress'].cuda())
    if task == 'strike':
        rs = fx['root_states'].clone().cuda()
        rs[:, 1] = b['tar_states']
        kw.update(root_states=rs[:, 0], tar=rs[:, 1])
        return kw, {'tar_states': rs[:, 1]}
    if task == 'location':
        kw['root_states'] = fx['root'].cuda()
    kw.update(tar=b['tar_dir' if task == 'heading' else 'tar_pos'], change_steps=b['change_steps'])
    if task == 'heading':
        kw.update(tar_speed=b['tar_speed'], tar_face_dir=b['tar_face_dir'])
    return kw, b


@pytest.mark.parametrize('task', TASKS)
def test_task_resample_with_reference_draws(task):
    """The reference's own draws injected: resampled targets equal its methods' output within ulps, change_steps exactly; update mode touches
    only the due envs, reset mode only the masked ones."""
    from ase_b200 import ops
    fx = G.load(f'task_{task}.pt')
    for mode, rec in fx['resample'].items():
        n = rec['progress'].shape[0]
        ids = rec['env_ids']
        u = torch.zeros(n, 4); u[ids] = rec['u']
        steps = None
        if rec['steps'] is not None:
            steps = torch.zeros(n, dtype=torch.int64); steps[ids] = rec['steps']
            steps = steps.cuda()
        kw, out = _resample_state(task, fx, rec)
        mask = None
        if mode == 'reset':
            mask = torch.zeros(n, dtype=torch.uint8, device='cuda'); mask[ids.cuda()] = 1
        ops.task_resample(task, reset_mask=mask, u_in=u.cuda(), steps_in=steps, params=fx['params'], **kw)
        for k, want in rec['after'].items():
            got = out[k].cpu()
            if want.dtype == torch.int64:
                assert torch.equal(got, want), (task, mode, k)
            else:
                assert torch.allclose(got, want, rtol=1e-6, atol=1e-6), (task, mode, k, float((got - want).abs().max()))
                keep = torch.ones(n, dtype=torch.bool); keep[ids] = False
                assert torch.equal(got[keep], want[keep]), (task, mode, k)


def _philox_case(task, n=4096, counter=0, seed=12345):
    from ase_b200 import ops
    g = torch.Generator().manual_seed(5)
    root = torch.randn(n, 13, generator=g).cuda()
    progress = torch.zeros(n, dtype=torch.int64, device='cuda')
    tar = torch.zeros(n, {'heading': 2, 'location': 2, 'reach': 3, 'strike': 13}[task], device='cuda')
    extra = {}
    if task == 'heading':
        extra = dict(tar_speed=torch.zeros(n, device='cuda'), tar_face_dir=torch.zeros(n, 2, device='cuda'))
    cs = None if task == 'strike' else torch.full((n,), -1, dtype=torch.int64, device='cuda')
    rng = torch.tensor([seed, counter], dtype=torch.int64, device='cuda')
    mask = torch.ones(n, dtype=torch.uint8, device='cuda')
    return dict(task=task, tar=tar, progress=progress, root_states=root, reset_mask=mask, change_steps=cs, rng=rng, **extra), ops


@pytest.mark.parametrize('task', TASKS)
def test_task_resample_philox_ranges_determinism_and_graph(task):
    kw, ops = _philox_case(task)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        ops.task_resample(**kw)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    first = {k: v.clone() for k, v in kw.items() if torch.is_tensor(v)}
    kw2, _ = _philox_case(task)
    ops.task_resample(**kw2)
    assert torch.equal(kw2['tar'], first['tar'])                     # same {seed, counter}: identical
    kw3, _ = _philox_case(task, counter=1)
    ops.task_resample(**kw3)
    assert not torch.equal(kw3['tar'], first['tar'])                 # another counter: other draws
    P = ops.TASK_PARAMS[task]
    tar, root = first['tar'].cpu(), first['root_states'].cpu()
    if task != 'strike':
        steps = first['change_steps'].cpu()
        assert int(steps.min()) >= P['change_steps_min'] and int(steps.max()) < P['change_steps_max']
        assert int(steps.max()) - int(steps.min()) > (P['change_steps_max'] - P['change_steps_min']) // 2
    if task == 'heading':
        sp = first['tar_speed'].cpu()
        assert float(sp.min()) >= P['speed_min'] and float(sp.max()) <= P['speed_max']
        assert torch.allclose(tar.norm(dim=-1), torch.ones(tar.shape[0]), atol=1e-6)
    elif task == 'location':
        d = tar - root[:, 0:2]
        assert float(d.abs().max()) <= P['dist_max'] * (1 + 1e-6)
    elif task == 'reach':
        assert float(tar[:, 0:2].abs().max()) <= P['dist_max'] and float(tar[:, 2].min()) >= 0.2 and float(tar[:, 2].max()) <= 2.0
    else:
        dist = (tar[:, 0:2] - root[:, 0:2]).norm(dim=-1)
        assert float(dist.min()) >= 0.5 - 1e-4 and float(dist.max()) <= 10.0 + 1e-4
        near = float((dist <= 1.5).float().mean())                   # near_prob 0.5 plus the far draws below 1.5 (~5 %)
        assert 0.45 < near < 0.65, near
        assert torch.all(tar[:, 2] == 0.9) and torch.all(tar[:, 7:] == 0.0)
        assert torch.allclose(tar[:, 3:7].norm(dim=-1), torch.ones(tar.shape[0]), atol=1e-6)
        assert float(tar[:, 3:5].abs().max()) == 0.0                 # a rotation about z only
    # CUDA graph: capture resample + the counter increment (a separate op), replay twice == two eager calls
    kg, _ = _philox_case(task)
    ke, _ = _philox_case(task)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.task_resample(**kg)
        kg['rng'][1:].add_(1)
    for _ in range(2):
        graph.replay()
        ops.task_resample(**ke)
        ke['rng'][1:].add_(1)
    torch.cuda.synchronize()
    assert int(kg['rng'][1]) == 2
    assert torch.equal(kg['tar'], ke['tar'])


def test_task_resample_update_mode_touches_only_due_envs():
    from ase_b200 import ops
    n = 1024
    progress = torch.arange(n, dtype=torch.int64, device='cuda') % 300
    cs = torch.full((n,), 150, dtype=torch.int64, device='cuda')
    tar = torch.full((n, 2), 3.0, device='cuda')
    rng = torch.tensor([7, 3], dtype=torch.int64, device='cuda')
    ops.task_resample('location', tar, progress, root_states=torch.zeros(n, 13, device='cuda'), change_steps=cs, rng=rng)
    due = (progress >= 150).cpu()
    assert torch.all(tar.cpu()[~due] == 3.0) and torch.all(cs.cpu()[~due] == 150)
    assert not torch.any(tar.cpu()[due] == 3.0)
    assert torch.all(cs.cpu()[due] - progress.cpu()[due] >= 100) and torch.all(cs.cpu()[due] - progress.cpu()[due] < 200)


# ------------------------------------------------------------------------------------------------------------------------------------
# the HRL agent on the synthetic env with each task
# ------------------------------------------------------------------------------------------------------------------------------------
def _hrl_agent(task, n=64, h=8, units=(128, 64), gemm_backend=0, **over):
    from ase_b200 import configs
    from ase_b200.agent import HRLAgent
    from ase_b200.synthetic_env import SyntheticHumanoidEnv
    env = SyntheticHumanoidEnv(n, device='cuda', seed=4, done_prob=0.05, demo_pool=256, task=task)
    cfg = configs.make('hrl', device='cuda:0', vec_env=env, num_actors=n, horizon_length=h, minibatch_size=128, mini_epochs=2, print_stats=False,
                       gemm_backend=gemm_backend, **over)
    cfg['net_params']['mlp']['units'] = list(units)
    cfg['llc_net_params'] = {'mlp': {'units': [128, 96, 64]}, 'disc': {'units': [128, 96, 64]}}
    return HRLAgent('t', cfg), env


@pytest.mark.parametrize('task', TASKS)
def test_hrl_agent_epoch_per_task(task, capfd):
    """HRLAgent epochs on SyntheticHumanoidEnv(task=...): observation width, finite training, the GAE returns against the oracle on the stored
    buffers, task rewards in [0, 1], targets resampled over the epochs, and the rollout captured in a CUDA graph (no eager fallback).

    The learner runs on the exact-fp32 SIMT backend here: this checks the env and the agent's plumbing.  On the FP16-plane backend (2) the
    location HLC at this toy size (units [128, 64], minibatch 128) raises the plane-scale overflow flag in its second epoch, because an
    actor gradient grows beyond the x117 window between two consecutive calls, and its actor gradients are then not finite.  That is a limit
    of the learner's scale prediction, unchanged by the task kernels; test_hlc_learner_at_task_widths covers backend 2 at the three widths."""
    torch.manual_seed(2)
    ag, env = _hrl_agent(task)
    assert ag.obs_shape[0] == OBS[task] and env.task.get_task_obs_size() == OBS[task] - 253
    ag.init_tensors(); ag.obs = ag.env_reset()
    tar0 = (env._tar_states if task == 'strike' else (env._tar_dir if task == 'heading' else env._tar_pos)).clone()
    for _ in range(4):                                   # the rollout graph is captured at the third epoch
        ag.update_epoch(); info = ag.train_epoch()
        for k, v in info.items():
            assert torch.isfinite(v).all(), (task, k)
    assert ag._rollout_graph is not None, task
    assert 'capture' not in capfd.readouterr().err
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')             # a replayed rollout (resampling included) never waits on the device
    try:
        with torch.no_grad():
            ag.set_eval()
            ag._play_steps_device()
    finally:
        torch.cuda.set_sync_debug_mode('default')
    with torch.no_grad():
        bd = ag.play_steps()
    eb = {k: v.cpu() for k, v in ag.experience_buffer.items()}
    assert eb['obses'].shape[-1] == OBS[task] and torch.isfinite(eb['obses']).all()
    assert float(eb['mus'].abs().max()) <= 1.0
    rew = 0.9 * eb['rewards'] + 0.1 * eb['disc_rewards']
    adv = O.discount_values(eb['dones'].float(), eb['values'], rew, eb['next_values'], 0.99, 0.95)
    assert torch.allclose(bd['returns'].cpu(), O.swap_and_flatten01(adv + eb['values']), rtol=1e-4, atol=1e-4)
    assert float(eb['rewards'].min()) >= 0.0 and float(eb['rewards'].max()) <= 1.0 + 1e-6
    tar1 = env._tar_states if task == 'strike' else (env._tar_dir if task == 'heading' else env._tar_pos)
    assert not torch.equal(tar0, tar1), task             # resets (and, except for strike, due envs) got new targets


def _hlc_checkpoint_from_layout(name, seed):
    """A random checkpoint with EXACTLY the layout of a shipped HLC checkpoint (tests/golden/checkpoint_layout_hlc_tasks.json, written by
    oracle/gen_golden_hrl_tasks.py from ase/data/models/*.pth): same keys, shapes, dtypes, optimizer state indices (the values as
    test_gpu_agent._checkpoint_from_layout makes them)."""
    import json, os
    lay = json.load(open(os.path.join(os.path.dirname(__file__), 'golden', 'checkpoint_layout_hlc_tasks.json')))[name]
    g = torch.Generator().manual_seed(seed)
    dt = {'torch.float32': torch.float32, 'torch.float64': torch.float64}
    w = {}
    for k, v in lay.items():
        if k == 'optimizer':
            st = {int(i): {'step': 6194400, 'exp_avg': 1e-3 * torch.randn(e['exp_avg'][0], generator=g),
                           'exp_avg_sq': 1e-6 * torch.rand(e['exp_avg_sq'][0], generator=g) + 1e-9} for i, e in v['state'].items()}
            w[k] = {'state': st, 'param_groups': [{'lr': 2e-5, 'betas': (0.9, 0.999), 'eps': 1e-8, 'weight_decay': 0.0, 'amsgrad': False,
                                                   'params': v['param_groups'][0]['params']}]}
        elif isinstance(v, dict):
            w[k] = {}
            for kk, (shape, dtype) in v.items():
                t = torch.randn(shape, generator=g, dtype=dt[dtype]) * (0.05 if dtype == 'torch.float32' else 1.0)
                if kk in ('running_var', 'count'):
                    t = t.abs() + 0.5
                if kk.endswith('sigma'):
                    t = torch.full(shape, -2.9)
                w[k][kk] = t
        else:
            w[k] = {'epoch': 129050, 'frame': 8355840000, 'last_mean_rewards': -100500, 'env_state': None}[k]
    return w, lay


@pytest.mark.parametrize('task', ['location', 'reach', 'strike'])
def test_hlc_checkpoint_layouts_restore_save_and_train(task, tmp_path):
    """restore / save round-trip of a random checkpoint with exactly the layout of ase_hlc_<task>_reallusion_sword_shield.pth, then an epoch."""
    from test_gpu_agent import _same_layout
    w, lay = _hlc_checkpoint_from_layout(f'ase_hlc_{task}_reallusion_sword_shield', seed=11)
    assert list(w['model']['a2c_network.actor_mlp.0.weight'].shape) == [1024, OBS[task]]
    fn = str(tmp_path / 'hlc.pth')
    torch.save(w, fn)
    ag, env = _hrl_agent(task, units=(1024, 512))
    ag.restore(fn)
    sd = ag.model.state_dict()
    for k, v in w['model'].items():
        assert torch.equal(sd[k].cpu(), v), k
    w2 = torch.load(ag.save(str(tmp_path / 'resaved')), map_location='cpu', weights_only=False)
    _same_layout(w2, lay)
    for k in w['model']:
        assert torch.equal(w2['model'][k], w['model'][k]), k
    ag.init_tensors(); ag.obs = ag.env_reset()
    ag.update_epoch(); info = ag.train_epoch()
    assert all(torch.isfinite(v).all() for v in info.values())


# ------------------------------------------------------------------------------------------------------------------------------------
# the HLC learner at the three new input widths: units [1024, 512], 64 actions, tanh mu
# ------------------------------------------------------------------------------------------------------------------------------------
HLC_CASES = {f'hlc_{t}': dict(kind='ppo', obs=OBS[t], act=64, units=(1024, 512), B=200, mu_tanh=True) for t in ('location', 'reach', 'strike')}


def _clip_decisions_stable(c, cfg, st, d):
    """No sample of the minibatch has its PPO ratio within 1e-4 of 1 +- e_clip (fp64 oracle: the clip fraction does not change when e_clip
    moves by +-1e-4).  A sample on that knife edge is clipped by whichever fp32 implementation rounds it over, and at 64 actions and
    B = 200 that one sample moves half the elements of the first actor layer's gradient beyond 1e-4 of its max: the minibatch seeds below
    are chosen so that no such sample occurs (with seeds 4100 / 4101 the strike width has one)."""
    fr = []
    for e in (-1e-4, 1e-4):
        cf = dict(cfg); cf['e_clip'] = cfg['e_clip'] + e
        s64 = O.LearnerState({k: v.double() for k, v in st.p.items()}, c['obs'], 0, 'ppo')
        s64.obs_rms = st.obs_rms.clone(); s64.obs_rms.mean, s64.obs_rms.var = s64.obs_rms.mean.double(), s64.obs_rms.var.double()
        r, _ = O.calc_gradients(s64, {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in d.items()}, cf, None,
                                apply_adam=False)
        fr.append(float(r['actor_clip_frac']))
    return fr[0] == fr[1]


@pytest.mark.parametrize('backend', [0, 2])
@pytest.mark.parametrize('name', list(HLC_CASES))
def test_hlc_learner_at_task_widths(name, backend):
    """Two teacher-forced calc_gradients steps against the fp32 and fp64 oracle with the bounds of the ppo_tanh_narrow case of
    tests/test_gpu_learner_shapes.py."""
    from test_gpu_fullsize import _three_way, _threads, _sync64
    from test_gpu_learner import _cuda, _check_vs_oracle_twin
    from test_learner_shapes_cpu import oracle_cfg, learner_kwargs, states, minibatch
    from test_gpu_learner_shapes import _check_adam, _plane_flags
    from ase_b200 import Learner
    _threads()
    c = HLC_CASES[name]
    cfg = oracle_cfg(c)
    P, st, st64 = states(c, seed=31)
    ln = Learner(**learner_kwargs(c, cfg), gemm_backend=backend)
    ln.load_named(P)
    for s in range(2):
        when = f'{name} backend {backend} step {s}'
        d, _ = minibatch(c, st, cfg, seed=4300 + s)
        assert _clip_decisions_stable(c, cfg, st, d), when
        out = ln.calc_gradients(_cuda(d), None)
        res, g32 = O.calc_gradients(st, d, cfg, None, apply_adam=False)
        _, g64 = O.calc_gradients(st64, {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in d.items()}, cfg, None,
                                  apply_adam=False)
        if backend == 2:
            assert _plane_flags(ln) == 0, when
        mine = {k: v.detach().cpu().clone() for k, v in ln.named_grads().items()}
        _check_vs_oracle_twin(ln, out, res, g32, when)
        if backend == 0:
            for k, g in g32.items():
                assert float((mine[k] - g).abs().max()) <= 1e-4 * max(float(g.abs().max()), 1e-9), (when, k)
        _three_way(mine, g32, g64, when)
        _check_adam(ln, cfg['lr'])
        O.adam_step(st, g32, cfg)
        _sync64(st, st64)
        for k, v in ln.named_parameters().items():
            v.copy_(st.p[k].to(v.device).reshape(v.shape))
