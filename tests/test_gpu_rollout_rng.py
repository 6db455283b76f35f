"""GPU tests of the rollout kernels' in-kernel Philox draws against the numpy oracle (oracle/philox_oracle.py): ase_policy_sample_rng,
ase_latent_update and ase_task_resample without injected draws, the counter / seed / stream addressing, the (0, 1) uniforms of the
Bernoulli and task draws at the draws whose top 24 bits are all ones, ase_rollout_post_step against fp64, and the device rollout with its
own generator against the reference-order rollout fed the oracle's tables.

Float errors are measured in units of 2^-24 relative to a scale of the result (see each check).  The module prints its worst errors at
teardown (pytest -s).  On an H100 80GB HBM3 (400 W power limit) they were: action 4.12, normal 2.57, latent 1.90, neglogp 1.80, task 1.58,
post_step 1.22; each bound below is 3-4x its measured worst error."""
import math
import types

import numpy as np
import pytest
import torch

import hrl_tasks_oracle as T
import philox_oracle as P
from test_philox_oracle_cpu import EDGE_BERNOULLI, EDGE_OFFSET, EDGE_REACH_HEIGHT

pytestmark = pytest.mark.gpu

ULP = 2.0 ** -24
BOUND = {'normal': 8.0, 'action': 12.0, 'neglogp': 6.0, 'latent': 6.0, 'task': 6.0, 'post_step': 4.0}
_WORST = {}


@pytest.fixture(scope='module', autouse=True)
def _report_worst_errors():
    yield
    print('\nworst error vs fp64 (units of 2^-24 x scale): ' + ', '.join(f'{k} {v:.2f} (bound {BOUND[k]:g})' for k, v in sorted(_WORST.items())))


def _check(kind, got, ref, scale, what):
    """max |got - ref| / (2^-24 * scale) <= BOUND[kind]; got a tensor, ref / scale fp64 arrays."""
    got = got.detach().cpu().double().numpy()
    ref, scale = np.broadcast_arrays(np.asarray(ref, np.float64), np.asarray(scale, np.float64))
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert np.all(np.isfinite(got)), what
    e = float((np.abs(got - ref) / (ULP * scale)).max()) if got.size else 0.0
    _WORST[kind] = max(_WORST.get(kind, 0.0), e)
    assert e <= BOUND[kind], (what, kind, e, BOUND[kind])


def _rng(seed, call):
    return torch.tensor([seed, call], dtype=torch.int64, device='cuda')


def _production_probs(n):
    """AMPAgent._build_rand_action_probs: p_env = 1 - exp(10 (i / (N - 1) - 1)), p_0 = 1, p_{N-1} = 0 (fp32 on the device)."""
    ids = torch.arange(n, dtype=torch.float32, device='cuda')
    p = 1.0 - torch.exp(10 * (ids / (n - 1.0) - 1.0))
    p[0] = 1.0; p[-1] = 0.0
    return p


def _probs(kind, n, g):
    if kind == 'zero':
        return torch.zeros(n, device='cuda')
    if kind == 'one':
        return torch.ones(n, device='cuda')
    if kind == 'uniform':
        return torch.rand(n, generator=g).cuda()
    return _production_probs(n)


def _sample(mu, logstd, probs, rng, sid, noise=None, mask=None):
    from ase_b200 import ops
    n, a = mu.shape
    out = dict(actions=torch.full_like(mu, float('nan')), neglogp=torch.full((n,), float('nan'), device='cuda'),
               sigma=torch.full_like(mu, float('nan')), mask=torch.full((n,), float('nan'), device='cuda'))
    ops.policy_sample_rng(mu, logstd, probs, rng, sid, out['actions'], out['neglogp'], out['sigma'], out['mask'], noise=noise, mask=mask)
    return out


def _check_sample(out, mu, logstd, probs, seed, call, sid, what):
    """One policy_sample_rng launch against the oracle: the normals through actions, neglogp, sigma and the Bernoulli mask."""
    mu64, ls64 = mu.cpu().double().numpy(), logstd.cpu().double().numpy()
    p = None if probs is None else probs.cpu().numpy()
    act, nlp, sig, mask, z = P.policy_sample(mu64, ls64, p, seed, call, sid)
    assert np.array_equal(out['mask'].cpu().numpy(), mask), (what, 'mask', np.nonzero(out['mask'].cpu().numpy() != mask)[0][:8])
    det = torch.from_numpy(mask == 0.0).to(mu.device)
    assert torch.equal(out['actions'][det], mu[det]), (what, 'deterministic rows')
    # a = mu + sigma z: expf, the normal, one product and one sum, each a few ulps of |mu| + sigma max(|z|, 1)
    _check('action', out['actions'], act, np.abs(mu64) + sig * np.maximum(np.abs(z), 1.0), what + ' actions')
    # neglogp: the kernel's t = (a - mu) / sigma carries a's rounding, |z| * ulp(a) / sigma per term, on top of the fp32 sums
    a_round = np.abs(z) * (np.abs(mu64) + sig * np.abs(z)) / sig
    _check('neglogp', out['neglogp'], nlp, 0.5 * (z * z).sum(-1) + P.HALF_LOG_2PI * mu.shape[1] + np.abs(ls64).sum() + a_round.sum(-1),
           what + ' neglogp')
    # sigma = expf(logstd) on every row: the same bits as torch.exp on the device, within an ulp of fp64
    s = out['sigma']
    assert torch.equal(s, torch.exp(logstd).expand_as(s)), (what, 'sigma')
    assert np.allclose(s[0].cpu().double().numpy(), np.exp(ls64), rtol=2 * ULP, atol=0), (what, 'sigma vs fp64')
    return z, mask


@pytest.mark.parametrize('act_dim', [1, 3, 4, 31, 128])
@pytest.mark.parametrize('rows', [1, 31, 33, 4096, 4097])
def test_policy_sample_rng_vs_oracle(rows, act_dim):
    g = torch.Generator().manual_seed(rows * 1000 + act_dim)
    mu = torch.randn(rows, act_dim, generator=g).cuda()
    logstd = (torch.rand(act_dim, generator=g) * 3.5 - 3.0).cuda()            # sigma in [0.05, 1.65]
    seed, call = 12345, 17 + rows + act_dim
    rng = _rng(seed, call)
    for kind in ('zero', 'one', 'uniform', 'production'):
        probs = _probs(kind, rows, g)
        out = _sample(mu, logstd, probs, rng, 0)
        z, mask = _check_sample(out, mu, logstd, probs, seed, call, 0, f'rows {rows} A {act_dim} p {kind}')
        if kind in ('zero', 'one'):
            assert np.all(mask == (1.0 if kind == 'one' else 0.0)), kind
        # the oracle's draws injected give the in-kernel result to fp32 rounding
        z32, m32 = torch.from_numpy(z).float().cuda(), torch.from_numpy(mask).float().cuda()
        inj = _sample(mu, logstd, probs, rng, 0, noise=z32, mask=m32)
        assert torch.equal(inj['mask'], out['mask']) and torch.equal(inj['sigma'], out['sigma'])
        sig = torch.exp(logstd.double()).cpu().numpy()
        _check('action', inj['actions'], out['actions'].cpu().double().numpy(),
               np.abs(mu.cpu().double().numpy()) + sig * np.maximum(np.abs(z), 1.0), f'rows {rows} A {act_dim} p {kind} injected')
    assert int(rng[1]) == call                                                 # the sampling kernel does not advance the counter
    # no eps-greedy: every row samples
    out = _sample(mu, logstd, None, rng, 0)
    _check_sample(out, mu, logstd, None, seed, call, 0, f'rows {rows} A {act_dim} no probs')


@pytest.mark.parametrize('zdim', [1, 3, 4, 13, 64, 127, 128])
def test_latent_update_vs_oracle(zdim):
    from ase_b200 import ops
    n = 333
    g = torch.Generator().manual_seed(zdim)
    seed, call = {1: (12345, 0), 3: (-987654321, 5), 4: (2 ** 40 + 3, 2 ** 32 + 1), 13: (7, 123456789), 64: (12345, 40), 127: (-1, 2 ** 63 - 1),
                  128: (0, 9)}[zdim]
    lat0 = torch.randn(n, zdim, generator=g)
    kind = torch.arange(n) % 4                     # 0 done, 1 due (steps == progress), 2 due (steps < progress), 3 untouched
    prog = torch.randint(0, 1000, (n,), generator=g, dtype=torch.int64)
    steps = prog.to(torch.int32).clone()
    steps[kind == 2] -= 7
    steps[kind == 3] += 1 + torch.randint(0, 50, (int((kind == 3).sum()),), generator=g, dtype=torch.int32)
    # progress beyond int32: reset_steps (int32) compares as int64
    prog[1], steps[1] = 2 ** 31 + 5, 2 ** 31 - 200
    prog[2], steps[2] = 2 ** 32 + 9, 1000
    prog[0] = 2 ** 31 + 5
    done = (kind == 0).to(torch.uint8)
    for smin, smax, use_done in ((1, 150, True), (40, 41, True), (1, 12, False)):
        lat, st = lat0.clone().cuda(), steps.clone().cuda()
        ops.latent_update(lat, st, prog.cuda(), done.cuda() if use_done else None, smin, smax, _rng(seed, call), 2)
        want_lat, want_steps, touched = P.latent_update(lat0.double().numpy(), steps.numpy(), prog.numpy(),
                                                        done.numpy() if use_done else np.zeros(n), smin, smax, seed, call, 2)
        what = f'Z {zdim} steps [{smin}, {smax}) done mask {use_done}'
        assert np.array_equal(st.cpu().numpy().astype(np.int64), want_steps), what
        assert touched[:3].all() and not touched[3] and touched.sum() < n
        keep = torch.from_numpy(~touched)
        assert torch.equal(lat.cpu()[keep], lat0[keep]), (what, 'untouched rows')
        t = torch.from_numpy(touched)
        # unit vectors: the error is absolute, a few ulps of 1
        _check('latent', lat.cpu()[t], want_lat[touched], 1.0, what)
        assert torch.allclose(lat.cpu()[t].double().norm(dim=-1), torch.ones(int(t.sum()), dtype=torch.float64), atol=16 * ULP)


@pytest.mark.parametrize('seed,call', [(12345, 2 ** 32 + 7), (2 ** 32 + 0x1234567, 5), (-987654321, 3), (-1, 2 ** 63 - 1)])
def test_counter_seed_and_stream_addressing(seed, call):
    """mu = 0, logstd = 0 and no eps-greedy: the actions are the raw normals.  Each stream's normals and Bernoulli draws against the
    oracle; streams 0-3, the next call and the seed of the next rank differ."""
    n, a = 257, 8
    mu, logstd = torch.zeros(n, a, device='cuda'), torch.zeros(a, device='cuda')
    probs = torch.full((n,), 0.5, device='cuda')
    outs, masks = [], []
    for sid in range(4):
        what = f'seed {seed} call {call} stream {sid}'
        out = _sample(mu, logstd, None, _rng(seed, call), sid)
        z, _ = _check_sample(out, mu, logstd, None, seed, call, sid, what)
        _check('normal', out['actions'], z, np.maximum(np.abs(z), 1.0), what + ' normals')
        outs.append(out)
        outm = _sample(mu, logstd, probs, _rng(seed, call), sid)
        _check_sample(outm, mu, logstd, probs, seed, call, sid, what + ' p 0.5')
        masks.append(outm['mask'])
    for i in range(4):
        for j in range(i + 1, 4):
            assert float((outs[i]['actions'] == outs[j]['actions']).float().mean()) < 0.01, (i, j)
            assert not torch.equal(masks[i], masks[j]), (i, j)
    rank1 = _sample(mu, logstd, None, _rng((seed + 1 + 2 ** 63) % 2 ** 64 - 2 ** 63, call), 0)
    assert float((rank1['actions'] == outs[0]['actions']).float().mean()) < 0.01
    nxt = _sample(mu, logstd, None, _rng(seed,(call + 1 + 2 ** 63) % 2 ** 64 - 2 ** 63), 0)
    assert float((nxt['actions'] == outs[0]['actions']).float().mean()) < 0.01


# ---- task_resample: the Philox path for all four tasks -----------------------------------------------------------------------------------
TASK_WIDTH = {'heading': 2, 'location': 2, 'reach': 3, 'strike': 13}
# scale of the target error: the angle (2 pi) for the directions and the strike rotation, |root| + the offset for positions
TASK_SCALE = {'heading': 2 * math.pi, 'location': 10.0, 'reach': 2.0, 'strike': 10.0 * 2 * math.pi}


def _task_state(task, n, g, progress=None, change_steps=None):
    root = torch.randn(n, 13, generator=g)
    tar = torch.full((n, TASK_WIDTH[task]), 5.0)
    st = dict(root=root, tar=tar, progress=torch.zeros(n, dtype=torch.int64) if progress is None else progress,
              change_steps=None if task == 'strike' else (torch.full((n,), -1, dtype=torch.int64) if change_steps is None else change_steps))
    if task == 'heading':
        st.update(tar_speed=torch.full((n,), 5.0), tar_face_dir=torch.full((n, 2), 5.0))
    return st


def _run_resample(task, st, mask, seed, call, sid):
    from ase_b200 import ops
    d = {k: (v.clone().cuda() if v is not None else None) for k, v in st.items()}
    ops.task_resample(task, d['tar'], d['progress'], root_states=d['root'], reset_mask=None if mask is None else mask.cuda(),
                      tar_speed=d.get('tar_speed'), tar_face_dir=d.get('tar_face_dir'), change_steps=d['change_steps'], rng=_rng(seed, call),
                      stream_id=sid)
    return {k: v.cpu() for k, v in d.items() if v is not None}


def _check_resample(task, st, got, go, seed, call, sid, what):
    n = st['tar'].shape[0]
    u, steps = P.task_draws(seed, call, sid, n, T.HRL_TASK_PARAMS[task], task)
    assert np.all(u < 1.0) and np.all(u > 0.0)
    ids = torch.from_numpy(np.nonzero(go)[0])
    keep = torch.from_numpy(~go)
    want = T.task_resample(task, T.HRL_TASK_PARAMS[task], torch.from_numpy(u[go]).double(), None if steps is None else torch.from_numpy(steps[go]),
                           st['root'][ids].double(), st['progress'][ids])
    names = {'heading': {'tar_dir': 'tar', 'tar_speed': 'tar_speed', 'tar_face_dir': 'tar_face_dir', 'change_steps': 'change_steps'},
             'location': {'tar_pos': 'tar', 'change_steps': 'change_steps'}, 'reach': {'tar_pos': 'tar', 'change_steps': 'change_steps'},
             'strike': {'tar_states': 'tar'}}[task]
    assert set(want) == set(names)
    for k, mine in names.items():
        g = got[mine]
        assert torch.equal(g[keep], st[mine][keep]), (what, k, 'rows that were not resampled')
        if k == 'change_steps':
            assert torch.equal(g[ids], want[k]), (what, k)
        else:
            scale = TASK_SCALE[task] + (st['root'][ids, 0:2].abs().max(-1, keepdim=True).values.double().numpy() if task in ('location', 'strike') else 0)
            _check('task', g[ids], want[k].numpy(), scale, f'{what} {k}')


@pytest.mark.parametrize('task', ['heading', 'location', 'reach', 'strike'])
def test_task_resample_philox_vs_oracle(task):
    """Reset mode (every env flagged and a ragged subset) and update mode (the due envs) with the in-kernel draws, against the fp64
    formulas fed the oracle's uniforms: targets within fp32 rounding, change_steps exact, other rows untouched."""
    n = 4097
    g = torch.Generator().manual_seed(11)
    st = _task_state(task, n, g)
    all_envs = np.ones(n, dtype=bool)
    got = _run_resample(task, st, torch.ones(n, dtype=torch.uint8), 12345, 77, 2)
    _check_resample(task, st, got, all_envs, 12345, 77, 2, f'{task} reset all')
    sub = (torch.rand(n, generator=g) < 0.3)
    got = _run_resample(task, st, sub.to(torch.uint8), -5, 2 ** 32 + 3, 2)
    _check_resample(task, st, got, sub.numpy(), -5, 2 ** 32 + 3, 2, f'{task} reset subset')
    if task != 'strike':
        prog = torch.randint(0, 300, (n,), generator=g, dtype=torch.int64)
        st = _task_state(task, n, g, progress=prog, change_steps=torch.full((n,), 150, dtype=torch.int64))
        got = _run_resample(task, st, None, 2 ** 40 + 1, 9, 0)
        _check_resample(task, st, got, (prog >= 150).numpy(), 2 ** 40 + 1, 9, 0, f'{task} update')


# ---- the draws whose top 24 bits are all ones ---------------------------------------------------------------------------------------
def test_edge_bernoulli_with_p_one_is_always_one():
    """rng = {12345, 3636}: the Bernoulli word of row 909 is 0xffffff44, whose (0, 1] uniform is exactly 1.0; with p = 1 every row must
    sample (torch.bernoulli(1.0) is always 1), or the env acts deterministically and the sample leaves the actor loss."""
    e = EDGE_BERNOULLI
    n = e['rows']
    g = torch.Generator().manual_seed(3)
    mu, logstd = torch.randn(n, 31, generator=g).cuda(), torch.full((31,), -1.0, device='cuda')
    out = _sample(mu, logstd, torch.ones(n, device='cuda'), _rng(e['seed'], e['call']), e['sid'] - 1)
    zero_rows = torch.nonzero(out['mask'] == 0).flatten().tolist()
    assert zero_rows == [], f"mask_out is 0 at rows {zero_rows} with p = 1"


def test_edge_task_uniforms_stay_below_one():
    """Reset-mode resampling at the draws whose uniform would be 1.0: the reach height stays below height_max (env 1420, rng {12345, 1086}),
    and the location / reach offsets stay below dist_max (env 3612, rng {12345, 103}), as torch.rand's [0, 1) gives."""
    for e, task, col, limit in ((EDGE_REACH_HEIGHT, 'reach', 2, 'height_max'), (EDGE_OFFSET, 'reach', 0, 'dist_max'),
                                (EDGE_OFFSET, 'location', 0, 'dist_max')):
        n = e['rows']
        st = _task_state(task, n, torch.Generator().manual_seed(1))
        st['root'].zero_()                           # location targets are root + offset: a zero root shows the offset itself
        got = _run_resample(task, st, torch.ones(n, dtype=torch.uint8), e['seed'], e['call'], e['sid'])
        v, top = float(got['tar'][e['row'], col]), T.HRL_TASK_PARAMS[task][limit]
        assert v < top, f"{task} target column {col} of env {e['row']} is {v!r}, not below {limit} = {top}"
        assert float(got['tar'][:, col].max()) < top


# ---- rollout_post_step ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [1, 31, 32, 33, 257, 4097])
def test_rollout_post_step_vs_fp64(n):
    from ase_b200 import ops
    g = torch.Generator().manual_seed(n)
    eps = 1e-5
    vrms = types.SimpleNamespace(running_mean=torch.tensor([0.37], dtype=torch.float64, device='cuda'),
                                 running_var=torch.tensor([2.3], dtype=torch.float64, device='cuda'), eps=eps)
    v = torch.randn(n, generator=g) * 4
    edge = torch.tensor([5.0, -5.0, 5.5, -7.0, 1e4, -1e4, math.nextafter(5.0, 6.0), math.nextafter(-5.0, -6.0)])
    v[:min(n, edge.numel())] = edge[:min(n, edge.numel())]
    for pattern in ('all', 'none', 'mixed'):
        dones = {'all': torch.ones(n), 'none': torch.zeros(n), 'mixed': (torch.rand(n, generator=g) < 0.4).float()}[pattern].to(torch.uint8)
        term = (torch.rand(n, generator=g) < 0.5).to(torch.uint8)
        if pattern == 'mixed' and n > 1:
            term[0], term[1] = 1, 0
        rew = torch.randn(n, generator=g)
        cur_r0, cur_l0 = torch.randn(n, generator=g), torch.randint(0, 300, (n,), generator=g).float()
        meter0 = torch.tensor([1.5, 20.0, 3.0])
        cur_r, cur_l, meter = cur_r0.clone().cuda(), cur_l0.clone().cuda(), meter0.clone().cuda()
        nv = torch.full((n,), float('nan'), device='cuda')
        rng = _rng(99, 2 ** 32 - 1)                  # the increment carries into the high word
        for _ in range(2):
            c_r, c_l, m = cur_r.clone(), cur_l.clone(), meter.clone()
            ops.rollout_post_step(rew.cuda(), dones.cuda(), term.cuda(), v.cuda(), vrms, nv, c_r, c_l, m, rng)
        assert int(rng[0]) == 99 and int(rng[1]) == 2 ** 32 + 1, 'rng[1] advances by exactly one per launch'
        what = f'n {n} {pattern}'
        want = (math.sqrt(2.3 + eps) * v.double().clamp(-5, 5) + 0.37) * (1 - term.double())
        _check('post_step', nv, want.numpy(), math.sqrt(2.3) * 5 + 0.37, what + ' next_values')
        assert torch.all(nv.cpu()[term.bool()] == 0.0), what
        d = dones.bool()
        r_sum, l_sum = cur_r0 + rew, cur_l0 + 1.0
        assert torch.equal(c_r.cpu(), torch.where(d, torch.zeros(n), r_sum)), what
        assert torch.equal(c_l.cpu(), torch.where(d, torch.zeros(n), l_sum)), what
        want_m = meter0.double() + torch.stack([r_sum.double()[d].sum(), l_sum.double()[d].sum(), d.double().sum()])
        # lengths and counts are integers below 2^24: exact in fp32 whatever the order of the atomics; the reward sum to fp32 reordering
        assert float(m[1]) == float(want_m[1]) and float(m[2]) == float(want_m[2]), what
        assert abs(float(m[0]) - float(want_m[0])) <= 1e-5 * (float(r_sum.abs()[d].sum()) + 1.5), what
        # without a counter: the same results
        c2_r, c2_l, m2 = cur_r.clone(), cur_l.clone(), meter.clone()
        nv2 = torch.empty_like(nv)
        ops.rollout_post_step(rew.cuda(), dones.cuda(), term.cuda(), v.cuda(), vrms, nv2, c2_r, c2_l, m2, None)
        assert torch.equal(nv2, nv) and torch.equal(c2_r, c_r) and torch.equal(c2_l, c_l), what


# ---- the device rollout with its own generator ----------------------------------------------------------------------------------------
def test_device_rollout_with_its_own_generator_equals_reference_order_rollout_fed_the_oracle():
    """rollout_ase.pt and its scripted env: the device rollout drawing from a fresh {seed, 0} Philox state, with nothing injected, against the
    reference-order rollout fed the oracle's tables for the same seed and streams (step n: call n; action noise stream 0, eps-greedy mask
    stream 1, latents stream 2, latent horizons stream 3)."""
    import golden_util as G
    from test_gpu_rollout import ScriptedEnv, _agent, _close, reference_order_rollout
    fx = G.load('rollout_ase.pt')
    H, N = fx['H'], fx['N']
    env_b = ScriptedEnv(fx, masked=True)
    b = _agent(fx, env_b, device_rollout=True, rollout_graph=False)
    seed = int(b._rng[0])
    assert seed == 12345 and int(b._rng[1]) == 0
    probs = b._rand_action_probs.cpu().numpy()
    assert probs[0] == 1.0 and probs[-1] == 0.0
    tb = dict(noise=torch.from_numpy(np.stack([P.normals(seed, n, 0, N, 31) for n in range(H)])).float().cuda(),
              mask=torch.from_numpy(np.stack([P.bernoulli(seed, n, 0, probs) for n in range(H)])).float().cuda(),
              z=torch.from_numpy(np.stack([P.latents(seed, n, 2, N, 64) for n in range(H)])).float().cuda(),
              steps=torch.from_numpy(np.stack([P.randint(seed, n, 2, N, 1, 6) for n in range(H)])).to(torch.int32).cuda())
    a, env_a = reference_order_rollout(fx, tb)
    b._ase_latents.copy_(fx['latents0'].cuda()); b._latent_reset_steps.copy_(fx['steps0'].cuda().to(torch.int32))
    b.obs = {'obs': env_b.cur}
    with torch.no_grad():
        b.play_steps()
    assert int(b._rng[1]) == H
    assert not hasattr(b, '_inject')
    for k in a.experience_buffer:
        x, y = a.experience_buffer[k], b.experience_buffer[k]
        if x.dtype == torch.uint8 or k == 'rand_action_mask':
            assert torch.equal(x, y), k
        else:
            _close(x, y, 'eb.' + k, rtol=1e-5, atol=1e-6)
    m = b.experience_buffer['rand_action_mask']
    assert 0 < float(m.mean()) < 1, 'the eps-greedy schedule draws both outcomes'
    _close(a._ase_latents, b._ase_latents, 'latents', rtol=1e-5, atol=1e-6)
    assert torch.equal(a._latent_reset_steps, b._latent_reset_steps)
    assert torch.equal(env_a.task.progress_buf, env_b.task.progress_buf)
    _close(a.current_rewards, b.current_rewards, 'current_rewards', 1e-6, 1e-6)
    _close(a._episode_meter, b._episode_meter, 'episode meter', 1e-5, 1e-5)
