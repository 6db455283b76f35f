"""The learner at ragged network and batch shapes (the case table of tests/test_learner_shapes_cpu.py) on every GEMM backend, against the
oracle in fp32 and fp64, and the FP16-plane scale-prediction window of backend 2 pinned at its edges.

The production-width tests (tests/test_gpu_fullsize.py, tests/test_gpu_learner.py) only ever give the tensor-core backends hidden widths
that are multiples of 128.  Here the operand-plane registry meets N <= 64 tiles, the BN switch at 64/65 and 128/129, M tails, partially
used ReLU-bit words, one- and four-layer trunks, the style-column write into the statically scaled planes on both its scalar and its
16-byte path, the learner without a diversity pass, an N = 1 mu head, and eval_* calls between training calls, which share the plane
registry and the scale slots with calc_gradients.

Each case runs 4 consecutive calc_gradients calls, teacher-forced like tests/test_gpu_fullsize.py: step 0 calibrates the FP16 plane
scales, steps 1 and 2 run on scales predicted from the previous call, and the parameters are re-announced before step 3 so that a
recalibration in the middle of training is covered too."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

import ase_oracle as O
import synth
from test_gpu_fullsize import _conditioned, _three_way, _stats, _threads, _sync64
from test_gpu_learner import _cuda, _check_vs_oracle_twin
from test_learner_shapes_cpu import CASES, oracle_cfg, learner_kwargs, states, minibatch, to64

pytestmark = pytest.mark.gpu

STEPS, THREE_WAY_STEPS, RECALIBRATE_AT = 4, (0, 1, 3), 3


def _plane_flags(ln):
    """The raw sticky FP16 plane-scale status (bit 0 overflow, bit 1 underflow) without raising."""
    from ase_b200 import lib as L
    from ase_b200.ops import _stream
    f = C.c_int(0)
    L.check(L.lib.ase_learner_plane_status(ln._h, C.byref(f), _stream()), 'ase_learner_plane_status')
    return f.value


def _check_eval(ln, c, st64, seed, when):
    """eval_actor_critic on B - 37 rows and eval_disc_enc on 2 Ba + 5 rows against the oracle in fp64 (after the calc_gradients call that
    moved the normalisers, with the teacher-forced parameters)."""
    g = torch.Generator().manual_seed(seed)
    n = c['B'] - 37
    obs = torch.randn(n, c['obs'], generator=g) * 1.5 + 0.3
    z = F.normalize(torch.randn(n, c['latent'], generator=g), dim=-1) if c['kind'] == 'ase' else None
    mu, val = ln.eval_actor_critic(obs.cuda(), None if z is None else z.cuda())
    on = st64.obs_rms.norm(obs.double())
    z64 = None if z is None else z.double()
    assert torch.allclose(mu.cpu().double(), O.eval_actor(st64.p, on, z64, mu_tanh=c.get('mu_tanh', False)), rtol=1e-4, atol=1e-4), when
    assert torch.allclose(val.cpu().double(), O.eval_critic(st64.p, on, z64), rtol=1e-4, atol=1e-4), when
    if c['kind'] == 'ppo':
        return
    na = 2 * c['Ba'] + 5
    amp = torch.randn(na, c['amp'], generator=g)
    logits, enc = ln.eval_disc_enc(amp.cuda())
    an = st64.amp_rms.norm(amp.double())
    assert torch.allclose(logits.cpu().double(), O.eval_disc(st64.p, an), rtol=1e-4, atol=1e-4), when
    if c['kind'] == 'ase':
        assert torch.allclose(enc.cpu().double(), O.eval_enc(st64.p, an), rtol=1e-4, atol=1e-5), when


def _check_adam(ln, lr):
    """torch.optim.Adam on the gradients the device produced, checked in isolation (tests/test_gpu_fullsize.py (e))."""
    p0, gd = ln.params.cpu().clone(), ln.grads.cpu().clone()
    m0, v0 = ln.exp_avg.cpu().clone(), ln.exp_avg_sq.cpu().clone()
    ln.adam_step()
    t, b1, b2, eps = ln.step, 0.9, 0.999, 1e-8
    m1 = b1 * m0 + (1 - b1) * gd
    v1 = b2 * v0 + (1 - b2) * gd * gd
    p1 = p0 - (lr / (1 - b1 ** t)) * m1 / (v1.sqrt() / (1 - b2 ** t) ** 0.5 + eps)
    assert float((ln.exp_avg.cpu() - m1).abs().max()) <= 1e-6 * float(m1.abs().max())
    assert float((ln.exp_avg_sq.cpu() - v1).abs().max()) <= 1e-6 * float(v1.abs().max())
    assert float((ln.params.cpu() - p1).abs().max()) <= 1e-3 * lr + 1.2e-7 * float(p1.abs().max())


def _check_flip_bounded(ln, out, res, mine, g32, g64, when):
    """Cases marked decision_flips (production widths at B = 333): a ReLU decision within fp32 rounding of zero flips in whichever fp32
    implementation happens to have it, and at this B the one sample it belongs to moves every weight gradient upstream by up to 1e-2 of
    its max, on up to a third of the elements.  Measured with seed 31: the fp32 oracle flips a decision of the third critic layer at
    step 3 (fp64 margin 3.5e-9 of the sum of |terms|), the SIMT backend one at step 1 (margin 2.2e-8); critic_mlp._mlp.0.weight then
    has 36 % / 18 % of its elements beyond 1e-4, worst 1.0e-2 / 3.5e-3, and the median of critic_mlp._mlp.0.bias moves by 8.8e-5 /
    6.9e-5 (the backend that did not flip is 4e-8 from fp64).  So this case is held to the production-width bounds of
    tests/test_gpu_fullsize.py, which a single flip respects, against both the fp32 oracle and fp64: median within 3e-5 of the tensor max
    for the discriminator, encoder and value-head tensors (1e-3 for the others), every element within 5e-2; scalars and logits at 1e-4
    as everywhere.  -> (worst ref32-vs-fp64, worst ours-vs-fp64)"""
    tr = ln.train_result(out)
    for k in tr:
        if k in res:
            v = float(res[k])
            assert abs(tr[k] - v) <= 1e-4 * max(1.0, abs(v)), (when, k, tr[k], v)
    assert torch.allclose(out['disc_agent_logit'].cpu(), res['disc_agent_logit'].flatten(), rtol=1e-4, atol=1e-4), when
    assert torch.allclose(out['disc_demo_logit'].cpu(), res['disc_demo_logit'].flatten(), rtol=1e-4, atol=1e-4), when
    worst_ref, worst_me = 0.0, 0.0
    for k in g32:
        x, m, r = _stats(mine[k], g32[k]), _stats(mine[k], g64[k]), _stats(g32[k], g64[k])
        worst_ref, worst_me = max(worst_ref, r[3]), max(worst_me, m[3])
        tol = 3e-5 if _conditioned(k) else 1e-3
        assert x[0] <= tol and m[0] <= tol and x[3] <= 5e-2 and m[3] <= 5e-2, (when, k, 'vs fp32', x, 'vs fp64', m)
    return worst_ref, worst_me


def _sweep(name, backend):
    _threads()
    from ase_b200 import Learner, lib as L
    c = CASES[name]
    cfg = oracle_cfg(c)
    P, st, st64 = states(c, seed=31)
    ln = Learner(**learner_kwargs(c, cfg), gemm_backend=backend)
    ln.load_named(P)
    if backend:
        L.lib.ase_gemm_tc_profile(1)
    summary = []
    try:
        for s in range(STEPS):
            when = f'{name} backend {backend} step {s}'
            if s == RECALIBRATE_AT:
                ln.params_changed()
            d, new_z = minibatch(c, st, cfg, seed=3100 + s)
            out = ln.calc_gradients(_cuda(d), None if new_z is None else new_z.cuda())
            res, g32 = O.calc_gradients(st, d, cfg, new_z, apply_adam=False)
            _, g64 = O.calc_gradients(st64, to64(d), cfg, None if new_z is None else new_z.double(), apply_adam=False)
            if backend == 2:                                        # (train_result raises on a flag as well)
                assert _plane_flags(ln) == 0, when
            mine = {k: v.detach().cpu().clone() for k, v in ln.named_grads().items()}
            if c.get('decision_flips'):
                summary.append((s,) + _check_flip_bounded(ln, out, res, mine, g32, g64, when))
            else:
                _check_vs_oracle_twin(ln, out, res, g32, when)      # scalars and logits at 1e-4; the bulk of every gradient tensor
                if backend == 0:                                    # exact fp32: every element
                    for k, g in g32.items():
                        assert float((mine[k] - g).abs().max()) <= 1e-4 * max(float(g.abs().max()), 1e-9), (when, k)
                if s in THREE_WAY_STEPS:
                    _, wr, wm = _three_way(mine, g32, g64, when)
                    summary.append((s, wr, wm))
            _check_adam(ln, cfg['lr'])
            # teacher forcing without params_changed: the plane scales stay predicted
            O.adam_step(st, g32, cfg)
            _sync64(st, st64)
            for k, v in ln.named_parameters().items():
                v.copy_(st.p[k].to(v.device).reshape(v.shape))
            assert torch.allclose(ln.running_mean_std.running_mean.cpu(), st.obs_rms.mean, rtol=1e-6, atol=1e-7), when
            if c['kind'] != 'ppo':
                assert torch.allclose(ln.amp_input_mean_std.running_var.cpu(), st.amp_rms.var, rtol=1e-5, atol=1e-9), when
            _check_eval(ln, c, st64, 3200 + s, when)
            if backend == 2:
                assert _plane_flags(ln) == 0, when + ' (eval)'
        if backend:
            n = C.c_int64()
            L.check(L.lib.ase_gemm_tc_profile_read(None, C.byref(n), None), 'profile_read')
            assert n.value >= 10 * STEPS, f"{name}: the tensor-core kernel was launched only {n.value} times: the learner fell back to SIMT"
    finally:
        if backend:
            L.lib.ase_gemm_tc_profile(0)
    return summary


@pytest.mark.parametrize('backend', [0, 1, 2])
@pytest.mark.parametrize('name', list(CASES))
def test_learner_shape_sweep(name, backend):
    print(f'{name} backend {backend} (step, worst ref32-vs-fp64, worst ours-vs-fp64):', _sweep(name, backend))


# ------------------------------------------------------------------------------------------------ FP16 plane-scale window
ACTOR = ('actor_mlp.', 'mu.')


def test_fp16_plane_scale_window_edges():
    """Backend 2 predicts each tensor's power-of-two scale from the previous call's max, so that max lands in [2^8, 2^9).  A value beyond
    60000 after scaling is an overflow (flagged by the epilogue in the same call): growth by x 64 always fits, x 512 never does.  A max
    below 2^-6 after scaling is an underflow (flagged at the start of the next call): shrinking by 2^-13 always fits, 2^-16 never does.

    Plain PPO with bounds_loss_coef = 0: d mu is then exactly linear in the advantages (the PPO clip decisions only depend on their sign),
    so scaling them by a power of two f scales every actor backward tensor by f and leaves the forward and the value branch alone.
    Each leg starts from a fresh calibration, since coming back from a shrink is itself a growth."""
    _threads()
    from ase_b200 import Learner, lib as L
    B, obs, act, units = 200, 258, 31, (160, 72)
    cfg = dict(O.DEFAULT_CFG); cfg['bounds_loss_coef'] = 0.0
    P = synth.params(O.amp_param_shapes(obs=obs, act=act, amp=0, units=units), seed=6)
    st = O.LearnerState(P, obs, 0, 'ppo')
    st64 = O.LearnerState({k: v.double() for k, v in P.items()}, obs, 0, 'ppo')
    d, _ = synth.minibatch(st, cfg, B, 0, seed=60, kind='ppo', obs_dim=obs, act=act)
    st.obs_rms.update(d['obs'])                          # the statistics the old policy of the minibatch was evaluated with ...
    st64.obs_rms = st.obs_rms.clone()
    for s in (st, st64):                                 # ... used unchanged by every call (update_rms=False on the device)
        s.obs_rms.train_forward = s.obs_rms.norm
    _, g32 = O.calc_gradients(st, d, cfg, None, apply_adam=False)
    _, g64 = O.calc_gradients(st64, to64(d), cfg, None, apply_adam=False)
    ln = Learner('ppo', obs, act, B, units=units, hparams={'learning_rate': cfg['lr'], 'bounds_loss_coef': 0.0}, gemm_backend=2)
    ln.load_named(P)
    ln.running_mean_std.load_state_dict({'running_mean': st.obs_rms.mean.cuda(), 'running_var': st.obs_rms.var.cuda(),
                                         'count': st.obs_rms.count.cuda()})
    dc = _cuda(d)

    def call(f):
        x = dict(dc); x['advantages'] = dc['advantages'] * f
        return ln.calc_gradients(x, update_rms=False)

    def check(f, when):
        scaled = lambda g: {k: (v * f if k.startswith(ACTOR) else v) for k, v in g.items()}
        mine = {k: v.detach().cpu().clone() for k, v in ln.named_grads().items()}
        _, wr, wm = _three_way(mine, scaled(g32), scaled(g64), when)
        return wr, wm

    def fresh():
        ln.params_changed()
        ln.train_result(call(1.0))
        check(1.0, 'calibration')

    worst = {}
    for f in (64.0, 2.0 ** -13):                         # inside the window: no flag, now or at the next call; fp32 accuracy
        fresh()
        ln.train_result(call(f))
        worst[f] = check(f, f'f = {f}')
        ln.train_result(call(f))
        assert _plane_flags(ln) == 0, f
    fresh()
    with pytest.raises(L.AseError):                      # growth beyond the window: reported by the very call
        ln.train_result(call(512.0))
    assert _plane_flags(ln) & 1
    ln.plane_flag_clear()
    fresh()
    ln.train_result(call(2.0 ** -16))                    # shrink beyond the window: the call itself is not flagged yet ...
    with pytest.raises(L.AseError):                      # ... the next call's train_result reports it
        ln.train_result(call(2.0 ** -16))
    assert _plane_flags(ln) == 2
    ln.plane_flag_clear()
    fresh()
    assert _plane_flags(ln) == 0
    print('plane-scale window (f: worst ref32-vs-fp64, worst ours-vs-fp64):', worst)


def test_fp16_plane_scale_miss_of_split_writers():
    """The two writers of FP16 planes that are not GEMM epilogues report a scale miss themselves, and each case below can only be
    flagged by that writer: a GEMM epilogue downstream would flag the same growth and hide a broken report.

    Latent columns (copy_cols) are written into planes with the static scale 64.  Right after params_changed every scale site
    calibrates exactly, so only static-scale writers can flag: a latent entry of 1000 (64000 after scaling) must set bit 0, one of
    900 (57600) must not.

    Weights are re-split in one batched launch with the scale predicted from their last exact split: adam_step marks the weight planes
    stale but keeps their sites known.  mu.weight grown x 512 without params_changed must set bit 0 in the next eval_actor_critic, x 64
    must not.  The mu output has no planes, so with want_value=False no epilogue can flag in its place."""
    _threads()
    from ase_b200 import Learner
    c = CASES['ase_ragged']
    cfg = oracle_cfg(c)
    P, st, _ = states(c, seed=5)
    d, new_z = minibatch(c, st, cfg, seed=50)
    dc, nz = _cuda(d), new_z.cuda()
    ln = Learner(**learner_kwargs(c, cfg), gemm_backend=2)
    n = c['B'] - 37
    obs, z = dc['obs'][:n], dc['ase_latents'][:n]

    for v, flagged in ((900.0, False), (1000.0, True)):
        ln.load_named(P)                                 # params_changed: every scale site calibrates exactly on the next call
        x = dict(dc); x['ase_latents'] = dc['ase_latents'].clone()
        x['ase_latents'][7, 5] = v
        ln.calc_gradients(x, nz, update_rms=False)
        assert _plane_flags(ln) == (1 if flagged else 0), v
        ln.plane_flag_clear()

    for f, flagged in ((64.0, False), (512.0, True)):
        ln.load_named(P)
        ln.train_result(ln.calc_gradients(dc, nz, update_rms=False))     # calibration (train_result raises on a flag)
        ln.eval_actor_critic(obs, z, want_value=False)
        assert _plane_flags(ln) == 0, f
        ln.adam_step()
        ln.named_parameters()['mu.weight'].mul_(f)
        ln.eval_actor_critic(obs, z, want_value=False)
        assert _plane_flags(ln) == (1 if flagged else 0), f
        ln.plane_flag_clear()
