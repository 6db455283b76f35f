"""Learner configurations at ragged network and batch shapes, each chosen for a branch of the tensor-core learner it reaches
(tests/test_gpu_learner_shapes.py runs them on every GEMM backend), and a CPU guard for that table: the oracle builds every shape in
fp32 and fp64, and its own fp32-vs-fp64 spread sits well inside the bounds the GPU test applies.  Needs neither a GPU nor the
compiled library."""
import pytest
import torch

import ase_oracle as O
import synth

# kind, obs / latent / act / amp dims, trunk widths, batch rows B and AMP rows Ba; `diversity` False gives Ra = B (no second actor pass)
CASES = {
    # BN = 64 tiles; M tails (Ra = 2B = 400, 3Ba = 150); latent and AMP planes with padded ldp; partially used ReLU-bit words
    'ase_ragged': dict(kind='ase', obs=253, latent=24, act=31, amp=350, units=(72, 40, 24), style=(40, 24), disc=(48, 40, 24),
                       B=200, Ba=50, diversity=True),
    # obs % 8 == 0: the style columns land 16-byte aligned in the static planes of Xa; widths at the 64/65 and 128/129 tile edges;
    # exactly one M tile
    'ase_aligned_style': dict(kind='ase', obs=256, latent=32, act=28, amp=352, units=(128, 129, 65), style=(64,), disc=(129, 64),
                              B=128, Ba=43, diversity=False),
    # ASE_MAX_LAYERS in every trunk: the deepest gradient-penalty chain, the most scale sites per call
    'ase_max_depth': dict(kind='ase', obs=253, latent=64, act=31, amp=1400, units=(96, 80, 64, 48), style=(96, 80, 64, 48),
                          disc=(96, 80, 64, 48), B=256, Ba=64, diversity=True),
    # one-layer trunks (the d w_logit column sum fused into the first masked GEMM); B below one 128-row tile; Ba == B
    'amp_one_layer': dict(kind='amp', obs=253, act=31, amp=1400, units=(130,), disc=(200,), B=96, Ba=96),
    # N = 1 mu head, K = 1 for its dX, tanh mu, B = 128 + 1
    'ppo_tanh_narrow': dict(kind='ppo', obs=258, act=1, units=(33, 17), B=129, mu_tanh=True),
    # production widths with a ragged M in every GEMM.  decision_flips: with ~10^6 ReLU decisions per step some lie within fp32 rounding
    # of zero, and at this B one flipped sample visibly moves the weight gradients upstream of it (tests/test_gpu_learner_shapes.py)
    'ase_production_ragged_batch': dict(kind='ase', obs=253, latent=64, act=31, amp=1400, units=(1024, 1024, 512), style=(512, 256),
                                        disc=(1024, 1024, 512), B=333, Ba=111, diversity=True, decision_flips=True),
}

HP_KEYS = ('e_clip', 'critic_coef', 'entropy_coef', 'bounds_loss_coef', 'disc_coef', 'disc_logit_reg', 'disc_grad_penalty',
           'disc_weight_decay', 'enc_coef', 'amp_diversity_bonus', 'amp_diversity_tar')


def param_shapes(c):
    if c['kind'] == 'ase':
        return O.ase_param_shapes(obs=c['obs'], z=c['latent'], act=c['act'], amp=c['amp'], units=c['units'], disc_units=c['disc'],
                                  style_units=c['style'])
    return O.amp_param_shapes(obs=c['obs'], act=c['act'], amp=c.get('amp', 0), units=c['units'], disc_units=c.get('disc', ()))


def oracle_cfg(c):
    cfg = dict(O.DEFAULT_CFG)
    cfg['amp_minibatch_size'] = c.get('Ba', 0)
    if c['kind'] != 'ase':
        cfg['enc_coef'] = 0.0
    if not c.get('diversity', False):
        cfg['amp_diversity_bonus'] = 0.0
    if c.get('mu_tanh'):
        cfg['mu_tanh'] = True
    return cfg


def learner_kwargs(c, cfg):
    """Keyword arguments of ase_b200.Learner for case c (besides gemm_backend)."""
    hp = {k: cfg[k] for k in HP_KEYS}
    hp['learning_rate'] = cfg['lr']
    kw = dict(kind=c['kind'], obs_dim=c['obs'], act_dim=c['act'], batch=c['B'], units=c['units'], hparams=hp,
              mu_activation='tanh' if c.get('mu_tanh') else 'None')
    if c['kind'] != 'ppo':
        kw.update(amp_dim=c['amp'], amp_batch=c['Ba'], disc_units=c['disc'])
    if c['kind'] == 'ase':
        kw.update(latent_dim=c['latent'], style_units=c['style'])
    return kw


def states(c, seed):
    """Seeded parameters, the fp32 oracle state and its fp64 twin."""
    P = synth.params(param_shapes(c), seed=seed)
    amp = c.get('amp', 0) if c['kind'] != 'ppo' else 0
    st = O.LearnerState(P, c['obs'], amp, c['kind'])
    st64 = O.LearnerState({k: v.double() for k, v in P.items()}, c['obs'], amp, c['kind'])
    return P, st, st64


def minibatch(c, st, cfg, seed):
    """(minibatch dict, the diversity pass's new latents or None)"""
    d, new_z = synth.minibatch(st, cfg, c['B'], c.get('Ba', 0), seed=seed, kind=c['kind'], obs_dim=c['obs'], amp_dim=c.get('amp', 0),
                               act=c['act'], zdim=c.get('latent', 64))
    return d, (new_z if c.get('diversity', False) else None)


def to64(d):
    return {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in d.items()}


def rel_err(a, b):
    """element-wise |a - b| / max|b| as float64"""
    return (a.double() - b.double()).abs().flatten() / max(float(b.double().abs().max()), 1e-30)


@pytest.mark.parametrize('name', list(CASES))
def test_oracle_builds_case_and_its_fp32_spread_is_small(name):
    """One oracle step per case in fp32 and fp64.  The GPU sweep holds a tensor-core gradient to a median within 2e-5 of the tensor max
    of the fp32 oracle, to no element beyond 1e-4 of it in 95 % of the tensor, and to 1e-4 of fp64 where the fp32 oracle is closer than
    that: the fp32 oracle must itself sit well inside those bounds at every shape, or they say nothing.  Measured (seed 3): median
    <= 5.1e-6, worst element <= 1.4e-5 of the tensor max, loss scalars <= 1.3e-6."""
    torch.manual_seed(0)
    c = CASES[name]
    cfg = oracle_cfg(c)
    P, st, st64 = states(c, seed=3)
    d, new_z = minibatch(c, st, cfg, seed=300)
    res, g32 = O.calc_gradients(st, d, cfg, new_z, apply_adam=False)
    res64, g64 = O.calc_gradients(st64, to64(d), cfg, None if new_z is None else new_z.double(), apply_adam=False)
    assert set(g32) == set(P) - {'sigma'}
    for k, g in g32.items():
        assert g.shape == P[k].shape and g.dtype == torch.float32 and g64[k].dtype == torch.float64, k
        assert torch.isfinite(g).all() and float(g.abs().max()) > 0, k
    if c['kind'] == 'ase' and not c.get('diversity', False):
        assert 'amp_diversity_loss' not in res
    worst = 0.0
    for k in g32:
        e = rel_err(g32[k], g64[k])
        worst = max(worst, float(e.max()))
        assert float(e.median()) <= 1e-5, (name, k, float(e.median()))
    assert worst <= 5e-5, (name, worst)
    for k in ('actor_loss', 'critic_loss', 'kl', 'disc_loss', 'disc_grad_penalty', 'enc_loss', 'amp_diversity_loss'):
        if k in res:
            assert abs(float(res[k]) - float(res64[k])) <= 1e-5 * max(1.0, abs(float(res64[k]))), (name, k)
    print(f'{name}: worst fp32-vs-fp64 gradient element {worst:.2e} of its tensor max')

