"""CPU tests of oracle/hrl_rollout_oracle.py, the restatement of the reference's HRL rollout (HRLAgent.env_step + play_steps +
prepare_dataset): fed the HLC draws the reference recorded, it reproduces the reference's own rollout (tests/golden/rollout_hrl.pt, written by
oracle/gen_golden_hrl_rollout.py) in fp32, and its fp64 twin stays close to both."""
import torch

import hrl_rollout_oracle as HO
import golden_util as G
import synth


def _err(a, b):
    """Worst absolute difference relative to max(1, |reference|)."""
    a, b = a.double(), b.double()
    assert a.shape == b.shape, (a.shape, b.shape)
    return float(((a - b).abs() / b.abs().clamp_min(1.0)).max())


def _run(dtype):
    fx = G.load('rollout_hrl.pt')
    return fx, HO.rollout(fx, synth.hrl_hlc_params(), synth.hrl_llc_params(), fx['hlc_sigma'], dtype)


def _compare(fx, o, tol):
    for k, ref in fx['eb'].items():
        if k == 'dones':
            assert torch.equal(o['eb'][k], ref.to(torch.uint8)), k
        else:
            assert _err(o['eb'][k], ref) <= tol, (k, _err(o['eb'][k], ref))
    assert _err(o['llc_actions'], fx['llc_actions']) <= tol, ('llc_actions', _err(o['llc_actions'], fx['llc_actions']))
    assert _err(o['returns'], fx['returns']) <= tol, ('returns', _err(o['returns'], fx['returns']))
    assert _err(o['advantages'], fx['dataset']['advantages']) <= tol * 10, 'advantages'
    v = fx['value_rms_after']
    assert _err(o['value_rms_after']['running_mean'], v['running_mean']) <= tol and _err(o['value_rms_after']['running_var'], v['running_var']) <= tol
    assert float(o['value_rms_after']['count']) == float(v['count'])


def test_fp32_oracle_reproduces_reference_hrl_rollout():
    fx, o = _run(torch.float32)
    _compare(fx, o, 1e-6)


def test_fp64_oracle_near_reference_hrl_rollout():
    fx, o = _run(torch.float64)
    _compare(fx, o, 1e-4)


def test_draw_counts_and_script_edges():
    """One HLC Normal draw per HLC step, one LLC action per sub-step; the edges the generator asserted are in the regenerated script."""
    fx = G.load('rollout_hrl.pt')
    N, H, L = fx['N'], fx['H'], fx['llc_steps']
    assert len(fx['rec']['normal']) == H and all(tuple(e.shape) == (N, 64) for e in fx['rec']['normal'])
    assert tuple(fx['llc_actions'].shape) == (H * L, N, 31)
    assert fx['hlc_sigma'] == float(torch.tensor(-2.3)) and fx['llc_disc_reward_scale'] == 2.0     # hrl_humanoid.yaml / ase_humanoid_hrl.yaml
    assert N % 16 != 0 and fx['obs_t'].shape == (H * L + 1, N, 258) and fx['amp_t'].shape == (H * L, N, 1400)
    acts = fx['eb']['actions']
    assert (acts.abs() > 1).all(-1).any()
    d = fx['dones_t'].view(H, L, N).bool()
    assert d[:, 0].any() and d[:, L // 2].any() and d[:, L - 1].any() and fx['dones_t'][-1].any()
    assert fx['term_t'].view(H, L, N)[:, :L - 1].bool().any()
