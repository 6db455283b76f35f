"""CPU tests of oracle/getup_oracle.py, the restatement of the device episode resets (ase_amp_state_init, ase_amp_history_init,
ase_recovery_step): fed the draws the reference recorded, it reproduces the reference's own resets (tests/golden/getup_reset.pt, written by
oracle/gen_golden_getup.py); fed the kernels' Philox draws, clip ids and init kinds follow the configured probabilities."""
import numpy as np
import pytest
import torch
from scipy import stats

import ase_oracle as O
import getup_oracle as GO
import golden_util as G

D, S = 31, 10


def _tables(fx):
    return O.synthetic_motion_tables(seed=fx['motion_seed'])


def _state(x, getup):
    dof = x['dof'].view(-1, D, 2)
    return dict(root=x['root'][:, 0].clone(), dof_pos=dof[..., 0].clone(), dof_vel=dof[..., 1].clone(),
                counter=x['counter'].clone() if getup else None, progress=x['progress'].clone(), reset=x['reset'].to(torch.uint8),
                terminate=x['terminate'].to(torch.uint8),          # read only by the getup case (its recovery draws are 0 otherwise)
                init_root=x['init_root'], init_dof_pos=x['init_dof_pos'], init_dof_vel=x['init_dof_vel'],
                fall_root=x['fall_root'], fall_dof_pos=x['fall_dof_pos'], fall_dof_vel=x['fall_dof_vel'])


def reset_with_oracle(fx, name):
    """The three steps of a reset in the oracle: state init, slot 0 + obs of the flagged envs, history init -> (state, obs, AMP buffer)."""
    x, rec = fx['inputs'], fx['modes'][name]
    mt = _tables(fx)
    p = dict(state_init=rec['state_init'], hybrid_prob=0.5, recovery_prob=0.2 if rec['getup'] else 0.0, fall_prob=0.1 if rec['getup'] else 0.0,
             recovery_steps=60)
    st = _state(x, rec['getup'])
    out = GO.state_init(mt, st, rec['mask'], rec['draws'], p)
    m = rec['mask'].bool()
    n = m.shape[0]
    body = x['body']
    obs = GO.obs_before(n)
    obs[m] = O.compute_humanoid_observations_max(body[m, :, 0:3], body[m, :, 3:7], body[m, :, 7:10], body[m, :, 10:13], True, True)
    amp = GO.amp_before(n, S)
    kb = body[m][:, O.KEY_BODY_IDS_SWORD_SHIELD, 0:3]
    amp[m, 0] = O.build_amp_observations(body[m, 0, 0:3], body[m, 0, 3:7], body[m, 0, 7:10], body[m, 0, 10:13], out['dof_pos'][m],
                                         out['dof_vel'][m], kb, True, True, O.DOF_OFFSETS_SWORD_SHIELD)
    amp = GO.history_init(mt, amp, out['kind'], out['motion_id'], out['motion_time'], fx['dt'])
    return out, obs, amp


@pytest.mark.parametrize('name', ['default', 'start', 'random', 'hybrid', 'hybrid_getup'])
def test_oracle_reproduces_reference_resets(name):
    fx = G.load('getup_reset.pt')
    rec, want = fx['modes'][name], fx['modes'][name]['after']
    out, obs, amp = reset_with_oracle(fx, name)
    assert torch.equal(out['kind'], rec['kind'])
    for k in ('progress', 'reset', 'terminate') + (('counter',) if rec['getup'] else ()):
        assert torch.equal(out[k].to(want[k].dtype), want[k]), (name, k)
    want_obs, want_amp = GO.fixture_buffers(fx, name)
    for k, got, w in (('root', out['root'], want['root']), ('dof_pos', out['dof_pos'], want['dof_pos']), ('dof_vel', out['dof_vel'], want['dof_vel']),
                      ('obs', obs, want_obs), ('amp', amp, want_amp)):
        assert torch.allclose(got, w, rtol=1e-6, atol=1e-6), (name, k, float((got - w).abs().max()))
    if name == 'hybrid_getup':
        rv = rec['kind'] == GO.RECOVERY
        assert int(rv.sum()) > 0 and torch.equal(out['root'][rv], fx['inputs']['root'][rv, 0])     # a recovery episode keeps its state


def test_oracle_recovery_sequence():
    q = G.load('getup_reset.pt')['recovery_seq']
    for i in range(q['counter'].shape[0]):
        c, r, t = GO.recovery_step(q['counter_in'][i], q['base_reset'][i], q['base_terminate'][i])
        assert torch.equal(c, q['counter'][i]) and torch.equal(r, q['reset'][i]) and torch.equal(t, q['terminate'][i])


def test_philox_clip_ids_follow_the_weights():
    w = np.array([4.0, 1.0, 2.0, 3.0, 0.0, 7.5])
    cdf = GO.motion_cdf(w)
    assert float(cdf[-1]) == 1.0
    n = 1 << 20
    d = GO.philox_draws(987654321, 3, 0, n, cdf, 64, dict(recovery_prob=0.2, fall_prob=0.1, hybrid_prob=0.5))
    counts = np.bincount(d['motion_id'].numpy(), minlength=len(w))
    assert counts[4] == 0                                                   # a zero-weight clip is never drawn
    keep = w > 0
    chi2, pval = stats.chisquare(counts[keep], n * w[keep] / w.sum())
    assert pval > 1e-3, (chi2, pval, counts)
    rows = np.bincount(d['fall_row'].numpy(), minlength=64)
    assert stats.chisquare(rows).pvalue > 1e-3 and rows.size == 64


def test_philox_init_kind_frequencies():
    n = 1 << 20
    p = dict(recovery_prob=0.2, fall_prob=0.1, hybrid_prob=0.5)
    d = GO.philox_draws(2 ** 40 + 5, 2 ** 33 + 1, 2, n, GO.motion_cdf([1.0, 1.0]), 16, p)
    rng = np.random.default_rng(0)
    term = torch.from_numpy((rng.random(n) < 0.4).astype(np.uint8))
    mask = torch.ones(n, dtype=torch.uint8)
    kind = GO.init_kinds(mask, term, d, 'Hybrid').numpy()
    t = term.numpy().astype(bool)
    assert not np.any((kind == GO.RECOVERY) & ~t)                           # recovery only on terminated envs
    freq = lambda k, sel=slice(None): float(np.mean(kind[sel] == k))
    se = lambda q, m: 4.0 * np.sqrt(q * (1 - q) / m)
    nt = int(t.sum())
    assert abs(freq(GO.RECOVERY, t) - 0.2) < se(0.2, nt)
    q_fall = 0.1
    assert abs(freq(GO.FALL, ~t) - q_fall) < se(q_fall, n - nt)
    assert abs(freq(GO.REF, ~t) - 0.9 * 0.5) < se(0.45, n - nt)
    assert abs(freq(GO.DEFAULT, ~t) - 0.9 * 0.5) < se(0.45, n - nt)
    assert abs(freq(GO.FALL, t) - 0.8 * 0.1) < se(0.08, nt)
    one = GO.philox_draws(1, 0, 0, 4096, GO.motion_cdf([1.0]), 1, dict(recovery_prob=1.0, fall_prob=1.0, hybrid_prob=1.0))
    assert bool(one['recovery'].all() and one['fall'].all() and one['hybrid'].all())      # p = 1 always fires
