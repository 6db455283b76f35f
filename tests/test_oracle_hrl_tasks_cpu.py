"""CPU suite: the oracle's restatement of the location / reach / strike tasks and of the four HRL tasks' target resampling
(oracle/hrl_tasks_oracle.py) against the committed outputs of the reference's own code (tests/golden/task_{heading,location,reach,strike}.pt,
written by oracle/gen_golden_hrl_tasks.py): observations, rewards, the strike termination flags, and the targets the reference's
_update_task / _reset_task / _reset_target methods wrote from their recorded draws."""
import pytest
import torch

import hrl_tasks_oracle as T
import golden_util as G

TOL = 1e-6


def _close(a, b, tol=TOL):
    assert a.shape == b.shape, (a.shape, b.shape)
    assert torch.allclose(a, b, rtol=tol, atol=tol), float((a - b).abs().max())


def test_location_obs_and_reward_match_reference_golden():
    fx = G.load('task_location.pt')
    root, tar = fx['root'], fx['tar_pos']
    _close(T.compute_location_observations(root, tar), fx['obs'])
    rew = T.compute_location_reward(root[:, 0:3], fx['prev'], root[:, 3:7], tar, fx['tar_speed'], fx['dt'])
    _close(rew, fx['reward'])
    # the edge rows: a target at the root (zero direction), pos_err exactly 0.5 (outside dist_mask), just inside it
    assert torch.equal(fx['obs'][0], torch.zeros(2)) and float(fx['reward'][0]) == pytest.approx(1.0)
    assert float(fx['reward'][2]) > float(fx['reward'][1])


def test_reach_obs_and_reward_match_reference_golden():
    fx = G.load('task_reach.pt')
    body, tar = fx['body'], fx['tar_pos']
    _close(T.compute_reach_observations(body[:, 0], tar), fx['obs'])
    _close(T.compute_reach_reward(body[:, fx['reach_body'], 0:3], tar), fx['reward'])
    assert float(fx['reward'][0]) == 1.0


def test_strike_obs_reward_and_reset_match_reference_golden():
    fx = G.load('task_strike.pt')
    rs = fx['root_states']
    _close(T.compute_strike_observations(rs[:, 0], rs[:, 1]), fx['obs'])
    _close(T.compute_strike_reward(rs[:, 1, 0:3], rs[:, 1, 3:7], rs[:, 0], fx['prev'], fx['dt']), fx['reward'])
    r = fx['reset']
    for et in (True, False):
        reset, term = T.compute_strike_reset(r['progress'], r['contact'], r['contact_body_ids'], r['pos'], r['tar_contact'], r['strike_body_ids'],
                                             r['max_episode_length'], et, r['heights'])
        assert torch.equal(reset, r[f'reset_{int(et)}']) and torch.equal(term, r[f'term_{int(et)}'])
    # progress gate: the same hit fails at progress 2 only; forces exactly at the thresholds, a z-only target force and a contact
    # through a strike body alone do not fail
    assert r['term_1'][:10].tolist() == [0, 0, 1, 0, 0, 0, 0, 0, 1, 0]
    assert int(r['term_1'].sum()) > 10 and int(r['reset_1'][11:14].sum()) == 2


@pytest.mark.parametrize('task', ['heading', 'location', 'reach', 'strike'])
def test_task_resampling_matches_reference_methods(task):
    """The oracle's per-env resampling arithmetic, fed the reference's recorded draws, gives the targets its methods wrote; rows that were
    not resampled keep their target."""
    fx = G.load(f'task_{task}.pt')
    params = fx['params']
    modes = ('reset',) if task == 'strike' else ('update', 'reset')
    assert tuple(fx['resample']) == modes
    for mode in modes:
        rec = fx['resample'][mode]
        ids = rec['env_ids']
        if mode == 'update':
            assert torch.equal(ids, (rec['progress'] >= rec['before']['change_steps']).nonzero().flatten())
        if task == 'strike':
            root = fx['root_states'][:, 0, 0:3]
        elif task == 'location':
            root = fx['root'][:, 0:3]
        else:
            root = torch.zeros(rec['progress'].shape[0], 3)
        new = T.task_resample(task, params, rec['u'], rec['steps'], root[ids], rec['progress'][ids])
        assert set(new) == set(rec['after'])
        keep = torch.ones(rec['progress'].shape[0], dtype=torch.bool); keep[ids] = False
        for k, v in new.items():
            if v.dtype == torch.int64:
                assert torch.equal(v, rec['after'][k][ids]), (mode, k)
            else:
                _close(v, rec['after'][k][ids])
            assert torch.equal(rec['after'][k][keep], rec['before'][k][keep]), (mode, k)
