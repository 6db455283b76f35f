"""CPU test of oracle/player_oracle.py, the fp64 restatement of the players' run loop, against tests/golden/player_{amp,ase,hrl}.pt: what
the reference's own AMPPlayerContinuous, ASEPlayer and HRLPlayer did (oracle/gen_golden_players.py).  Fed the recorded draws and the same
numpy seed, the restatement reproduces every printed line, the numpy latent countdown and every env action."""
import pytest
import torch

import golden_util as G
import player_oracle as PO


def _runs():
    return [(kind, i) for kind, cnt in (('amp', 2), ('ase', 3), ('hrl', 2)) for i in range(cnt)]


def lines_equal(mine, ref):
    """run()'s printed lines: words equal, numbers within 1e-6 relative (the reference sums in fp32)."""
    assert len(mine) == len(ref), (mine, ref)
    for a, b in zip(mine, ref):
        ta, tb = a.split(), b.split()
        assert len(ta) == len(tb), (a, b)
        for x, y in zip(ta, tb):
            if x.endswith(':') or y.endswith(':') or x.isalpha():
                assert x == y, (a, b)
            else:
                assert abs(float(x) - float(y)) <= 1e-6 * max(1.0, abs(float(y))), (a, b)


def format_lines(lines):
    return [' '.join(str(t) for t in ln) for ln in lines]


@pytest.mark.parametrize('kind,i', _runs())
def test_oracle_reproduces_the_reference_players(kind, i):
    fx = G.load(f'player_{kind}.pt')[i]
    res, env = PO.run_fixture(fx)
    lines_equal(format_lines(res['lines']), fx['lines'])
    assert res['countdown'] == fx['rec']['countdown']
    acts = torch.stack(env.actions)
    assert acts.shape == fx['actions'].shape
    ref = fx['actions'].double()
    assert float((acts - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max())), kind


def test_fixtures_hold_their_edge_cases():
    """Head outputs clamped onto a non-unit box, a step that pushes games_played past games_num, a segment restart at max_steps, a
    single-env run, stochastic and deterministic runs."""
    seen_det = set()
    for kind, i in _runs():
        fx = G.load(f'player_{kind}.pt')[i]
        res, _ = PO.run_fixture(fx)
        seen_det.add(fx['determenistic'])
        if fx['N'] > 1:
            assert res['games_played'] >= fx['games_num']
    assert seen_det == {True, False}
    amp = PO.run_fixture(G.load('player_amp.pt')[0])[0]
    assert amp['games_played'] > G.load('player_amp.pt')[0]['games_num']
    assert G.load('player_ase.pt')[2]['N'] == 1
