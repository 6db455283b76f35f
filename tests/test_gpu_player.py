"""GPU tests of the evaluation players (ase_b200/player.py over csrc/player_kernels.cu):

  * AMPPlayer, ASEPlayer and HRLPlayer against what the reference's own AMPPlayerContinuous, ASEPlayer and HRLPlayer did
    (tests/golden/player_*.pt, oracle/gen_golden_players.py), fed the recorded draws and numpy seed: every printed line, the numpy latent
    countdown and every env action (HRL: every LLC sub-step), on the three GEMM backends.  The fixtures hold stochastic and deterministic runs,
    head outputs beyond +-1 on a non-unit action box, a step that pushes games_played past games_num, segments restarted at max_steps, a
    global latent resample on a step with resets, and a single-env run;
  * the action head bit for bit against the reference's fp32 op sequence;
  * an HRL player over an LLC checkpoint in the shipped ase_llc layout;
  * the in-kernel Philox path run twice from the same seed gives the same run, and no synchronising torch call happens inside a window;
  * restore() of a checkpoint this package's ASEAgent.save() wrote, and construction through an rl_games player factory with the env created
    through rl_games.common.env_configurations."""
import contextlib
import io

import numpy as np
import pytest
import torch

import golden_util as G
import player_oracle as PO
from test_oracle_player_cpu import lines_equal

pytestmark = pytest.mark.gpu

N, D, AMP, A, Z, TASK, UNITS, LOW, HIGH = 24, PO.D, PO.AMP, PO.A, PO.Z, PO.TASK, PO.UNITS, PO.LOW, PO.HIGH


class _Box:
    def __init__(self, low, high):
        self.low, self.high = np.asarray(low, dtype=np.float32), np.asarray(high, dtype=np.float32)
        self.shape = self.low.shape


class _Task:
    def __init__(self, n):
        self.num_envs, self.viewer = n, None

    def get_task_obs_size(self):
        return TASK


class GpuScriptEnv(PO.ScriptEnv):
    """oracle/player_oracle.ScriptEnv (the script of the fixtures) on the GPU, with the vec-env surface the players use and the mask-driven
    reset."""

    def __init__(self, tables, n, obs_dim=D, amp_dim=AMP, act_low=LOW, act_high=HIGH):
        super().__init__(tables, device='cuda')
        self.task = _Task(n)
        self.env = self
        self.observation_space = _Box(-np.inf * np.ones(obs_dim), np.inf * np.ones(obs_dim))
        self.amp_observation_space = _Box(-np.inf * np.ones(amp_dim), np.inf * np.ones(amp_dim))
        self.action_space = _Box(act_low, act_high)

    def get_env_info(self):
        return {'action_space': self.action_space, 'observation_space': self.observation_space, 'amp_observation_space': self.amp_observation_space}

    def reset_done(self, mask):
        self.cur = torch.where(mask.bool().unsqueeze(1), self.reset_obs_t[self.t % self.T], self.cur)
        return self.cur


class _Recorded:
    """The fixture's draws in call order on the device.  Steps a window runs after the run stopped take further draws; they change no
    statistic, so any table serves them."""

    def __init__(self, tabs):
        self.tabs = [t.float().cuda() for t in tabs] or [None]

    def __getitem__(self, k):
        return self.tabs[min(k, len(self.tabs) - 1)]


def _net(units):
    return {'space': {'continuous': {'sigma_init': {'name': 'const_initializer', 'val': -1.0}}}, 'mlp': {'units': list(units)},
            'disc': {'units': list(units)}}


def _player_config(kind, env, backend, det, games, max_steps, tmp_path):
    from ase_b200 import configs
    cfg = configs.make(kind, vec_env=env, device='cuda:0', gemm_backend=backend, net_params=_net(UNITS), seed=3,
                       player={'games_num': games, 'determenistic': det, 'max_steps': max_steps})
    if kind == 'ase':
        cfg.update(latent_steps_min=1, latent_steps_max=4)
    if kind == 'hrl':
        torch.save(PO.checkpoint(PO.params('llc', 31), PO.rms(D - TASK, 32), PO.rms(AMP, 33)), tmp_path / 'llc.pth')
        cfg.update(llc_net_params=_net(UNITS), latent_dim=Z, llc_steps=3, llc_checkpoint=str(tmp_path / 'llc.pth'))
    return cfg


def _make_player(kind, env, backend, det, games, max_steps, tmp_path):
    from ase_b200 import player as PL
    cls = {'amp': PL.AMPPlayer, 'ase': PL.ASEPlayer, 'hrl': PL.HRLPlayer}[kind]
    pl = cls(_player_config(kind, env, backend, det, games, max_steps, tmp_path))
    fn = tmp_path / f'{kind}.pth'
    torch.save(PO.checkpoint(PO.params(kind, 11), PO.rms(D, 12), None if kind == 'hrl' else PO.rms(AMP, 13)), fn)
    pl.restore(str(fn))
    return pl


def _run_captured(pl):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        res = pl.run()
    return res, buf.getvalue().strip().splitlines()


def _runs():
    return [(kind, i) for kind, cnt in (('amp', 2), ('ase', 3), ('hrl', 2)) for i in range(cnt)]


@pytest.mark.parametrize('backend', [0, 1, 2])
@pytest.mark.parametrize('kind,i', _runs())
def test_player_reproduces_the_reference_player(kind, i, backend, tmp_path):
    """Fed the reference's recorded draws and numpy seed: its printed lines (counts exact, sums within 1e-6), its numpy latent countdown and
    every env action.  The actions pass through the network, whose GEMMs sum in another order than the CPU fp32 reference on every backend:
    1e-4 relative to the largest action (the bit-exact part, the action head, is checked on its own below)."""
    fx = G.load(f'player_{kind}.pt')[i]
    n = fx['N']
    env = GpuScriptEnv(PO.tables(n, fx['table_seed']), n)
    pl = _make_player(kind, env, backend, fx['determenistic'], fx['games_num'], fx['max_steps'], tmp_path)
    pl._inject = {'noise': _Recorded(fx['rec']['normal']), 'z': _Recorded(PO.latent_tables(fx['rec'], n))}
    countdown = []
    if kind == 'ase':
        real = pl._reset_latent_step_count

        def rec_count():
            real()
            countdown.append(int(pl._latent_step_count))
        pl._reset_latent_step_count = rec_count
    np.random.seed(fx['np_seed'])
    res, lines = _run_captured(pl)
    lines_equal(lines, fx['lines'])
    assert countdown[:len(fx['rec']['countdown'])] == fx['rec']['countdown']
    k = fx['actions'].shape[0]
    assert len(env.actions) >= k
    mine = torch.stack(env.actions[:k]).cpu()
    ref = fx['actions']
    err = float((mine - ref).abs().max())
    assert err <= 1e-4 * max(1.0, float(ref.abs().max())), (kind, i, backend, err)
    assert res['games_played'] >= fx['games_num'] or n == 1


def test_action_head_is_the_reference_formula_bit_for_bit():
    """ase_player_act against the reference's op sequence in fp32 torch on the same device: Normal.sample as loc + scale * eps,
    clamp(-1, 1), rescale_actions(low, high) = a * ((high - low) / 2) + (high + low) / 2.  The normalised copy (F.normalize) reduces in
    another order: 1 ulp-level tolerance."""
    from ase_b200 import ops
    g = torch.Generator().manual_seed(0)
    mu = (torch.randn(777, A, generator=g) * 3.0).cuda()
    logstd = torch.linspace(-2.9, 0.3, A).cuda()
    eps = torch.randn(777, A, generator=g).cuda()
    low, high = torch.tensor(LOW).cuda(), torch.tensor(HIGH).cuda()
    for stochastic in (False, True):
        a = mu + torch.exp(logstd) * eps if stochastic else mu
        a = torch.clamp(a, -1.0, 1.0)
        want = a * ((high - low) / 2.0) + (high + low) / 2.0
        got, unit = torch.empty_like(mu), torch.empty_like(mu)
        ops.player_act(mu, logstd if stochastic else None, low, high, None, 0, actions=got, unit_out=unit, noise=eps if stochastic else None)
        assert torch.equal(got, want), float((got - want).abs().max())
        assert torch.allclose(unit, torch.nn.functional.normalize(a, dim=-1), rtol=1e-6, atol=1e-7)


def test_hrl_player_takes_its_llc_from_a_checkpoint_in_the_shipped_layout(tmp_path):
    """HRLPlayer over a frozen LLC restored from a checkpoint with exactly the key set, shapes and dtypes of the shipped
    ase_llc_reallusion_sword_shield.pth (tests/golden/checkpoint_layout.json)."""
    import json
    import os
    from ase_b200 import configs
    from ase_b200.player import HRLPlayer
    lay = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'checkpoint_layout.json')))['ase_llc_reallusion_sword_shield']
    g = torch.Generator().manual_seed(5)

    def fill(spec):
        return {k: (torch.rand(shape, generator=g, dtype=getattr(torch, dt.split('.')[1])) * 0.1 + (1.0 if 'var' in k or k == 'count' else 0.0))
                for k, (shape, dt) in spec.items()}
    w = {k: fill(lay[k]) for k in ('model', 'running_mean_std', 'reward_mean_std', 'amp_input_mean_std')}
    w.update(epoch=1, frame=0, last_mean_rewards=0.0, env_state=None, optimizer={})
    assert list(w['model']) == list(lay['model'])
    torch.save(w, tmp_path / 'llc.pth')
    n, obs = 8, 253 + TASK
    T = 12
    tb = {'obs_t': torch.randn(T + 1, n, obs, generator=g), 'reset_obs_t': torch.randn(T, n, obs, generator=g),
          'rew_t': torch.rand(T, n, generator=g), 'dones_t': (torch.rand(T, n, generator=g) < 0.3).to(torch.uint8),
          'amp_t': torch.randn(T, n, 1400, generator=g)}
    env = GpuScriptEnv(tb, n, obs_dim=obs, amp_dim=1400, act_low=-np.ones(31), act_high=np.ones(31))
    cfg = configs.make('hrl', vec_env=env, device='cuda:0', net_params=_net(UNITS), llc_checkpoint=str(tmp_path / 'llc.pth'),
                       player={'games_num': 6, 'max_steps': 50})
    with contextlib.redirect_stdout(io.StringIO()):
        pl = HRLPlayer(cfg)
    assert torch.equal(pl._llc.named_parameters()['mu.weight'].cpu(), w['model']['a2c_network.mu.weight'])
    assert torch.equal(pl._llc.amp_input_mean_std.running_var.cpu(), w['amp_input_mean_std']['running_var'])
    res, lines = _run_captured(pl)
    assert res['games_played'] >= 6 and torch.stack(env.actions).abs().max() <= 1.0


def test_philox_run_repeats_from_the_same_seed_and_never_syncs_inside_a_window(tmp_path):
    runs = []
    for rep in range(2):
        env = GpuScriptEnv(PO.tables(N, 8), N)
        pl = _make_player('ase', env, 2, False, 60, 200, tmp_path)
        read = pl._read_window

        def guarded(w, read=read):           # the one host read of a window happens outside the check
            torch.cuda.set_sync_debug_mode(0)
            try:
                return read(w)
            finally:
                torch.cuda.set_sync_debug_mode('error')
        pl._read_window = guarded
        np.random.seed(1)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode('error')
        try:
            res, lines = _run_captured(pl)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        runs.append((res, lines, torch.stack(env.actions).cpu()))
    assert runs[0][0] == runs[1][0] and runs[0][1] == runs[1][1]
    assert torch.equal(runs[0][2], runs[1][2])
    assert runs[0][0]['games_played'] >= 60


def test_restore_from_agent_save_and_player_factory(tmp_path):
    import os, sys
    shims = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle', 'shims')
    if shims not in sys.path:
        sys.path.insert(0, shims)
    from rl_games.common import env_configurations, object_factory
    from ase_b200 import configs
    from ase_b200.agent import ASEAgent
    from ase_b200.player import ASEPlayer
    env = GpuScriptEnv(PO.tables(N, 9), N)
    ag = ASEAgent('t', configs.make('ase', vec_env=env, device='cuda:0', num_actors=N, horizon_length=2, minibatch_size=2 * N,
                                    amp_minibatch_size=N, net_params=_net(UNITS), seed=4))
    ag.model.running_mean_std.running_mean.uniform_(-0.5, 0.5)
    fn = ag.save(str(tmp_path / 'nn' / 'Humanoid'))
    # run.py:147-150,156-166: the env registered under the config's env_name, the players by algo name; no 'vec_env' key, so the player
    # creates its env through rl_games.common.env_configurations as BasePlayer does
    env_configurations.register('rlgpu', {'env_creator': lambda **kw: env, 'vecenv_type': 'RLGPU'})
    player_factory = object_factory.ObjectFactory()
    player_factory.register_builder('ase', lambda **kwargs: ASEPlayer(**kwargs))
    cfg = configs.make('ase', device='cuda:0', net_params=_net(UNITS), player={'games_num': 5, 'max_steps': 20})
    assert cfg['env_name'] == 'rlgpu' and 'vec_env' not in cfg
    pl = player_factory.create('ase', config=cfg)
    assert pl.env is env
    assert isinstance(pl, ASEPlayer)
    pl.restore(fn)
    assert torch.equal(pl.model.params, ag.model.params)
    assert torch.equal(pl.model.running_mean_std.running_mean, ag.model.running_mean_std.running_mean)
    assert torch.equal(pl.model.amp_input_mean_std.running_var, ag.model.amp_input_mean_std.running_var)
    res, lines = _run_captured(pl)
    assert res['games_played'] >= 5 and lines[-1].startswith('av reward:')
