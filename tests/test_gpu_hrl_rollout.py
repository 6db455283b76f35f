"""GPU tests of the HRL rollout (HRLAgent.play_steps over a frozen full-size ASE LLC, config 5):

  1. reference-pinned: tests/golden/rollout_hrl.pt holds what the reference's own HRLAgent produced over a scripted vec-env (oracle/
     gen_golden_hrl_rollout.py): every experience-buffer tensor, the LLC actions it passed to each env sub-step, the returns and the prepared
     dataset.  The agent's reference-order rollout, fed the same script and the recorded HLC draws, must reproduce them on every GEMM
     backend, and the worst errors against the fixture and the fp64 oracle (oracle/hrl_rollout_oracle.py) are printed;
  2. the device rollout (mask-driven resets, no host sync) fed the same draws equals the reference-order rollout;
  3. the CUDA-graph replay of the device rollout is bit-identical to its eager run from the same Philox counter;
  4. the logged mean episode reward is llc_steps x the mean of the finished episodes' accumulated (per-step mean) rewards, as the
     reference's HRLAgent._get_mean_rewards reports it."""
import numpy as np
import pytest
import torch

import golden_util as G
import hrl_rollout_oracle as HO
import synth

pytestmark = pytest.mark.gpu


class _Task:
    def __init__(self, n):
        self.num_envs, self.viewer = n, None
        self.progress_buf = torch.zeros(n, dtype=torch.int64, device='cuda')

    def get_task_obs_size(self):
        return 5


class ScriptedHRLEnv:
    """CUDA twin of oracle/ref_harness.FakeVecEnv + the script gen_golden_hrl_rollout used: per-sub-step tables indexed by the step counter,
    resets from the reset table of the current HLC step; the LLC actions passed to step() are recorded into `rec` [K, N, 31]."""

    def __init__(self, fx, masked=False):
        self.N, self.L = fx['N'], fx['llc_steps']
        K = fx['H'] * self.L
        self.obs_t, self.reset_obs_t, self.amp_t = fx['obs_t'].cuda(), fx['reset_obs_t'].cuda(), fx['amp_t'].cuda()
        self.rew_t, self.dones_t, self.term_t = fx['rew_t'].cuda(), fx['dones_t'].cuda(), fx['term_t'].cuda()
        self.rec = torch.zeros(K, self.N, 31, device='cuda')
        self.task = _Task(self.N)
        self.env = self

        class Box:
            def __init__(s, d): s.shape = (d,); s.low = -np.ones(d, dtype=np.float32); s.high = np.ones(d, dtype=np.float32)
        self.observation_space, self.amp_observation_space, self.action_space = Box(258), Box(1400), Box(31)
        if masked:
            self.reset_done = self._reset_done
        self.rewind()

    def rewind(self):
        """State after train()'s initial env_reset(None): that is where the reference's play_steps started from."""
        self.t = 0
        self.cur = self.reset_obs_t[0].clone()
        self.task.progress_buf.zero_()
        self.rec.zero_()

    def get_env_info(self):
        return {'action_space': self.action_space, 'observation_space': self.observation_space, 'amp_observation_space': self.amp_observation_space}

    def step(self, actions):
        t = self.t
        self.rec[t].copy_(actions)
        self.cur = self.obs_t[t + 1].clone()
        self.t += 1
        self.task.progress_buf += 1
        return self.cur, self.rew_t[t].clone(), self.dones_t[t].clone(), {'amp_obs': self.amp_t[t].clone(), 'terminate': self.term_t[t].clone()}

    def reset(self, env_ids=None):
        if env_ids is None:
            env_ids = torch.arange(self.N, device='cuda')
        if len(env_ids) > 0:
            self.task.progress_buf[env_ids] = 0
            self.cur[env_ids] = self.reset_obs_t[self.t // self.L][env_ids]
        return self.cur

    def _reset_done(self, mask):
        m = mask.bool()
        self.task.progress_buf.masked_fill_(m, 0)
        self.cur = torch.where(m.unsqueeze(1), self.reset_obs_t[self.t // self.L], self.cur)
        return self.cur


_CACHE = {}


def _fixture():
    if 'fx' not in _CACHE:
        _CACHE['fx'] = G.load('rollout_hrl.pt')
    return _CACHE['fx']


def _fp64():
    if 'fp64' not in _CACHE:
        fx = _fixture()
        _CACHE['fp64'] = HO.rollout(fx, synth.hrl_hlc_params(), synth.hrl_llc_params(), fx['hlc_sigma'], torch.float64)
    return _CACHE['fp64']


@pytest.fixture(scope='module')
def llc_checkpoint(tmp_path_factory):
    """The LLC as an rl_games checkpoint (what config['llc_checkpoint'] names): the fixture's seeded weights and shipped statistics."""
    fx = _fixture()
    w = {'model': {'a2c_network.' + k: v for k, v in synth.hrl_llc_params().items()}}
    w.update({k: {kk: vv.clone() for kk, vv in v.items()} for k, v in fx['llc_rms'].items()})
    fn = str(tmp_path_factory.mktemp('llc') / 'llc.pth')
    torch.save(w, fn)
    return fn


def _agent(fx, env, ckpt, backend, **over):
    from ase_b200 import configs
    from ase_b200.agent import HRLAgent
    N, H = fx['N'], fx['H']
    cfg = configs.make('hrl', device='cuda:0', vec_env=env, num_actors=N, horizon_length=H, minibatch_size=N * H // 2, print_stats=False,
                       gemm_backend=backend, llc_checkpoint=ckpt, **over)
    ag = HRLAgent('t', cfg)
    ag.model.load_named(synth.hrl_hlc_params())           # the log-std stays the config's constant
    ag.model.set_stats_weights({k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in fx['hlc_rms'].items()})
    ag.init_tensors()
    ag.obs = {'obs': env.cur}
    return ag


def _err(a, b):
    """Worst absolute difference relative to max(1, |reference|)."""
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    assert a.shape == b.shape, (a.shape, b.shape)
    return float(((a - b).abs() / b.abs().clamp_min(1.0)).max())


def _close(a, b, name, rtol=1e-4, atol=1e-5):
    a, b = a.detach().cpu().float(), b.detach().cpu().float()
    assert a.shape == b.shape, (name, a.shape, b.shape)
    assert torch.allclose(a, b, rtol=rtol, atol=atol), (name, float((a - b).abs().max()))


def reference_order_rollout(fx, ckpt, backend):
    env = ScriptedHRLEnv(fx)
    ag = _agent(fx, env, ckpt, backend, device_rollout=False)
    rec = [t.cuda() for t in fx['rec']['normal']]
    used = [0]

    def take(shape):
        v = rec[used[0]]; used[0] += 1
        assert tuple(shape) == tuple(v.shape)
        return v
    ag._draw_normal = take
    with torch.no_grad():
        bd = ag.play_steps()
    assert used[0] == len(rec), f"the rollout consumed {used[0]} HLC draws, the reference {len(rec)}"
    assert env.t == fx['H'] * fx['llc_steps']
    return ag, env, bd


@pytest.mark.parametrize('backend', [0, 1, 2])
def test_reference_order_hrl_rollout_vs_reference_golden(backend, llc_checkpoint):
    fx = _fixture()
    ag, env, bd = reference_order_rollout(fx, llc_checkpoint, backend)
    eb = ag.experience_buffer
    for k, ref in fx['eb'].items():
        if k == 'dones':
            assert torch.equal(eb[k].cpu(), ref.to(torch.uint8)), k
        else:
            _close(eb[k], ref, 'eb.' + k)
    _close(eb['next_obses'], fx['obs_t'][fx['llc_steps']::fx['llc_steps']], 'eb.next_obses', 0, 0)
    _close(env.rec, fx['llc_actions'], 'llc_actions')
    _close(bd['returns'], fx['returns'], 'returns')
    if backend == 2:
        assert ag._llc.plane_status() == 0 and ag.model.plane_status() == 0
    # the numbers the fixture does not bound tightly: worst errors against the reference (fp32) and the fp64 oracle
    o64 = _fp64()
    rep = {k: (_err(m, r32), _err(m, r64)) for k, m, r32, r64 in (
        ('llc_actions', env.rec, fx['llc_actions'], o64['llc_actions']),
        ('disc_rewards', eb['disc_rewards'], fx['eb']['disc_rewards'], o64['eb']['disc_rewards']),
        ('values', eb['values'], fx['eb']['values'], o64['eb']['values']),
        ('returns', bd['returns'], fx['returns'], o64['returns']))}
    ref_vs_64 = {k: _err(r32, r64) for k, r32, r64 in (('llc_actions', fx['llc_actions'], o64['llc_actions']),
                                                       ('disc_rewards', fx['eb']['disc_rewards'], o64['eb']['disc_rewards']),
                                                       ('values', fx['eb']['values'], o64['eb']['values']), ('returns', fx['returns'], o64['returns']))}
    print(f'\nHRL rollout backend {backend}: worst error (vs reference fp32, vs fp64) ' +
          ', '.join(f'{k} ({a:.2e}, {b:.2e})' for k, (a, b) in rep.items()) +
          '; reference fp32 vs fp64 ' + ', '.join(f'{k} {v:.2e}' for k, v in ref_vs_64.items()))
    ag.set_train()
    bd.pop('played_frames')
    ag.prepare_dataset(bd)
    _close(ag.dataset.values_dict['advantages'].reshape(fx['dataset']['advantages'].shape), fx['dataset']['advantages'], 'dataset.advantages', 2e-4, 2e-5)
    v = fx['value_rms_after']
    _close(ag.model.value_mean_std.running_mean, v['running_mean'], 'value_rms.mean', 1e-6, 1e-7)
    _close(ag.model.value_mean_std.running_var, v['running_var'], 'value_rms.var', 1e-5, 1e-8)
    assert float(ag.model.value_mean_std.count) == float(v['count'])


def _rewind(ag, env, rng0):
    """Back to the state the rollout started from, writing device state in place (a captured graph reads these very tensors)."""
    env.rewind()
    ag.obs = {'obs': env.cur}
    ag._rng.copy_(rng0)
    ag.current_rewards.zero_(); ag.current_lengths.zero_(); ag._episode_meter.zero_()


@pytest.mark.parametrize('backend', [0, 2])
def test_device_hrl_rollout_equals_reference_order_and_never_syncs(backend, llc_checkpoint):
    fx = _fixture()
    a, env_a, _ = reference_order_rollout(fx, llc_checkpoint, backend)
    env_b = ScriptedHRLEnv(fx, masked=True)
    b = _agent(fx, env_b, llc_checkpoint, backend, device_rollout=True, rollout_graph=False)
    b._inject = {'noise': torch.stack(fx['rec']['normal']).cuda()}
    rng0 = b._rng.clone()
    with torch.no_grad():
        b.set_eval()
        b._rollout_loop()                          # warms every lazily initialised path (and the plane scales) before syncs are forbidden
    _rewind(b, env_b, rng0)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        with torch.no_grad():
            b._rollout_loop()
    finally:
        torch.cuda.set_sync_debug_mode('default')
    for k in a.experience_buffer:
        x, y = a.experience_buffer[k], b.experience_buffer[k]
        if x.dtype == torch.uint8:
            assert torch.equal(x, y), k
        else:
            _close(x, y, 'eb.' + k, rtol=1e-5, atol=1e-6)
    _close(env_a.rec, env_b.rec, 'llc_actions', rtol=1e-5, atol=1e-6)
    _close(a.current_rewards, b.current_rewards, 'current_rewards', 1e-6, 1e-6)
    _close(a._episode_meter, b._episode_meter, 'episode meter', 1e-5, 1e-5)
    if backend == 2:
        assert b._llc.plane_status() == 0


@pytest.mark.parametrize('backend', [0, 2])
def test_hrl_rollout_graph_replay_is_bit_identical_to_eager(backend, llc_checkpoint):
    """In-kernel Philox draws (no injection): the captured HRL rollout replays exactly what the eager device rollout computed."""
    fx = _fixture()
    env = ScriptedHRLEnv(fx, masked=True)
    ag = _agent(fx, env, llc_checkpoint, backend, device_rollout=True)
    rng0 = ag._rng.clone()
    with torch.no_grad():
        ag.set_eval()
        ag._rollout_loop()                         # settles the plane scales, as _play_steps_device does before it captures
        _rewind(ag, env, rng0)
        ag._rollout_loop()
        torch.cuda.synchronize()
        eager = {k: v.clone() for k, v in ag.experience_buffer.items()}
        eager.update(llc_actions=env.rec.clone(), rng=ag._rng.clone(), current_rewards=ag.current_rewards.clone(), meter=ag._episode_meter.clone())
        _rewind(ag, env, rng0)
        for b in ag.experience_buffer.values():
            b.zero_()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):                  # capture does not execute: the device state is still the rewound one
            ag._rollout_loop()
        g.replay()
    torch.cuda.synchronize()
    replay = {k: v for k, v in ag.experience_buffer.items()}
    replay.update(llc_actions=env.rec, rng=ag._rng, current_rewards=ag.current_rewards, meter=ag._episode_meter)
    assert int(eager['rng'][1]) == int(rng0[1]) + fx['H']
    for k, v in eager.items():
        assert torch.equal(v, replay[k]), k
    assert float(eager['actions'].std()) > 0 and eager['dones'].any()


def test_hrl_logged_mean_reward_is_llc_steps_times_episode_mean(tmp_path):
    """hrl_agent.py:172-175: HRLAgent logs llc_steps x the mean accumulated reward of the finished episodes (each HLC step accumulates the
    mean of its llc_steps sub-step rewards)."""
    from ase_b200 import configs
    from ase_b200.agent import HRLAgent
    from ase_b200.synthetic_env import SyntheticHumanoidEnv
    torch.manual_seed(2)
    n, h = 64, 8
    env = SyntheticHumanoidEnv(n, device='cuda', seed=4, done_prob=0.05, demo_pool=256, heading_task=True)
    cfg = configs.make('hrl', device='cuda:0', vec_env=env, num_actors=n, horizon_length=h, minibatch_size=128, mini_epochs=1, print_stats=False,
                       gemm_backend=0, max_epochs=3, train_dir=str(tmp_path))
    cfg['net_params']['mlp']['units'] = [128, 64]
    cfg['llc_net_params'] = {'mlp': {'units': [128, 96, 64]}, 'disc': {'units': [128, 96, 64]}}
    ag = HRLAgent('t', cfg)
    rollouts = []
    play = ag.play_steps

    def recording_play_steps():
        bd = play()
        rollouts.append((ag.experience_buffer['rewards'][..., 0].cpu().double(), ag.experience_buffer['dones'].cpu().bool()))
        return bd
    ag.play_steps = recording_play_steps
    ag.train()
    assert len(rollouts) == len(ag.epoch_log) == 4
    cur = torch.zeros(n, dtype=torch.float64)
    checked = 0
    for (rew, dones), r in zip(rollouts, ag.epoch_log):
        total, count = 0.0, 0
        for t in range(h):
            cur += rew[t]
            total += float(cur[dones[t]].sum()); count += int(dones[t].sum())
            cur[dones[t]] = 0.0
        if count:
            expect = ag._llc_steps * total / count
            assert abs(r['mean_rewards'] - expect) <= 1e-5 * max(1.0, abs(expect)), (r['epoch'], r['mean_rewards'], expect, r['mean_rewards'] / expect)
            checked += 1
    assert checked >= 2
