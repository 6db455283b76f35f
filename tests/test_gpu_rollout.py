"""GPU tests of the rollout (play_steps / prepare_dataset):

  1. reference-pinned: tests/golden/rollout_ase.pt holds what the reference's own ASEAgent.play_steps + prepare_dataset produced over a
     scripted vec-env with every random draw recorded (oracle/gen_golden.py gen_rollout).  The agent's reference-order rollout, fed the same
     env script and the same draws, must reproduce every experience-buffer tensor, the latents / latent horizons / progress counters it
     leaves behind, the returns and the prepared dataset.
  2. the device rollout (mask-driven resets, in-kernel draws, no host sync) must be the same function of (env script, per-env draws) as
     the reference-order rollout -- checked with injected per-env draw tables -- and must not synchronise (torch sync-debug mode);
  3. the CUDA-graph replay of the device rollout must produce bit-identical buffers to its eager run with the same Philox counter."""
import pytest
import torch

import ase_oracle as O
import synth
import golden_util as G

pytestmark = pytest.mark.gpu


class _Task:
    def __init__(self, n, progress):
        self.num_envs, self.viewer = n, None
        self.progress_buf = progress.clone().cuda()

    def get_task_obs_size(self):
        return 0


class ScriptedEnv:
    """CUDA twin of oracle/ref_harness.FakeVecEnv + the script gen_rollout used: observations / rewards / dones / AMP observations are
    tables indexed by the step counter; reset(env_ids) zeroes progress_buf and swaps in rows of the reset table."""

    def __init__(self, fx, masked=False):
        import numpy as np
        self.fx = fx
        self.N = fx['N']
        self.t = 0
        self.obs_t, self.reset_obs_t = fx['obs_t'].cuda(), fx['reset_obs_t'].cuda()
        self.amp_t, self.rew_t = fx['amp_t'].cuda(), fx['rew_t'].cuda()
        self.dones_t, self.term_t = fx['dones_t'].cuda(), fx['term_t'].cuda()
        # state after train()'s initial full reset (common_agent.py:89 env_reset(None)): progress 0 everywhere, observations from the
        # reset table of step 0 -- that is where gen_rollout's play_steps started from
        self.task = _Task(self.N, torch.zeros_like(fx['progress0']))
        self.env = self
        self.cur = self.reset_obs_t[0].clone()

        class Box:
            def __init__(s, d): s.shape = (d,); s.low = -np.ones(d, dtype=np.float32); s.high = np.ones(d, dtype=np.float32)
        self.observation_space, self.amp_observation_space, self.action_space = Box(253), Box(1400), Box(31)
        if masked:
            self.reset_done = self._reset_done

    def get_env_info(self):
        return {'action_space': self.action_space, 'observation_space': self.observation_space, 'amp_observation_space': self.amp_observation_space}

    def step(self, actions):
        t = self.t
        self.cur = self.obs_t[t + 1].clone()
        self.t += 1
        self.task.progress_buf += 1
        return self.cur, self.rew_t[t].clone(), self.dones_t[t].clone(), {'amp_obs': self.amp_t[t].clone(), 'terminate': self.term_t[t].clone()}

    def reset(self, env_ids=None):
        if env_ids is None:
            env_ids = torch.arange(self.N, device='cuda')
        if len(env_ids) > 0:
            self.task.progress_buf[env_ids] = 0
            self.cur[env_ids] = self.reset_obs_t[self.t][env_ids]
        return self.cur

    def _reset_done(self, mask):
        m = mask.bool()
        self.task.progress_buf.masked_fill_(m, 0)
        self.cur = torch.where(m.unsqueeze(1), self.reset_obs_t[self.t], self.cur)
        return self.cur

    def fetch_amp_obs_demo(self, n):
        return torch.zeros(n, 1400, device='cuda')


def _agent(fx, env, **over):
    from ase_b200 import configs
    from ase_b200.agent import ASEAgent
    cfg = configs.make('ase', device='cuda:0', vec_env=env, num_actors=fx['N'], horizon_length=fx['H'], minibatch_size=64, amp_minibatch_size=32,
                       latent_steps_min=1, latent_steps_max=6, print_stats=False, amp_obs_demo_buffer_size=256, amp_replay_buffer_size=256,
                       amp_batch_size=32, **over)
    cfg['net_params']['mlp']['units'] = list(fx['units']); cfg['net_params']['disc']['units'] = list(fx['disc_units'])
    ag = ASEAgent('t', cfg)
    P = synth.params(O.ase_param_shapes(units=fx['units'], disc_units=fx['disc_units']), seed=fx['param_seed'])
    ag.model.load_named(P)
    ag.model.set_stats_weights({k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in fx['rms_state'].items()})
    ag.init_tensors()
    return ag


def _close(a, b, name, rtol=1e-4, atol=1e-5):
    a, b = a.detach().cpu().float(), b.detach().cpu().float()
    assert a.shape == b.shape, (name, a.shape, b.shape)
    assert torch.allclose(a, b, rtol=rtol, atol=atol), (name, float((a - b).abs().max()))


def test_play_steps_and_prepare_dataset_vs_reference_golden():
    fx = G.load('rollout_ase.pt')
    env = ScriptedEnv(fx)
    ag = _agent(fx, env, device_rollout=False)
    rec = {k: [t.cuda() for t in v] for k, v in fx['rec'].items()}
    cur = {k: 0 for k in rec}

    def take(k):
        v = rec[k][cur[k]]; cur[k] += 1
        return v
    ag._draw_normal = lambda shape: take('normal')
    ag._draw_bernoulli = lambda p: take('bernoulli')
    ag._sample_latents = lambda n: take('latents')
    ag._draw_latent_steps = lambda n: take('randint').to(torch.int32)
    # state train() leaves behind before the first epoch (the draws of that initial full reset are in the fixture too)
    ag._ase_latents.copy_(fx['latents0'].cuda()); ag._latent_reset_steps.copy_(fx['steps0'].cuda().to(torch.int32))
    ag.obs = {'obs': env.cur}
    with torch.no_grad():
        bd = ag.play_steps()
    for k in rec:
        assert cur[k] == len(rec[k]), f"{k}: the rollout consumed {cur[k]} draws, the reference {len(rec[k])}"
    eb = ag.experience_buffer
    for k, ref in fx['eb'].items():
        mine = eb[k]
        if k == 'dones':
            assert torch.equal(mine.cpu(), ref.to(torch.uint8)), k
        else:
            _close(mine, ref, 'eb.' + k)
    _close(eb['amp_obs'], fx['amp_t'], 'eb.amp_obs', 0, 0); _close(eb['next_obses'], fx['obs_t'][1:], 'eb.next_obses', 0, 0)
    _close(ag._ase_latents, fx['latents_end'], 'latents_end', 0, 1e-7)
    assert torch.equal(ag._latent_reset_steps.cpu().long(), fx['steps_end'].long())
    assert torch.equal(env.task.progress_buf.cpu(), fx['progress_end'])
    for k, ref in fx['batch'].items():
        _close(bd[k], ref, 'batch.' + k)
    ag.set_train()
    bd.pop('played_frames')
    ag.prepare_dataset(bd)
    for k, ref in fx['dataset'].items():
        mine = ag.dataset.values_dict[k] if k in ag.dataset.values_dict else None
        assert mine is not None, k
        _close(mine.reshape(ref.shape), ref, 'dataset.' + k, rtol=2e-4, atol=2e-5)
    v = fx['value_rms_after']
    _close(ag.model.value_mean_std.running_mean, v['running_mean'], 'value_rms.mean', 1e-6, 1e-7)
    _close(ag.model.value_mean_std.running_var, v['running_var'], 'value_rms.var', 1e-5, 1e-8)
    assert float(ag.model.value_mean_std.count) == float(v['count'])


def _tables(fx, seed):
    g = torch.Generator().manual_seed(seed)
    H, N = fx['H'], fx['N']
    return dict(noise=torch.randn(H, N, 31, generator=g).cuda(), mask=(torch.rand(H, N, generator=g) < 0.7).float().cuda(),
                z=torch.nn.functional.normalize(torch.randn(H, N, 64, generator=g), dim=-1).cuda(),
                steps=torch.randint(1, 6, (H, N), generator=g, dtype=torch.int32).cuda())


def reference_order_rollout(fx, tb):
    """The reference-order rollout drawing from the per-env tables tb (noise / mask / z / steps, each [H, N, ...]) -> (agent, env)."""
    env_a = ScriptedEnv(fx)
    a = _agent(fx, env_a, device_rollout=False)
    step = {'n': -1}
    a._draw_normal = lambda shape: (step.__setitem__('n', step['n'] + 1), tb['noise'][step['n']])[1]
    a._draw_bernoulli = lambda p: tb['mask'][step['n']]
    # env_reset and _update_latents of step n run before that step's action noise is drawn: both read row n = step['n'] + 1
    a._reset_latents = lambda ids: a._ase_latents.__setitem__(ids, tb['z'][step['n'] + 1][ids])

    def pre():
        n = step['n'] + 1
        new = a._latent_reset_steps <= env_a.task.progress_buf
        ids = new.nonzero(as_tuple=False).flatten()
        if ids.numel() > 0:
            a._ase_latents[ids] = tb['z'][n][ids]
            a._latent_reset_steps[ids] += tb['steps'][n][ids]
    a._pre_action = pre
    a._reset_latent_step_count = lambda ids: a._latent_reset_steps.__setitem__(ids, tb['steps'][step['n'] + 1][ids])
    a._ase_latents.copy_(fx['latents0'].cuda()); a._latent_reset_steps.copy_(fx['steps0'].cuda().to(torch.int32))
    a.obs = {'obs': env_a.cur}
    with torch.no_grad():
        a.play_steps()
    return a, env_a


def test_device_rollout_equals_reference_order_rollout_and_never_syncs():
    fx = G.load('rollout_ase.pt')
    tb = _tables(fx, 5)
    # (a) reference-order rollout drawing from per-env tables
    a, env_a = reference_order_rollout(fx, tb)
    # (b) device rollout with the same tables injected into the kernels
    env_b = ScriptedEnv(fx, masked=True)
    b = _agent(fx, env_b, device_rollout=True, rollout_graph=False)
    b._ase_latents.copy_(fx['latents0'].cuda()); b._latent_reset_steps.copy_(fx['steps0'].cuda().to(torch.int32))
    b._inject = tb
    b.obs = {'obs': env_b.cur}
    b.model.eval_actor_critic(env_b.cur, b._ase_latents)         # warm every lazily initialised path before forbidding syncs
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        with torch.no_grad():
            b.set_eval()
            b._rollout_loop()
    finally:
        torch.cuda.set_sync_debug_mode('default')
    for k in a.experience_buffer:
        x, y = a.experience_buffer[k], b.experience_buffer[k]
        if x.dtype == torch.uint8:
            assert torch.equal(x, y), k
        else:
            _close(x, y, 'eb.' + k, rtol=1e-5, atol=1e-6)
    _close(a._ase_latents, b._ase_latents, 'latents', 0, 0)
    assert torch.equal(a._latent_reset_steps, b._latent_reset_steps)
    assert torch.equal(env_a.task.progress_buf, env_b.task.progress_buf)
    _close(a.current_rewards, b.current_rewards, 'current_rewards', 1e-6, 1e-6)
    _close(a._episode_meter, b._episode_meter, 'episode meter', 1e-5, 1e-5)


def _synthetic_agent(graph, seed=3):
    from ase_b200 import configs
    from ase_b200.agent import ASEAgent
    from ase_b200.synthetic_env import SyntheticHumanoidEnv
    torch.manual_seed(seed)
    env = SyntheticHumanoidEnv(64, device='cuda', seed=3, done_prob=0.05, demo_pool=512, pool=4)
    cfg = configs.make('ase', device='cuda:0', vec_env=env, num_actors=64, horizon_length=8, minibatch_size=128, amp_minibatch_size=32, mini_epochs=2,
                       amp_obs_demo_buffer_size=2048, amp_replay_buffer_size=2048, amp_batch_size=64, print_stats=False, rollout_graph=graph, seed=11,
                       latent_steps_min=1, latent_steps_max=12)
    cfg['net_params']['mlp']['units'] = [128, 96, 64]; cfg['net_params']['disc']['units'] = [128, 96, 64]
    ag = ASEAgent('t', cfg)
    ag.init_tensors(); ag.obs = ag.env_reset(); ag._init_train()
    return ag, env


def test_cuda_graph_rollout_matches_eager_and_persists_state():
    """Same seeds, same Philox counters: 5 epochs with the rollout replayed from a CUDA graph (captured at epoch 3) must leave the same
    experience buffers, latents and env progress as 5 eager epochs; the default torch generator (env dones) is graph-safe."""
    res = []
    for graph in (False, True):
        ag, env = _synthetic_agent(graph)
        snaps = []
        for ep in range(5):
            torch.manual_seed(100 + ep)          # the env's per-step draws come from the default generator
            ag.update_epoch(); ag.train_epoch()
            snaps.append({k: v.clone() for k, v in ag.experience_buffer.items()})
        assert (ag._rollout_graph is not None) == graph
        res.append((snaps, ag._ase_latents.clone(), env.task.progress_buf.clone(), int(ag._rng[1])))
    (s0, l0, p0, c0), (s1, l1, p1, c1) = res
    assert c0 == c1 == 5 * 8
    # epoch 0's rollout precedes any training: bit for bit
    for k in s0[0]:
        assert torch.equal(s0[0][k], s1[0][k]), k
    # later epochs: the parameters of the two runs differ in the last bits (split-K / column-sum REDs are unordered), the draws do not:
    # masks, dones, latents bit-equal; everything computed from the networks to 1e-4
    for ep in (1, 2, 3, 4):
        for k in s0[ep]:
            if s0[ep][k].dtype == torch.uint8 or k in ('rand_action_mask', 'ase_latents'):
                assert torch.equal(s0[ep][k], s1[ep][k]), (ep, k)
            else:
                _close(s0[ep][k], s1[ep][k], f'epoch {ep} eb.{k}', rtol=1e-4, atol=1e-4)
    _close(l0, l1, 'latents', 0, 0)
    assert torch.equal(p0, p1)


def test_rollout_state_persists_across_play_steps():
    """ADVICE r1 (high): a rollout must not start by resetting every env and every latent (`done_indices = []`, amp_agent.py:64)."""
    for dev in (False, True):
        from ase_b200 import configs
        ag, env = _synthetic_agent(False)
        ag._device_rollout = dev
        env.done_prob = 0.0
        ag._latent_steps_min, ag._latent_steps_max = 1000, 1001
        ag._latent_reset_steps[:] = 5000
        with torch.no_grad():
            ag.play_steps()
        lat, prog = ag._ase_latents.clone(), env.task.progress_buf.clone()
        with torch.no_grad():
            ag.play_steps()
        assert torch.equal(ag._ase_latents, lat), "latents were resampled at the start of a rollout"
        assert torch.equal(env.task.progress_buf, prog + ag.horizon_length), "envs were reset at the start of a rollout"


def test_compute_humanoid_reset_vs_reference_golden():
    from ase_b200 import ops
    fx = G.load('humanoid_reset.pt')
    N, J = fx['pos'].shape[:2]
    body = torch.zeros(N, J, 13); body[..., 0:3] = fx['pos']
    is_contact = torch.zeros(J, dtype=torch.uint8); is_contact[fx['contact_body_ids']] = 1
    for et in (1, 0):
        r, t = ops.compute_humanoid_reset(fx['progress'].cuda(), fx['contact'].cuda(), is_contact.cuda(), body.cuda(), fx['max_episode_length'], bool(et),
                                          fx['heights'].cuda())
        assert torch.equal(r.cpu().long(), fx[f'reset_{et}'].long()), et
        assert torch.equal(t.cpu().long(), fx[f'term_{et}'].long()), et


def test_save_restore_roundtrip_and_reference_checkpoint_layout(tmp_path):
    """save() / restore() (common_agent.py:141-170): the file has the rl_games layout (SURVEY.md Appendix B: model incl. the _enc_mlp
    aliases and sigma, f64 RMS buffers, torch.optim.Adam state with `step`), restore() brings back parameters, Adam moments, RMS
    statistics, epoch and frame; training continues identically from the restored state."""
    ag, env = _synthetic_agent(False)
    for _ in range(2):
        ag.update_epoch(); ag.train_epoch()
    ag.frame = 1234
    fn = ag.save(str(tmp_path / 'ckpt'))
    w = torch.load(fn, map_location='cpu', weights_only=False)
    assert set(w.keys()) >= {'model', 'running_mean_std', 'reward_mean_std', 'amp_input_mean_std', 'optimizer', 'epoch', 'frame', 'last_mean_rewards'}
    assert 'a2c_network.sigma' in w['model'] and 'a2c_network._enc_mlp.0.weight' in w['model'] and 'a2c_network._disc_mlp.0.weight' in w['model']
    assert w['running_mean_std']['running_mean'].dtype == torch.float64 and w['amp_input_mean_std']['count'].dtype == torch.float64
    st1 = w['optimizer']['state'][1]
    assert set(st1.keys()) == {'step', 'exp_avg', 'exp_avg_sq'} and 0 not in w['optimizer']['state']      # param 0 = frozen sigma: no state
    ag2, env2 = _synthetic_agent(False, seed=9)
    ag2.restore(fn)
    assert ag2.epoch_num == ag.epoch_num and ag2.frame == 1234 and ag2.model.step == ag.model.step
    assert torch.equal(ag2.model.params, ag.model.params) and torch.equal(ag2.model.exp_avg, ag.model.exp_avg)
    assert torch.equal(ag2.model.exp_avg_sq, ag.model.exp_avg_sq)
    assert torch.equal(ag2.model.running_mean_std.running_var, ag.model.running_mean_std.running_var)
    assert torch.equal(ag2.model.amp_input_mean_std.running_mean, ag.model.amp_input_mean_std.running_mean)
    # one more identical minibatch update on both
    d = {k: torch.randn_like(v) if v.dtype == torch.float32 else v for k, v in ag._mb_bufs.items()}
    d['rand_action_mask'] = (d['rand_action_mask'] > 0).float()
    d['sigma'] = d['sigma'].abs() + 0.05
    nz = torch.nn.functional.normalize(torch.randn(ag.minibatch_size, 64, device='cuda'), dim=-1)
    outs = []
    for a in (ag, ag2):
        a.model.calc_gradients(d, nz)
        a.model.adam_step()
        outs.append(a.model.params.clone())
    assert torch.allclose(outs[0], outs[1], rtol=0, atol=1e-6)


def test_train_loop_saves_checkpoints_and_stops_after_max_epochs(tmp_path):
    ag, env = _synthetic_agent(False)
    ag.max_epochs, ag.save_freq = 3, 2
    ag.train_dir, ag.experiment_name = str(tmp_path), 'exp'
    import os
    ag.nn_dir = os.path.join(str(tmp_path), 'exp', 'nn')
    _, epochs = ag.train()
    assert epochs == 4                               # `epoch_num > max_epochs` (common_agent.py:149): one more than max_epochs
    assert os.path.exists(os.path.join(ag.nn_dir, ag.config.get('name', 't') + '.pth'))
    assert all('plane_status' not in r['scalars'] for r in ag.epoch_log) and len(ag.epoch_log) == 4
