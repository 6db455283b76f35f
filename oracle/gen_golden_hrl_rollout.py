"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/rollout_hrl.pt by executing the UNMODIFIED reference HRLAgent (the checkout named by
ASE_REFERENCE_ROOT, through oracle/shims): HRLAgent.__init__ reads the reference's own ase_humanoid_hrl.yaml as its llc_config and
restores an rl_games-layout LLC checkpoint, both written to a temporary directory; then train()'s initial reset, play_steps and
prepare_dataset run over a scripted vec-env (ref_harness.FakeVecEnv) whose tables synth.hrl_rollout_script regenerates from a seed.
The HLC's Normal.sample draws are recorded in call order, and so are the LLC actions the reference passes to each env step.
Usage: python oracle/gen_golden_hrl_rollout.py"""
import copy
import json
import os
import shutil
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_harness as rh          # noqa: E402
import synth                      # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), 'tests', 'golden')
DISC_FLOOR = 1e-4


def _llc_checkpoint(path, P, llc_rms):
    """An rl_games checkpoint of the LLC (the layout of the shipped ase_llc_*.pth, tests/golden/checkpoint_layout.json): the reference's
    own ASEAgent at production widths holding the seeded weights and the shipped normaliser statistics writes it."""
    agent, _ = rh.make_ref_agent('ase', num_envs=8, overrides={'minibatch_size': 256, 'amp_minibatch_size': 64})
    sd = {'a2c_network.' + k: v.clone() for k, v in P.items()}
    for k in list(sd):
        if '_disc_mlp' in k:
            sd[k.replace('_disc_mlp', '_enc_mlp')] = sd[k]
    agent.model.load_state_dict(sd, strict=True)
    agent.running_mean_std.load_state_dict(llc_rms['running_mean_std'])
    agent.value_mean_std.load_state_dict(llc_rms['reward_mean_std'])
    agent._amp_input_mean_std.load_state_dict(llc_rms['amp_input_mean_std'])
    w = agent.get_full_state_weights()
    w['env_state'] = None
    lay = json.load(open(os.path.join(OUT, 'checkpoint_layout.json')))['ase_llc_reallusion_sword_shield']
    assert list(w) == list(lay), (list(w), list(lay))
    for k in ('model', 'running_mean_std', 'reward_mean_std', 'amp_input_mean_std'):
        assert {kk: [list(v.shape), str(v.dtype)] for kk, v in w[k].items()} == lay[k], k
    torch.save(w, path)


def _make_hrl_agent(tmp, N, H, vec_env):
    """HRLAgent as rl_games' Runner builds it from hrl_humanoid.yaml (run.py:153-170), over the scripted vec-env."""
    rh._setup_path()
    from rl_games.common import vecenv
    from rl_games.common.tr_helpers import DefaultRewardsShaper
    from learning import hrl_agent, hrl_models, hrl_network_builder
    params = copy.deepcopy(rh.load_train_cfg('hrl_humanoid.yaml'))['params']
    builder = hrl_network_builder.HRLBuilder()
    builder.load(params['network'])
    config = params['config']
    config.update(horizon_length=H, minibatch_size=H * N // 2, llc_checkpoint='llc.pth', env_name='scripted_hrl', num_actors=N, device='cpu')
    config['network'] = hrl_models.ModelHRLContinuous(builder)
    config['reward_shaper'] = DefaultRewardsShaper(**config['reward_shaper'])
    vecenv.register('scripted_hrl', lambda name, n, **kw: vec_env)
    # llc_config names ase/data/cfg/train/rlg/ase_humanoid_hrl.yaml relative to the working directory (hrl_agent.py:29)
    os.makedirs(os.path.join(tmp, os.path.dirname(config['llc_config'])))
    shutil.copy(os.path.join(rh.REF_ROOT, config['llc_config']), os.path.join(tmp, config['llc_config']))
    cwd = os.getcwd()
    os.chdir(tmp)
    try:
        agent = hrl_agent.HRLAgent(base_name='oracle', config=config)
    finally:
        os.chdir(cwd)
    return agent, config


def gen_hrl_rollout():
    N, H, L = 24, 6, 5
    K = H * L
    s = synth.hrl_rollout_script(N=N, H=H, llc_steps=L)
    obs_t, reset_obs_t, amp_t, rew_t, dones_t, term_t = (s[k] for k in ('obs_t', 'reset_obs_t', 'amp_t', 'rew_t', 'dones_t', 'term_t'))
    rh._setup_path()
    vec_env = rh.FakeVecEnv(N, obs_dim=258, amp_dim=1400, act_dim=31)
    vec_env.env.task.get_task_obs_size = lambda: 5
    tmp = tempfile.mkdtemp()
    try:
        _llc_checkpoint(os.path.join(tmp, 'llc.pth'), synth.hrl_llc_params(), s['llc_rms'])
        torch.manual_seed(0)
        agent, config = _make_hrl_agent(tmp, N, H, vec_env)
    finally:
        shutil.rmtree(tmp)
    llc = agent._llc_agent
    assert agent._llc_steps == L and agent._task_size == 5 and agent._latent_dim == 64 and llc._disc_reward_scale == 2
    sigma0 = agent.model.a2c_network.sigma.detach().clone()
    assert torch.all(sigma0 == -2.3), sigma0            # hrl_humanoid.yaml sigma_init
    sd = {'a2c_network.' + k: v.clone() for k, v in synth.hrl_hlc_params().items()}
    sd['a2c_network.sigma'] = sigma0
    agent.model.load_state_dict(sd, strict=True)
    agent.running_mean_std.load_state_dict(s['hlc_rms']['running_mean_std'])
    agent.value_mean_std.load_state_dict(s['hlc_rms']['reward_mean_std'])

    g = torch.Generator().manual_seed(92)
    cur = {'obs': None}
    llc_actions = []

    def script(t, actions):
        llc_actions.append(actions.clone())
        cur['obs'] = obs_t[t + 1].clone()
        return cur['obs'], rew_t[t].clone(), dones_t[t].clone(), {'amp_obs': amp_t[t].clone(), 'terminate': term_t[t].clone()}

    def reset_fn(env_ids):
        if env_ids is None:
            env_ids = torch.arange(N)
        if cur['obs'] is None:
            cur['obs'] = obs_t[0].clone()
        if len(env_ids) > 0:
            cur['obs'][env_ids] = reset_obs_t[vec_env.t // L][env_ids]
        return cur['obs']
    vec_env.script, vec_env.reset_fn = script, reset_fn

    # recorded HLC draws; HLC step 1 drives env 4 beyond +-1 on every action component
    rec = []
    real_sample = torch.distributions.Normal.sample

    def rec_sample(self, sample_shape=torch.Size()):
        eps = torch.randn(self.loc.shape, generator=g)
        if len(rec) == 1:
            eps[4] = torch.sign(self.loc[4]) * (eps[4].abs() + 12.0)
        rec.append(eps.clone())
        return self.loc + self.scale * eps
    # what the LLC sees: its normalised observations and its discriminator logits (instance attributes wrap the reference methods)
    seen = {'llc_obs': [], 'logits': []}
    real_pre, real_disc = llc._preproc_obs, llc._eval_disc
    llc._preproc_obs = lambda x: (lambda y: (seen['llc_obs'].append(y.clone()), y)[1])(real_pre(x))
    llc._eval_disc = lambda x: (lambda y: (seen['logits'].append(y.clone()), y)[1])(real_disc(x))
    torch.distributions.Normal.sample = rec_sample
    try:
        agent.init_tensors()
        agent.obs = agent.env_reset()                    # train(): resets every env
        agent.set_eval()
        with torch.no_grad():
            batch_dict = agent.play_steps()
        agent.set_train()
        batch_dict.pop('played_frames')
        agent.prepare_dataset(batch_dict)
    finally:
        torch.distributions.Normal.sample = real_sample
    assert len(rec) == H and len(llc_actions) == K and len(seen['logits']) == K and vec_env.t == K

    eb = {k: v.clone() for k, v in agent.experience_buffer.tensor_dict.items() if k in (
        'obses', 'actions', 'mus', 'neglogpacs', 'values', 'rewards', 'disc_rewards', 'dones', 'next_values', 'sigmas', 'next_obses')}
    assert torch.equal(eb['next_obses'], obs_t[L::L])
    del eb['next_obses']                               # (== the scripted inputs)
    llc_actions = torch.stack(llc_actions)
    acts = eb['actions']

    # ---- edges
    out_of_range = acts.abs() > 1.0
    assert out_of_range.any() and out_of_range.all(-1).any(), "HLC actions beyond +-1, one row on every component"
    pre = torch.stack(seen['llc_obs'])
    assert int((pre.abs() == 5.0).sum(-1).max()) > 100, "LLC observation rows at the +-5 clamp of the normaliser"
    d = dones_t.view(H, L, N).bool()
    assert d[:, 0].any() and d[:, L // 2].any() and d[:, L - 1].any(), "dones on the first, a middle and the last sub-step"
    assert term_t.view(H, L, N)[:, :L - 1].bool().any(), "a termination inside an HLC step"
    assert dones_t[K - 1].any() and eb['dones'][H - 1].any(), "a done on the rollout's last sub-step"
    logits = torch.stack(seen['logits'])
    floor = (1 - 1 / (1 + torch.exp(-logits))) < DISC_FLOOR
    assert floor.sum() >= 2 and float(logits[floor].min()) > 12.0, "AMP rows on the 1e-4 floor of 1 - prob, far from its edge"
    assert (llc_actions.abs() == 1.0).any(), "clamped LLC actions"

    ds = {k: v.clone() for k, v in agent.dataset.values_dict.items() if k in ('advantages', 'returns', 'old_values')}
    out = dict(N=N, H=H, llc_steps=L, hlc_param_seed=synth.HRL_HLC_PARAM_SEED, llc_param_seed=synth.HRL_LLC_PARAM_SEED,
               rec={'normal': rec}, eb=eb, llc_actions=llc_actions, returns=batch_dict['returns'].clone(), dataset=ds,
               value_rms_after={'running_mean': agent.value_mean_std.running_mean.clone(), 'running_var': agent.value_mean_std.running_var.clone(),
                                'count': agent.value_mean_std.count.clone()},
               cfg={k: config[k] for k in ('gamma', 'tau', 'task_reward_w', 'disc_reward_w')}, llc_disc_reward_scale=float(llc._disc_reward_scale),
               hlc_sigma=float(sigma0[0]))
    out['synth_inputs'] = 'hrl_rollout_script'
    torch.save(out, os.path.join(OUT, 'rollout_hrl.pt'))
    print('rollout_hrl.pt', os.path.getsize(os.path.join(OUT, 'rollout_hrl.pt')), 'bytes;', 'out-of-range action components', int(out_of_range.sum()),
          'dones', int(dones_t.sum()), 'floor rows', int(floor.sum()), 'max logit', float(logits.max()))


if __name__ == '__main__':
    gen_hrl_rollout()
