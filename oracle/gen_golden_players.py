"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/player_{amp,ase,hrl}.pt by executing the UNMODIFIED reference players -- learning/
amp_players.AMPPlayerContinuous, ase_players.ASEPlayer and hrl_players.HRLPlayer (the checkout named by ASE_REFERENCE_ROOT, through
oracle/shims) -- as run.py's --test path does: construction from the shipped train config (network widths reduced), restore() of an rl_games
checkpoint, then run() over a scripted vec-env.  HRLPlayer reads the reference's own ase_humanoid_hrl.yaml as its llc_config (copied to a
temporary directory, widths reduced, CPU device) and restores its LLC from an rl_games checkpoint.  Recorded: the actions passed to every env
step (HRL: every LLC sub-step), the eps of every Normal.sample, the latent rows of every sample_latents call with the env ids they went to,
the numpy countdown values, and every line run() prints.  Usage: python oracle/gen_golden_players.py"""
import contextlib
import copy
import io
import os
import shutil
import sys
import tempfile

import numpy as np
import torch
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ase_oracle as O            # noqa: E402
import player_oracle as PO        # noqa: E402
import ref_harness as rh          # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), 'tests', 'golden')
D, AMP, A, Z, TASK, UNITS, LOW, HIGH = PO.D, PO.AMP, PO.A, PO.Z, PO.TASK, PO.UNITS, PO.LOW, PO.HIGH
params, rms, checkpoint = PO.params, PO.rms, PO.checkpoint
NP_SEED = 7


def _install_shims():
    """The reference players subclass rl_games.algos_torch.players.PpoPlayerContinuous and call players.rescale_actions."""
    rh._setup_path()
    from rl_games.algos_torch import players, ppo_player
    players.PpoPlayerContinuous = ppo_player.PpoPlayerContinuous
    players.rescale_actions = ppo_player.rescale_actions


def _net_params(params_):
    net = params_['network']
    net['mlp']['units'] = list(UNITS)
    if 'disc' in net:
        net['disc']['units'] = list(UNITS)
    net['space']['continuous']['sigma_init']['val'] = -1.0
    return net


class ScriptedEnv(rh.FakeVecEnv):
    def __init__(self, tb, n):
        super().__init__(n, obs_dim=D, amp_dim=AMP, act_dim=A)
        from gym import spaces
        self.env.action_space = spaces.Box(np.array(LOW), np.array(HIGH))
        self.env.task.set_char_color = lambda col, env_ids: None
        self.env.task.get_task_obs_size = lambda: TASK
        self.tb, self.T, self.actions = tb, tb['rew_t'].shape[0], []
        self.cur = tb['reset_obs_t'][0].clone()
        self.observation_space, self.action_space = self.env.observation_space, self.env.action_space
        self.amp_observation_space = self.env.amp_observation_space
        self.task = self.env.task

    def step(self, actions):
        t = self.t % self.T
        self.actions.append(actions.clone())
        self.t += 1
        self.cur = self.tb['obs_t'][t + 1].clone()
        return self.cur, self.tb['rew_t'][t].clone(), self.tb['dones_t'][t].clone(), {'amp_obs': self.tb['amp_t'][t].clone()}

    def reset(self, env_ids=None):
        if env_ids is None:
            self.cur = self.tb['reset_obs_t'][self.t % self.T].clone()
        elif len(env_ids) > 0:
            ids = torch.as_tensor(env_ids, dtype=torch.long).reshape(-1)
            self.cur[ids] = self.tb['reset_obs_t'][self.t % self.T][ids]
        return self.cur


def _make(kind, n, det, games, max_steps, tmp, env):
    from rl_games.common import env_configurations
    from learning import amp_models, amp_network_builder, amp_players, ase_models, ase_network_builder, ase_players
    from learning import hrl_models, hrl_network_builder, hrl_players
    env_configurations.register('scripted', {'env_creator': lambda **kw: env, 'vecenv_type': 'RLGPU'})
    yaml_name = {'amp': 'amp_humanoid.yaml', 'ase': 'ase_humanoid.yaml', 'hrl': 'hrl_humanoid.yaml'}[kind]
    params_ = copy.deepcopy(rh.load_train_cfg(yaml_name))['params']
    net = _net_params(params_)
    builder = {'amp': amp_network_builder.AMPBuilder, 'ase': ase_network_builder.ASEBuilder, 'hrl': hrl_network_builder.HRLBuilder}[kind]()
    builder.load(net)
    model = {'amp': amp_models.ModelAMPContinuous, 'ase': ase_models.ModelASEContinuous, 'hrl': hrl_models.ModelHRLContinuous}[kind](builder)
    config = params_['config']
    config.update(network=model, env_name='scripted', player={'device_name': 'cpu', 'games_num': games, 'determenistic': det})
    if kind == 'ase':
        config.update(latent_steps_min=1, latent_steps_max=4)
    if kind != 'hrl':
        cls = {'amp': amp_players.AMPPlayerContinuous, 'ase': ase_players.ASEPlayer}[kind]
        player = cls(config)
    else:
        # llc_config names ase/data/cfg/train/rlg/ase_humanoid_hrl.yaml relative to the working directory (hrl_players.py:20)
        llc_yaml = yaml.load(open(os.path.join(rh.REF_ROOT, config['llc_config'])), Loader=yaml.SafeLoader)
        _net_params(llc_yaml['params'])
        llc_yaml['params']['config']['player'] = {'device_name': 'cpu'}
        os.makedirs(os.path.join(tmp, os.path.dirname(config['llc_config'])), exist_ok=True)
        with open(os.path.join(tmp, config['llc_config']), 'w') as f:
            yaml.dump(llc_yaml, f)
        torch.save(checkpoint(params('llc', 31), rms(D - TASK, 32), rms(AMP, 33)), os.path.join(tmp, 'llc.pth'))
        config.update(llc_steps=3, llc_checkpoint='llc.pth')
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            player = hrl_players.HRLPlayer(config)
        finally:
            os.chdir(cwd)
    ck = os.path.join(tmp, kind + '.pth')
    torch.save(checkpoint(params(kind, 11), rms(D, 12), None if kind == 'hrl' else rms(AMP, 13)), ck)
    player.restore(ck)
    player.max_steps = max_steps
    return player


def gen_run(kind, n, det, games, max_steps, seed=5):
    _install_shims()
    tb = PO.tables(n, seed)
    env = ScriptedEnv(tb, n)
    tmp = tempfile.mkdtemp()
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            player = _make(kind, n, det, games, max_steps, tmp, env)
    finally:
        shutil.rmtree(tmp)
    g = torch.Generator().manual_seed(92 + n)
    rec = {'normal': [], 'latents': [], 'latent_ids': [], 'countdown': []}
    real_sample = torch.distributions.Normal.sample

    def rec_sample(self, sample_shape=torch.Size()):
        eps = torch.randn(self.loc.shape, generator=g)
        rec['normal'].append(eps.clone())
        return self.loc + self.scale * eps
    if kind == 'ase':
        net = player.model.a2c_network

        def sample_latents(k):
            z = torch.nn.functional.normalize(torch.randn(k, Z, generator=g), dim=-1)
            rec['latents'].append(z.clone())
            return z
        net.sample_latents = sample_latents
        real_reset, real_count = player._reset_latents, player._reset_latent_step_count

        def reset_latents(done_env_ids=None):
            rec['latent_ids'].append(None if done_env_ids is None else torch.as_tensor(done_env_ids, dtype=torch.long).reshape(-1).clone())
            return real_reset(done_env_ids)

        def reset_count():
            real_count()
            rec['countdown'].append(int(player._latent_step_count))
        player._reset_latents, player._reset_latent_step_count = reset_latents, reset_count
    buf = io.StringIO()
    torch.distributions.Normal.sample = rec_sample
    np.random.seed(NP_SEED)
    try:
        with contextlib.redirect_stdout(buf):
            player.run()
    finally:
        torch.distributions.Normal.sample = real_sample
    lines = [ln for ln in buf.getvalue().splitlines() if not ln.startswith('=>')]
    acts = torch.stack(env.actions).detach()
    # ---- edges
    steps_run = sum(1 for ln in lines if ln.startswith('reward:'))
    assert steps_run >= 1 and lines[-1].startswith('av reward:')
    if kind != 'hrl':
        low, high = torch.tensor(LOW), torch.tensor(HIGH)
        assert ((acts == low) | (acts == high)).any(), "head outputs beyond +-1 clamped onto the non-unit box"
    return {'kind': kind, 'N': n, 'determenistic': det, 'games_num': games, 'max_steps': max_steps, 'llc_steps': 3, 'task_size': TASK,
            'low': torch.tensor(LOW), 'high': torch.tensor(HIGH), 'units': UNITS, 'table_seed': seed, 'np_seed': NP_SEED, 'rec': rec,
            'actions': acts, 'lines': lines, 'env_steps': env.t}


def main():
    runs = {'amp': [gen_run('amp', 24, False, 40, 9), gen_run('amp', 24, True, 40, 9)],
            'ase': [gen_run('ase', 24, True, 40, 9), gen_run('ase', 24, False, 40, 9), gen_run('ase', 1, False, 3, 40)],
            'hrl': [gen_run('hrl', 24, False, 40, 3), gen_run('hrl', 24, True, 40, 3)]}
    # the edge cases the fixtures must hold
    ase = runs['ase'][0]
    resets_all = [i for i, ids in enumerate(ase['rec']['latent_ids']) if ids is None]
    assert any(i > 0 and ase['rec']['latent_ids'][i - 1] is not None and len(ase['rec']['latent_ids'][i - 1]) > 0 for i in resets_all), \
        "a global latent resample on a step where some envs also reset"
    for r in runs['amp'] + runs['ase'] + runs['hrl']:
        if r['N'] > 1:       # a segment ends early only when games_num is reached, so more player steps than max_steps means a restart
            assert r['env_steps'] // (r['llc_steps'] if r['kind'] == 'hrl' else 1) > r['max_steps'], \
                ("max_steps small enough that the outer loop restarts a segment", r['kind'], r['env_steps'])
    assert any(ln.startswith('reward:') and float(ln.split()[3]) > 0 for ln in runs['ase'][2]['lines'])
    for kind, rs in runs.items():
        torch.save(rs, os.path.join(OUT, f'player_{kind}.pt'))
        print(f'player_{kind}.pt', os.path.getsize(os.path.join(OUT, f'player_{kind}.pt')), 'bytes;',
              [(r['N'], r['determenistic'], len(r['lines']), r['env_steps']) for r in rs])


if __name__ == '__main__':
    main()
