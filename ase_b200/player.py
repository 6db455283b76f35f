"""Evaluation players: the `--test --checkpoint x.pth` half of ase/run.py (runner.player_factory, run.py:156-166).

    AMPPlayer  learning/amp_players.py:8-83 over learning/common_player.py:10-188   (AMPPlayerContinuous)
    ASEPlayer  learning/ase_players.py:9-152
    HRLPlayer  learning/hrl_players.py:18-260                                      (a task policy over a frozen ASE low-level controller)

Same config keys and rl_games BasePlayer defaults (config['player']: games_num 2000, determenistic True, n_game_life 1, print_stats True,
max_steps 27000), the same `restore(fn)` and the same printed lines as the reference's run().  The network runs through
`Learner.eval_actor_critic`; the latent writes, the action head and the episode bookkeeping are the mask-driven kernels of
csrc/player_kernels.cu.  The reference reads `done.nonzero()` and two `.item()` sums back every step; here the episode statistics stay on
the device and the host reads them once per window of `WINDOW` steps (every step when the batch is a single env, which ends its segment on
its first done, common_player.py:116).  Steps issued in a window after the run reached `games_num` episodes change no statistic, so the
printed lines and totals are the reference's.  Those steps still step the env (up to WINDOW - 1 times more than the reference) and, in
the ASE player, still run the latent countdown and the colour draws, so after run() the env and the global numpy state are ahead of where
the reference leaves them.

Differences from the reference that do not change results:
  * resets go through the env's mask-driven `reset_done(mask)` when it has one (else `reset(env_ids)`, the reference's order, which reads
    the done ids back);
  * headless runs skip `set_char_color` (it needs the ids on the host; there is nothing to colour without a viewer) but still take the three
    numpy uniforms `_change_char_color` draws, so the latent schedule follows the same numpy seed as the reference's;
  * the HRL player does not compute the env-0 discriminator reward of every LLC sub-step (hrl_players.py:184-194): the reference discards it;
  * run() returns its totals as a dict (the reference returns None)."""
import os

import numpy as np
import torch

from . import ops
from .agent import build_frozen_llc, net_params
from .learner import Learner

WINDOW = 32                 # player steps between two reads of the device statistics
_STATUS_BYTES = 32          # sizeof(AsePlayerStatus)


class AMPPlayer:
    kind = 'amp'
    _mu_activation = 'None'

    def __init__(self, config):
        self.config = config
        # rl_games 1.1.4 BasePlayer.__init__: the env from env_configurations unless one is handed over (config['vec_env'], as for the agents)
        self.env_name = config.get('env_name')
        self.env_config = config.get('env_config', {})
        self.env = config.get('vec_env')
        if self.env is None:
            from rl_games.common import env_configurations
            self.env = env_configurations.configurations[self.env_name]['env_creator'](**self.env_config)
        self.env_info = config.get('env_info') or self.env.get_env_info()
        self.value_size = self.env_info.get('value_size', 1)
        self.num_agents = self.env_info.get('agents', 1)
        assert self.value_size == 1 and self.num_agents == 1
        self.action_space = self.env_info['action_space']
        self.observation_space = self.env_info['observation_space']
        self.obs_shape = self.observation_space.shape
        self.player_config = config.get('player', {})
        pc = self.player_config
        self.device = torch.device(config.get('device', pc.get('device_name', 'cuda')))
        self.render_env = pc.get('render', False)
        self.games_num = pc.get('games_num', 2000)
        self.is_determenistic = pc.get('determenistic', True)
        self.n_game_life = pc.get('n_game_life', 1)
        self.print_stats = pc.get('print_stats', True)
        self.max_steps = pc.get('max_steps', 108000 // 4)
        self.normalize_input = config['normalize_input']
        assert self.normalize_input, "the engine implements the shipped configs (normalize_input True)"
        self._load_config_params(config)
        self.num_envs = self.env.task.num_envs
        self._setup_action_space()
        self.model = self._build_net(config)
        n, dev = self.num_envs, self.device
        self._rng = torch.tensor([int(config.get('seed', 0) or 0) * 1000003 + 4099, 0], dtype=torch.int64, device=dev)
        self._cr = torch.zeros(n, device=dev)
        self._steps = torch.zeros(n, device=dev)
        self._done_mask = torch.zeros(n, dtype=torch.uint8, device=dev)
        self._actions = torch.zeros(n, self.action_space.shape[0], device=dev)
        self._window = 1 if n // self.num_agents == 1 else WINDOW
        # AsePlayerStatus, then one {done count, reward sum, steps sum} record per step of the window: one buffer, one copy per window
        self._stat = torch.zeros(_STATUS_BYTES + 24 * self._window, dtype=torch.uint8, device=dev)
        self._records = self._stat[_STATUS_BYTES:].view(torch.float64).view(self._window, 3)
        self._host = torch.zeros(self._stat.shape, dtype=torch.uint8).pin_memory()
        self._scratch = torch.zeros(ops.lib.ase_player_scratch_bytes(n), dtype=torch.uint8, device=dev)
        self._event = torch.cuda.Event()
        self._inject = None        # tests: {'noise': [...], 'z': [...]} tables consumed in call order instead of the in-kernel draws

    # ------------------------------------------------------------------ construction
    def _load_config_params(self, config):
        self._normalize_amp_input = config.get('normalize_amp_input', True)
        self._disc_reward_scale = config['disc_reward_scale']

    def _setup_action_space(self):
        """common_player.py:184-188."""
        self.actions_num = self.action_space.shape[0]
        self.actions_low = torch.from_numpy(np.asarray(self.action_space.low).copy()).float().to(self.device)
        self.actions_high = torch.from_numpy(np.asarray(self.action_space.high).copy()).float().to(self.device)

    def _learner_kwargs(self, config):
        np_ = net_params(config)
        # (the learner needs a batch of at least 2 rows; eval_actor_critic takes any row count up to it)
        return dict(obs_dim=self.obs_shape[0], act_dim=self.actions_num, batch=max(2, self.num_envs), units=tuple(np_['mlp']['units']),
                    device=self.device, gemm_backend=config.get('gemm_backend', 2), sigma_init=np_['space']['continuous']['sigma_init'].get('val', 0.0),
                    mu_activation=self._mu_activation)

    def _build_net(self, config):
        kw = self._learner_kwargs(config)
        if self.kind != 'ppo':
            kw.update(amp_dim=self.env.amp_observation_space.shape[0], amp_batch=2, disc_units=tuple(net_params(config)['disc']['units']))
        ln = Learner(self.kind, **kw)
        ln.init_reference(seed=config.get('seed', 0) or 0)
        for r in (ln.running_mean_std, ln.value_mean_std, ln.amp_input_mean_std):
            if r is not None:
                r.eval()
        return ln

    def restore(self, fn):
        """rl_games BasePlayer.restore + amp_players.py:16-22: model, running_mean_std and (AMP / ASE) amp_input_mean_std of an rl_games
        checkpoint (the reference's own .pth files and those this package's agents save)."""
        if fn == 'Base':
            return
        w = torch.load(fn, map_location='cpu', weights_only=False)
        self.model.load_state_dict(w['model'])
        self.model.set_stats_weights(w)

    # ------------------------------------------------------------------ one player step
    def _draw(self, name):
        if self._inject is None:
            return None
        k = self._calls[name]
        self._calls[name] = k + 1
        return self._inject[name][k]

    def env_reset(self, full=False):
        """CommonPlayer.env_reset: every env at the start of a segment, else the envs that finished on the previous step."""
        if full:
            return self.env.reset()
        if hasattr(self.env, 'reset_done'):
            return self.env.reset_done(self._done_mask)
        return self.env.reset(self._done_mask.nonzero(as_tuple=False)[:, 0])        # the reference's order: reads the ids back

    def _latents(self):
        return None

    def get_action(self, obs):
        """ase_players.py:33-59 / PpoPlayerContinuous.get_action: head, Normal.sample unless deterministic, clamp, rescale_actions."""
        mu, _ = self.model.eval_actor_critic(obs, self._latents(), want_value=False)
        ops.player_act(mu, None if self.is_determenistic else self.model.sigma, self.actions_low, self.actions_high, self._rng, 0,
                       actions=self._actions, noise=None if self.is_determenistic else self._draw('noise'))
        return self._actions

    def _step(self, obs, slot):
        """One player step after the reset: action, env.step, bookkeeping into record `slot`.  Returns the env's next observation."""
        obs, r, done, info = self.env.step(self.get_action(obs))
        self._post_step(info)
        ops.player_post_step(r, done, 0, 1, None, None, self._cr, self._steps, self._done_mask, self._n_games, self._stat[:_STATUS_BYTES],
                             self._records[slot], self._scratch, self._rng)
        return obs

    def _post_step(self, info):
        """amp_players.py:33-37: the discriminator print runs only with a viewer."""
        if self.env.task.viewer:
            self._amp_debug(info)

    def _amp_debug(self, info):
        """amp_players.py:47-59 (env 0)."""
        logits, _ = self.model.eval_disc_enc(info['amp_obs'][0:1], want_enc=False)
        dr, _, _ = ops.amp_rewards(logits, None, None, self._disc_reward_scale)
        print("disc_pred: ", logits.cpu().numpy()[0, 0], dr.cpu().numpy()[0])

    # ------------------------------------------------------------------ run
    def _begin_run(self):
        pass

    def _read_window(self, w):
        """The window's one host read: status and the step records, through pinned memory."""
        self._host.copy_(self._stat, non_blocking=True)
        self._event.record()
        self._event.synchronize()
        a = self._host.numpy()
        totals = a[0:16].view(np.float64)
        games = int(a[16:24].view(np.int64)[0])
        stopped = bool(a[24:28].view(np.int32)[0])
        recs = a[_STATUS_BYTES:_STATUS_BYTES + 24 * w].view(np.float64).reshape(w, 3)
        return float(totals[0]), float(totals[1]), games, stopped, recs

    def run(self):
        """common_player.py:25-127 (hrl_players.py:63-167): segments of at most max_steps steps, each starting from a full env reset; a
        'reward: .. steps: ..' line per step with finished episodes, then the totals.  Returns {'games_played', 'sum_rewards', 'sum_steps',
        'av_reward', 'av_steps'}."""
        n_game_life = self.n_game_life
        n_games = self.games_num * n_game_life
        self._n_games = n_games
        self._calls = {'noise': 0, 'z': 0}
        self._stat.zero_()
        self._begin_run()
        sum_rewards, sum_steps, games_played, stopped = 0.0, 0.0, 0, False
        for _ in range(n_games):
            if stopped:
                break
            obs = self.env_reset(full=True)
            self._cr.zero_(); self._steps.zero_(); self._done_mask.zero_()
            n = 0
            while n < self.max_steps:
                w = min(self._window, self.max_steps - n)
                self._records[:w].zero_()
                for k in range(w):
                    obs = self.env_reset()
                    obs = self._step(obs, k)
                n += w
                sum_rewards, sum_steps, games_played, stopped, recs = self._read_window(w)
                finished = False
                for cnt, rs, ss in recs:
                    if cnt > 0:
                        finished = True
                        if self.print_stats:
                            print('reward:', float(rs) / int(cnt), 'steps:', float(ss) / int(cnt))
                if stopped or (finished and self._window == 1):
                    break
        print(sum_rewards)
        av_reward = sum_rewards / games_played * n_game_life
        av_steps = sum_steps / games_played * n_game_life
        print('av reward:', av_reward, 'av steps:', av_steps)
        return {'games_played': games_played, 'sum_rewards': sum_rewards, 'sum_steps': sum_steps, 'av_reward': av_reward, 'av_steps': av_steps}


class ASEPlayer(AMPPlayer):
    kind = 'ase'

    def _load_config_params(self, config):
        super()._load_config_params(config)
        self._latent_dim = config['latent_dim']
        self._latent_steps_min = config.get('latent_steps_min', np.inf)
        self._latent_steps_max = config.get('latent_steps_max', np.inf)
        self._enc_reward_scale = config['enc_reward_scale']

    def _learner_kwargs(self, config):
        kw = super()._learner_kwargs(config)
        kw.update(latent_dim=self._latent_dim)
        return kw

    def _build_net(self, config):
        ln = super()._build_net(config)
        self._ase_latents = torch.zeros(self.num_envs, self._latent_dim, device=self.device)
        return ln

    def _latents(self):
        return self._ase_latents

    def _begin_run(self):
        self._reset_latent_step_count()                   # ase_players.py:28-31

    def env_reset(self, full=False):
        """ase_players.py:61-64: the env reset, then _reset_latents of the same envs."""
        obs = super().env_reset(full)
        self._reset_latents(full, 4 if full else 2)
        return obs

    def _reset_latents(self, all_envs, stream_id):
        """ase_players.py:71-80: fresh latents for every env (all_envs) or the envs done on the previous step, then _change_char_color.
        The three callers draw from Philox streams of their own (a segment's full reset and its first step share the counter)."""
        ops.player_latents(self._ase_latents, self._done_mask, all_envs, self._rng, stream_id, z_in=self._draw('z'))
        self._change_char_color(None if all_envs else self._done_mask)

    def _update_latents(self):
        """ase_players.py:82-94: the global countdown is host numpy state, as in the reference."""
        if self._latent_step_count <= 0:
            self._reset_latents(True, 3)
            self._reset_latent_step_count()
            if self.env.task.viewer:
                print("Sampling new amp latents------------------------------")
                self._change_char_color(None)
        else:
            self._latent_step_count -= 1

    def _reset_latent_step_count(self):
        self._latent_step_count = np.random.randint(self._latent_steps_min, self._latent_steps_max)

    def _change_char_color(self, mask):
        """ase_players.py:143-152.  The three uniforms are drawn on every call, with or without a viewer; the colour is set only with one."""
        base_col = np.array([0.4, 0.4, 0.4])
        range_col = np.array([0.0706, 0.149, 0.2863])
        range_sum = np.linalg.norm(range_col)
        rand_col = np.random.uniform(0.0, 1.0, size=3)
        rand_col = range_sum * rand_col / np.linalg.norm(rand_col)
        rand_col += base_col
        if self.env.task.viewer:
            env_ids = torch.arange(self.num_envs, device=self.device) if mask is None else mask.nonzero(as_tuple=False)[:, 0]
            self.env.task.set_char_color(rand_col, env_ids)

    def get_action(self, obs):
        self._update_latents()
        return super().get_action(obs)

    def _amp_debug(self, info):
        """ase_players.py:127-141 (env 0)."""
        logits, enc = self.model.eval_disc_enc(info['amp_obs'][0:1])
        dr, er, _ = ops.amp_rewards(logits, enc, self._ase_latents[0:1], self._disc_reward_scale, self._enc_reward_scale)
        print("disc_pred: ", logits.cpu().numpy()[0, 0], dr.cpu().numpy()[0], er.cpu().numpy()[0])


class HRLPlayer(AMPPlayer):
    kind = 'ppo'
    _mu_activation = 'tanh'            # HRLBuilder.Network: the HLC's mu is tanh(mu) (hrl_network_builder.py:26-29)

    def __init__(self, config):
        llc_config = config.get('llc_config')
        if llc_config:                 # hrl_players.py:20-23: the LLC's train config, relative to the working directory
            import yaml
            with open(os.path.join(os.getcwd(), llc_config), 'r') as f:
                params = yaml.load(f, Loader=yaml.SafeLoader)['params']
            self._llc_net_params, self._latent_dim = params['network'], params['config']['latent_dim']
        else:
            self._llc_net_params, self._latent_dim = config['llc_net_params'], config['latent_dim']
        super().__init__(config)
        self._task_size = self.env.task.get_task_obs_size()
        self._llc_steps = config['llc_steps']
        llc_checkpoint = config['llc_checkpoint']
        assert llc_checkpoint != ""
        llc_cfg = {'llc_net_params': self._llc_net_params, 'llc_checkpoint': llc_checkpoint, 'gemm_backend': config.get('gemm_backend', 2)}
        self._llc = build_frozen_llc(llc_cfg, self.env_info, self.obs_shape[0] - self._task_size, self._latent_dim, max(2, self.num_envs), self.device)
        print("Loaded LLC checkpoint from {:s}".format(llc_checkpoint))
        n = self.num_envs
        self._z = torch.zeros(n, self._latent_dim, device=self.device)
        self._sub_rewards = torch.zeros(n, device=self.device)
        self._sub_dones = torch.zeros(n, device=self.device)

    def _load_config_params(self, config):
        pass

    def _setup_action_space(self):
        """hrl_players.py:238-241: the HLC acts in the LLC's latent space; the env's bounds rescale the LLC's actions."""
        super()._setup_action_space()
        self.actions_num = self._latent_dim

    def _post_step(self, info):
        pass

    def _step(self, obs, slot):
        """get_action (hrl_players.py:36-61) then env_step (:169-208): the clamped HLC action, L2-normalised, is the latent of llc_steps
        frozen-LLC sub-steps; the step's reward is their mean and it is done when any sub-step was."""
        mu, _ = self.model.eval_actor_critic(obs, None, want_value=False)
        ops.player_act(mu, None if self.is_determenistic else self.model.sigma, None, None, self._rng, 0, unit_out=self._z,
                       noise=None if self.is_determenistic else self._draw('noise'))
        for t in range(self._llc_steps):
            llc_obs = obs[..., :obs.shape[-1] - self._task_size]
            llc_mu, _ = self._llc.eval_actor_critic(llc_obs, self._z, want_value=False)
            ops.player_act(llc_mu, None, self.actions_low, self.actions_high, None, 0, actions=self._actions)
            obs, r, done, _ = self.env.step(self._actions)
            ops.player_post_step(r, done, t, self._llc_steps, self._sub_rewards, self._sub_dones, self._cr, self._steps, self._done_mask,
                                 self._n_games, self._stat[:_STATUS_BYTES], self._records[slot], self._scratch, self._rng)
        return obs
