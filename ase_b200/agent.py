"""Host-side mirror of the reference's rl_games agents for the training hot path:

    CommonAgent  learning/common_agent.py:25-564   (plain PPO; HRL high-level policy learner)
    AMPAgent     learning/amp_agent.py:21-628
    ASEAgent     learning/ase_agent.py:12-538
    HRLAgent     learning/hrl_agent.py:24-268      (task training over a frozen ASE low-level controller)

Same public surface (`play_steps`, `prepare_dataset`, `train_actor_critic` / `calc_gradients`, `train_epoch`,
`train`, `get_full_state_weights` / `set_full_state_weights`, `train_result` keys) and the same config keys
(data/cfg/train/rlg/*.yaml), so `run.py`'s `algo_factory.register_builder('ase', lambda **kw: ASEAgent(**kw))`
works unchanged (INTEGRATION.md).  All arithmetic runs in libase_b200.so through `Learner` / `ops`; torch is
used for device buffers, indexing (gathers, ring buffers), RNG draws and torch.distributed.

Differences from the reference that do not change results:
  * no per-minibatch `.item()`: train_result scalars stay on the device (lr_schedule is `constant`);
  * demo / replay AMP observations are gathered per minibatch (amp_minibatch_size rows) through composed
    indices instead of materialising two [batch, 1400] copies per epoch (same rows, same order);
  * the diversity loss' second actor pass is batched with the first (2B rows)."""
import math
import os
import time

import numpy as np
import torch

from . import ops
from .learner import Learner
from .replay_buffer import ReplayBuffer


def swap_and_flatten01(x):
    """rl_games a2c_common.swap_and_flatten01: env-major flatten, row = env * H + t."""
    s = x.shape
    return x.transpose(0, 1).reshape(s[0] * s[1], *s[2:])


class AMPDataset:
    """learning/amp_datasets.py:4-31: one global permutation, contiguous slices, reshuffle when exhausted."""

    def __init__(self, batch_size, minibatch_size, device):
        self.batch_size, self.minibatch_size, self.device = batch_size, minibatch_size, device
        self.length = batch_size // minibatch_size
        self._idx_buf = torch.randperm(batch_size, device=device)
        self.values_dict = {}

    def __len__(self):
        return self.length

    def update_values_dict(self, d):
        self.values_dict = d

    def sample_indices(self, idx):
        start, end = idx * self.minibatch_size, (idx + 1) * self.minibatch_size
        sample_idx = self._idx_buf[start:end].clone()
        if end >= self.batch_size:
            self._idx_buf[:] = torch.randperm(self.batch_size, device=self.device)
        return sample_idx


class CommonAgent:
    kind = 'ppo'

    def __init__(self, base_name, config):
        self.config = config
        self.name = base_name
        self.ppo_device = torch.device(config.get('device', 'cuda:0'))
        self.vec_env = config.get('vec_env')
        if self.vec_env is None:     # drop-in path: rl_games creates the env exactly as A2CBase does
            from rl_games.common import vecenv
            self.vec_env = vecenv.create_vec_env(config['env_name'], config['num_actors'], **config.get('env_config', {}))
        self.env_info = config.get('env_info') or self.vec_env.get_env_info()
        self.num_actors = config['num_actors']
        self.num_agents = self.env_info.get('agents', 1)
        self.value_size = self.env_info.get('value_size', 1)
        assert self.value_size == 1 and self.num_agents == 1
        self.obs_shape = self.env_info['observation_space'].shape
        self.actions_num = self.env_info['action_space'].shape[0]
        self.horizon_length = config['horizon_length']
        self.batch_size = self.horizon_length * self.num_actors
        self.batch_size_envs = self.batch_size
        self.minibatch_size = config['minibatch_size']
        self.mini_epochs_num = config['mini_epochs']
        assert self.batch_size % self.minibatch_size == 0
        self.normalize_input = config['normalize_input']
        self.normalize_value = config.get('normalize_value', False)
        self.normalize_advantage = config['normalize_advantage']
        assert self.normalize_input and self.normalize_value and self.normalize_advantage, "the engine implements the shipped configs (normalize_* True)"
        self.gamma, self.tau = config['gamma'], config['tau']
        self.e_clip = config['e_clip']
        assert not config.get('clip_value', False) and not config.get('truncate_grads', False), "clip_value/truncate_grads are False in every shipped config"
        self.last_lr = float(config['learning_rate'])
        assert config.get('lr_schedule', 'constant') in ('constant', None)
        self.max_epochs = config.get('max_epochs', 1e6)
        self.save_freq = config.get('save_frequency', 0)
        self._save_intermediate = config.get('save_intermediate', False)
        # rl_games A2CBase: <train_dir>/<experiment name>/nn/<config name>.pth (common_agent.py:92)
        self.train_dir = config.get('train_dir', 'runs')
        self.experiment_name = config.get('full_experiment_name') or (config.get('name', base_name) + time.strftime('_%d-%H-%M-%S'))
        self.nn_dir = os.path.join(self.train_dir, self.experiment_name, 'nn')
        self.print_stats = config.get('print_stats', True)
        self.writer = config.get('writer', None)          # optional tensorboardX-like object with add_scalar(tag, value, step)
        # run.py hands its RLGPUAlgoObserver over as config['features']['observer'] (rl_games A2CBase): after_init / after_print_stats are
        # honoured; process_infos(infos, done_indices) only by the reference-order rollout (the device rollout keeps no index lists)
        self.algo_observer = (config.get('features') or {}).get('observer')
        self.mean_rewards = None
        self.clip_actions = config.get('clip_actions', True)
        self.multi_gpu = config.get('multi_gpu', False)
        self.rank, self.rank_size = 0, 1
        if self.multi_gpu:
            import torch.distributed as dist
            self.rank, self.rank_size = dist.get_rank(), dist.get_world_size()
            if self.ppo_device.type == 'cuda':
                from .dist_utils import init_comm
                init_comm()            # the library's own NCCL communicator: the per-minibatch allreduce goes through the C ABI
        self._load_config_params(config)
        self.model = self._build_learner(config)
        self.peer_adam = False
        if self.multi_gpu and self.ppo_device.type == 'cuda' and config.get('peer_adam', True):
            from .dist_utils import init_peer
            self.peer_adam = init_peer(self.model)      # gradient sum + Adam as one kernel over NVLink peer memory (falls back to NCCL)
        self.dataset = AMPDataset(self.batch_size, self.minibatch_size, self.ppo_device)
        self.epoch_num = 0
        self.frame = 0
        self.train_result = None
        self.rnn_states = None
        self.is_rnn = False
        self.has_central_value = False
        self._eval_mode = False
        self._timing = {}
        # rollout flavour: 'device_rollout' (default True) uses the mask-driven zero-sync step when the env offers reset_done();
        # 'rollout_graph' (default True) additionally captures the whole rollout in one CUDA graph
        self._device_rollout = bool(config.get('device_rollout', True))
        self._rollout_graph_enabled = bool(config.get('rollout_graph', True))
        # 'minibatch_graph' (default True): from the third epoch on, gather + calc_gradients of a minibatch are one CUDA graph launch
        self._mb_graph_enabled = bool(config.get('minibatch_graph', True))
        self._graphs_on = True
        if self.algo_observer is not None and hasattr(self.algo_observer, 'after_init'):
            self.algo_observer.after_init(self)       # rl_games A2CBase.__init__

    # ------------------------------------------------------------------ construction helpers
    def _load_config_params(self, config):
        pass

    def _net_params(self, config):
        """YAML `network` section: from rl_games' model builder when dropped into run.py, else config['net_params']."""
        net = config.get('network')
        if net is not None and hasattr(net, 'network_builder'):
            return net.network_builder.params
        return config['net_params']

    def _learner_kwargs(self, config):
        np_ = self._net_params(config)
        hp = {k: config[k] for k in ('e_clip', 'critic_coef', 'entropy_coef', 'bounds_loss_coef', 'learning_rate') if k in config}
        sigma = np_['space']['continuous']['sigma_init'].get('val', 0.0)
        return dict(obs_dim=self.obs_shape[0], act_dim=self.actions_num, batch=self.minibatch_size, units=tuple(np_['mlp']['units']),
                    hparams=hp, device=self.ppo_device, gemm_backend=config.get('gemm_backend', 2), sigma_init=sigma,
                    mu_activation=getattr(self, '_mu_activation', 'None'))

    def _build_learner(self, config):
        kw = self._learner_kwargs(config)
        ln = Learner(self.kind, **kw)
        ln.init_reference(seed=config.get('seed', 0) or 0)
        return ln

    # ------------------------------------------------------------------ rl_games-style state
    def set_eval(self):
        self._eval_mode = True
        for r in self._rms_modules():
            r.eval()

    def set_train(self):
        self._eval_mode = False
        for r in self._rms_modules():
            r.train()

    def _rms_modules(self):
        m = [self.model.running_mean_std, self.model.value_mean_std]
        if self.model.amp_input_mean_std is not None:
            m.append(self.model.amp_input_mean_std)
        return m

    @property
    def running_mean_std(self): return self.model.running_mean_std
    @property
    def value_mean_std(self): return self.model.value_mean_std

    def get_stats_weights(self):
        return self.model.get_stats_weights()

    def get_full_state_weights(self):
        """rl_games A2CBase.get_full_state_weights: the on-disk contract (SURVEY.md Appendix B)."""
        st = self.get_stats_weights()
        st['model'] = self.model.state_dict()
        st['epoch'] = self.epoch_num
        st['optimizer'] = self._optimizer_state_dict()
        st['frame'] = self.frame
        st['last_mean_rewards'] = -100500
        st['env_state'] = self.vec_env.get_env_state() if hasattr(self.vec_env, 'get_env_state') else None      # a2c_common.get_full_state_weights
        return st

    def set_full_state_weights(self, w):
        """common_agent.py:157-170."""
        self.model.load_state_dict(w['model'])
        self.model.set_stats_weights(w)
        self.epoch_num = w.get('epoch', 0)
        self.frame = w.get('frame', 0)
        self.last_mean_rewards = w.get('last_mean_rewards', -100500)
        if 'optimizer' in w:
            self._load_optimizer_state_dict(w['optimizer'])
        self.model.params_changed()
        if hasattr(self.vec_env, 'set_env_state'):
            self.vec_env.set_env_state(w.get('env_state', None))

    def save(self, fn):
        """rl_games A2CBase.save -> torch_ext.save_checkpoint(fn, get_full_state_weights()): writes fn + '.pth' (common_agent.py:141-150)."""
        d = os.path.dirname(fn)
        if d:
            os.makedirs(d, exist_ok=True)
        state = self.get_full_state_weights()
        state = {k: ({kk: (vv.detach().cpu().clone() if torch.is_tensor(vv) else vv) for kk, vv in v.items()} if isinstance(v, dict) and k != 'optimizer' else v)
                 for k, v in state.items()}
        state['optimizer']['state'] = {i: {kk: (vv.cpu() if torch.is_tensor(vv) else vv) for kk, vv in st.items()} for i, st in state['optimizer']['state'].items()}
        torch.save(state, fn + '.pth')
        return fn + '.pth'

    def restore(self, fn):
        """rl_games A2CBase.restore -> set_full_state_weights(torch_ext.load_checkpoint(fn)): what run.py / the Runner call for --checkpoint
        and what HRLAgent does with the LLC checkpoint (hrl_agent.py:202-213).  Accepts the reference's own .pth files."""
        w = torch.load(fn, map_location='cpu', weights_only=False)
        self.set_full_state_weights(w)

    def _optimizer_state_dict(self):
        """torch.optim.Adam.state_dict() layout: param index 0 is the frozen sigma (no state), 1.. follow parameters()."""
        state = {}
        names = list(self.model.named_parameters().keys())
        for i, k in enumerate(names):
            v = self.model.named_parameters()[k]
            off = v.storage_offset()
            sl = slice(off, off + v.numel())
            state[i + 1] = {'step': self.model.step, 'exp_avg': self.model.exp_avg[sl].view(v.shape).clone(),
                            'exp_avg_sq': self.model.exp_avg_sq[sl].view(v.shape).clone()}
        hp = self.model.hp
        return {'state': state, 'param_groups': [{'lr': self.last_lr, 'betas': (hp['beta1'], hp['beta2']), 'eps': hp['adam_eps'],
                                                  'weight_decay': 0.0, 'amsgrad': False, 'params': list(range(len(names) + 1))}]}

    def _load_optimizer_state_dict(self, sd):
        names = list(self.model.named_parameters().keys())
        step = 0
        for i, k in enumerate(names):
            s = sd['state'].get(i + 1)
            if s is None:
                continue
            v = self.model.named_parameters()[k]
            off = v.storage_offset()
            self.model.exp_avg[off:off + v.numel()].copy_(s['exp_avg'].reshape(-1))
            self.model.exp_avg_sq[off:off + v.numel()].copy_(s['exp_avg_sq'].reshape(-1))
            step = int(s['step'])
        self.model.step = step

    # ------------------------------------------------------------------ buffers
    def init_tensors(self):
        H, N, dev = self.horizon_length, self.num_actors, self.ppo_device
        f = lambda *s: torch.zeros((H, N) + s, device=dev, dtype=torch.float32)
        obs = self.obs_shape[0]
        self.experience_buffer = {
            'obses': f(obs), 'next_obses': f(obs), 'rewards': f(1), 'values': f(1), 'next_values': f(1), 'neglogpacs': f(),
            'dones': torch.zeros(H, N, device=dev, dtype=torch.uint8), 'actions': f(self.actions_num), 'mus': f(self.actions_num),
            'sigmas': f(self.actions_num)}
        self.update_list = ['actions', 'neglogpacs', 'values', 'mus', 'sigmas']
        self.tensor_list = self.update_list + ['obses', 'dones', 'next_obses']
        self.current_rewards = torch.zeros(N, 1, device=dev)
        self.current_lengths = torch.zeros(N, device=dev)
        self.dones = torch.ones(N, dtype=torch.uint8, device=dev)
        self._no_dones = torch.zeros(N, dtype=torch.uint8, device=dev)
        self._episode_meter = torch.zeros(3, device=dev)       # finished episodes: sum of rewards, sum of lengths, count (game_rewards / game_lengths)
        # device RNG state of the rollout kernels: {seed, call counter}
        self._rng = torch.tensor([int(self.config.get('seed', 0) or 0) * 1000003 + 12345 + self.rank, 0], dtype=torch.int64, device=dev)
        self._rollout_graph, self._rollout_warm = None, 0

    def env_reset(self, env_ids=None):
        obs = self.vec_env.reset(env_ids)
        return {'obs': obs}

    def env_step(self, actions):
        if self.clip_actions:
            actions = torch.clamp(actions, -1.0, 1.0)     # rescale_actions is the identity for +-1 bounds (vec_task.py:22)
        obs, rewards, dones, infos = self.vec_env.step(actions)
        return {'obs': obs}, rewards.unsqueeze(1), dones, infos

    # ------------------------------------------------------------------ rollout (learning/common_agent.py:244-307)
    def _latents(self):
        return None

    def _pre_action(self):
        pass

    def _rand_action_probs_tensor(self):
        return None

    # RNG hooks of the reference-order rollout (tests inject the reference's own draws here)
    def _draw_normal(self, shape):
        return torch.randn(shape, device=self.ppo_device, dtype=torch.float32)

    def _draw_bernoulli(self, probs):
        return torch.bernoulli(probs)

    def get_action_values(self, obs_dict, latents=None, rand_action_probs=None):
        """ase_agent.py:117-148 / amp_agent.py:139-169 (eval mode): actor+critic forward, sample, eps-greedy mask."""
        mu, v = self.model.eval_actor_critic(obs_dict['obs'], latents)
        noise = self._draw_normal(mu.shape)
        mask = None if rand_action_probs is None else self._draw_bernoulli(rand_action_probs)
        actions, nlp, sig = ops.policy_sample(mu, self.model.sigma, noise, mask)
        values = self.model.value_mean_std(v, unnorm=True)
        res = {'actions': actions, 'neglogpacs': nlp, 'values': values, 'mus': mu, 'sigmas': sig}
        if mask is not None:
            res['rand_action_mask'] = mask
        return res

    def _eval_critic(self, obs_dict, latents=None):
        _, v = self.model.eval_actor_critic(obs_dict['obs'], latents, want_value=True, want_actor=False)
        return self.model.value_mean_std(v, unnorm=True)

    def _extra_buffer_writes(self, n, res_dict, infos):
        pass

    def play_steps(self):
        """common_agent.py:244-307 / amp_agent.py:61-137 / ase_agent.py:36-115.  Two implementations of the same step sequence:
        the DEVICE rollout (no host sync: masks instead of nonzero() index lists, in-kernel Philox draws, optionally one CUDA graph for
        the whole rollout) when the env offers a mask-driven reset (`reset_done`), else the reference-order rollout (index lists, eager
        torch draws) that any rl_games vec-env works with."""
        self.set_eval()
        if self._device_rollout and hasattr(self.vec_env, 'reset_done'):
            self._play_steps_device()
        else:
            self._play_steps_reference()
        eb = self.experience_buffer
        mb_rewards, extra = self._final_rewards()
        mb_advs = ops.discount_values(eb['dones'], eb['values'], mb_rewards, eb['next_values'], self.gamma, self.tau)
        mb_returns = mb_advs + eb['values']
        batch_dict = {k: swap_and_flatten01(eb[k]) for k in self.tensor_list}
        batch_dict['returns'] = swap_and_flatten01(mb_returns)
        batch_dict['played_frames'] = self.batch_size
        for k, v in extra.items():
            batch_dict[k] = swap_and_flatten01(v)
        return batch_dict

    def _play_steps_reference(self):
        eb = self.experience_buffer
        # amp_agent.py:64 / ase_agent.py:40 `done_indices = []`: the first step of a rollout resets NOTHING (vec_env.reset(None) would
        # reset every env, humanoid.py:125-128, and ASEAgent.env_reset(None) every latent)
        done_indices = torch.empty(0, dtype=torch.long, device=self.ppo_device)
        for n in range(self.horizon_length):
            self.obs = self.env_reset(done_indices)
            eb['obses'][n] = self.obs['obs']
            self._pre_action()
            res = self.get_action_values(self.obs, self._latents(), self._rand_action_probs_tensor())
            for k in self.update_list:
                eb[k][n] = res[k]
            self.obs, rewards, self.dones, infos = self.env_step(res['actions'])
            eb['rewards'][n] = rewards
            eb['next_obses'][n] = self.obs['obs']
            eb['dones'][n] = self.dones
            self._extra_buffer_writes(n, res, infos)
            terminated = infos['terminate'].float().unsqueeze(-1)
            next_vals = self._eval_critic(self.obs, self._latents())
            next_vals = next_vals * (1.0 - terminated)
            eb['next_values'][n] = next_vals
            self.current_rewards += rewards
            self.current_lengths += 1
            done_indices = self.dones.nonzero(as_tuple=False)[:, 0]      # (host sync, as in the reference: ase_agent.py:78-79)
            self._episode_meter[0] += self.current_rewards[done_indices].sum(); self._episode_meter[1] += self.current_lengths[done_indices].sum()
            self._episode_meter[2] += done_indices.numel()
            if self.algo_observer is not None and hasattr(self.algo_observer, 'process_infos'):
                self.algo_observer.process_infos(infos, done_indices)          # amp_agent.py:107 / ase_agent.py:84
            not_dones = 1.0 - self.dones.float()
            self.current_rewards = self.current_rewards * not_dones.unsqueeze(1)
            self.current_lengths = self.current_lengths * not_dones

    # ------------------------------------------------------------------ device rollout
    def _device_latent_step(self, done_mask, n):
        pass

    def _rollout_loop(self):
        """One rollout as a fixed sequence of device work: nothing here reads a device value on the host."""
        eb, N = self.experience_buffer, self.num_actors
        logstd, vrms = self.model.sigma, self.model.value_mean_std
        probs = self._rand_action_probs_tensor()
        mask_out = eb.get('rand_action_mask')
        done_mask = self._no_dones
        inj = getattr(self, '_inject', None)           # tests: per-env draw tables [H, N, ...] instead of the in-kernel generator
        for n in range(self.horizon_length):
            obs = self.vec_env.reset_done(done_mask)                   # step 0 resets nothing (done_indices = [] in the reference)
            self.obs = {'obs': obs}
            eb['obses'][n].copy_(obs)
            self._device_latent_step(done_mask, n)
            lat = self._latents()
            mu, v = self.model.eval_actor_critic(obs, lat)
            eb['mus'][n].copy_(mu)
            ops.policy_sample_rng(mu, logstd, probs, self._rng, 0, eb['actions'][n], eb['neglogpacs'][n], eb['sigmas'][n],
                                  None if mask_out is None else mask_out[n], noise=None if inj is None else inj['noise'][n],
                                  mask=None if (inj is None or probs is None) else inj['mask'][n])
            vrms(v, unnorm=True, out=eb['values'][n])
            self.obs, rewards, self.dones, infos = self.env_step(eb['actions'][n])
            eb['rewards'][n].copy_(rewards)
            eb['next_obses'][n].copy_(self.obs['obs'])
            eb['dones'][n].copy_(self.dones)
            self._extra_buffer_writes_device(n, infos)
            _, vn = self.model.eval_actor_critic(self.obs['obs'], self._latents(), want_value=True, want_actor=False)
            ops.rollout_post_step(rewards, eb['dones'][n], infos['terminate'], vn, vrms, eb['next_values'][n], self.current_rewards,
                                  self.current_lengths, self._episode_meter, self._rng)
            done_mask = eb['dones'][n]

    def _extra_buffer_writes_device(self, n, infos):
        pass

    def _play_steps_device(self):
        if not (self._rollout_graph_enabled and self._graphs_on):
            self._rollout_loop()
            return
        if self._rollout_graph is None:
            if self._rollout_warm < 2:             # the learner calibrates its FP16 plane scales on its first calls: capture a settled schedule
                self._rollout_warm += 1
                self._rollout_loop()
                return
            g = torch.cuda.CUDAGraph()
            try:
                with torch.cuda.graph(g):
                    self._rollout_loop()
            except Exception as ex:     # a vec-env whose step cannot be captured: keep the eager device rollout
                import sys
                sys.stderr.write(f"ase_b200: CUDA-graph capture of the rollout failed ({type(ex).__name__}: {ex}); running it eagerly\n")
                self._rollout_graph_enabled = False
                torch.cuda.synchronize()
                self._rollout_loop()
                return
            self._rollout_graph = g
            g.replay()                              # capture does not execute
            return
        self._rollout_graph.replay()
        if hasattr(self.vec_env, 'on_graph_replay'):
            self.vec_env.on_graph_replay(self.horizon_length)

    def _final_rewards(self):
        return self.experience_buffer['rewards'], {}

    def discount_values(self, mb_fdones, mb_values, mb_rewards, mb_next_values):
        return ops.discount_values(mb_fdones.to(torch.uint8), mb_values, mb_rewards, mb_next_values, self.gamma, self.tau)

    # ------------------------------------------------------------------ dataset (common_agent.py:309-351)
    def _calc_advs(self, batch_dict):
        return ops.calc_advs(batch_dict['returns'], batch_dict['values'], None)

    def prepare_dataset(self, batch_dict):
        advantages = self._calc_advs(batch_dict)
        values = self.model.value_mean_std(batch_dict['values'])        # train mode: two sequential updates
        returns = self.model.value_mean_std(batch_dict['returns'])
        d = {'old_values': values, 'old_logp_actions': batch_dict['neglogpacs'], 'advantages': advantages, 'returns': returns,
             'actions': batch_dict['actions'], 'obs': batch_dict['obses'], 'mu': batch_dict['mus'], 'sigma': batch_dict['sigmas']}
        self.dataset.update_values_dict(d)

    def _gather(self, pairs):
        """pairs: [(key, source tensor [n, ...], int64 row indices)] -> {key: rows}; fp32 contiguous sources go through ONE fused
        ase_gather_rows launch into per-key staging buffers (AMPDataset._get_item issues one indexing kernel per tensor)."""
        bufs = self.__dict__.setdefault('_mb_bufs', {})
        out, items = {}, []
        for k, v, idx in pairs:
            if v.dtype != torch.float32 or not v.is_contiguous() or not v.is_cuda:
                out[k] = v[idx]
                continue
            shape = (idx.shape[0],) + tuple(v.shape[1:])
            dst = bufs.get(k)
            if dst is None or tuple(dst.shape) != shape:
                dst = bufs[k] = torch.empty(shape, dtype=torch.float32, device=v.device)
            items.append((v, dst, idx))
            out[k] = dst
        if items:
            ops.gather_rows(items)
        return out

    def _minibatch_pairs(self, i):
        """[(key, source tensor, int64 row indices)] of minibatch i, and {alias key: key} for tensors that are the same rows twice."""
        idx = self.dataset.sample_indices(i)
        return [(k, v, idx) for k, v in self.dataset.values_dict.items() if v is not None], {}

    def _minibatch(self, i):
        pairs, alias = self._minibatch_pairs(i)
        mb = self._gather(pairs)
        for k, src in alias.items():
            mb[k] = mb[src]
        return mb, pairs[0][2]

    # ------------------------------------------------------------------ one minibatch update = one CUDA graph launch
    def set_graphs(self, enabled):
        """Switch the captured CUDA graphs (rollout, minibatch update) on / off; captured graphs are kept.  bench.py turns them off for the one
        epoch it instruments per launch."""
        self._graphs_on = bool(enabled)

    def _static_dataset(self):
        """The epoch's dataset tensors are fresh allocations every epoch; the captured gather needs stable addresses: copy them into
        persistent buffers (~1 GB per epoch at config-3 sizes, 0.3 ms)."""
        store = self.__dict__.setdefault('_ds_static', {})

        def pin(k, v):
            b = store.get(k)
            if b is None or b.shape != v.shape or b.dtype != v.dtype:
                b = store[k] = torch.empty(v.shape, dtype=v.dtype, device=v.device)
            b.copy_(v)
            return b
        vd = self.dataset.values_dict
        for k, v in list(vd.items()):
            if v is not None and v.is_cuda:
                vd[k] = pin(k, v)
        if getattr(self, '_amp_obs_flat', None) is not None:
            self._amp_obs_flat = pin('__amp_obs_flat', self._amp_obs_flat)

    def _train_minibatch(self, i):
        use_graph = self._mb_graph_enabled and self._graphs_on and self.ppo_device.type == 'cuda' and self.epoch_num >= 3
        if not use_graph:
            mb, _ = self._minibatch(i)
            self.train_actor_critic(mb)
            return
        pairs, alias = self._minibatch_pairs(i)
        sig = tuple((k, v.data_ptr(), tuple(v.shape), idx.shape[0]) for k, v, idx in pairs) + tuple(sorted(alias.items()))
        st = self.__dict__.get('_mb_graph_state')
        if st is None or st['sig'] != sig:
            if st is not None and st.get('recaptures', 0) >= 3:        # sources keep moving (an env that reallocates): stay eager
                mb, _ = self._minibatch(i)
                self.train_actor_critic(mb)
                return
            st = self._capture_minibatch(pairs, alias, sig, (st or {}).get('recaptures', -1) + 1)
        # feed the static index / latent buffers, replay, finish (allreduce + Adam + train_result row) eagerly
        seen = {}
        for (k, v, idx), sidx in zip(pairs, st['idx']):
            if id(idx) not in seen:
                sidx.copy_(idx); seen[id(idx)] = True
        nz = self._new_latents(self.minibatch_size)
        if nz is not None:
            st['newz'].copy_(nz)
        st['graph'].replay()
        self._finish_update(st['out'])

    def _capture_minibatch(self, pairs, alias, sig, recaptures):
        by_idx, sidx_list, items, mb = {}, [], [], {}
        bufs = self.__dict__.setdefault('_mb_bufs', {})
        for k, v, idx in pairs:
            assert v.dtype == torch.float32 and v.is_contiguous() and v.is_cuda, k
            sidx = by_idx.get(id(idx))
            if sidx is None:
                sidx = by_idx[id(idx)] = idx.clone()
            sidx_list.append(sidx)
            shape = (idx.shape[0],) + tuple(v.shape[1:])
            dst = bufs.get(k)
            if dst is None or tuple(dst.shape) != shape:
                dst = bufs[k] = torch.empty(shape, dtype=torch.float32, device=v.device)
            items.append((v, dst, sidx))
            mb[k] = dst
        for k, src in alias.items():
            mb[k] = mb[src]
        nz = self._new_latents(self.minibatch_size)
        newz = None if nz is None else nz.clone()
        self.set_train()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ops.gather_rows(items)
            out = self.model.calc_gradients(mb, newz, update_rms=True)
        st = {'sig': sig, 'graph': g, 'idx': sidx_list, 'newz': newz, 'out': out, 'recaptures': recaptures}
        self._mb_graph_state = st
        return st

    # ------------------------------------------------------------------ update (common_agent.py:353-435)
    def _new_latents(self, n):
        return None

    def calc_gradients(self, input_dict):
        self.set_train()
        out = self.model.calc_gradients(input_dict, self._new_latents(input_dict['obs'].shape[0]), update_rms=True)
        self._finish_update(out)

    def _finish_update(self, out):
        """Gradient averaging over ranks (one allreduce through the C ABI), Adam, and the train_result row of this minibatch."""
        scale = 1.0
        if self.multi_gpu:
            from .dist_utils import allreduce_grads
            scale = allreduce_grads(self.model.grads)       # one flat NCCL sum per minibatch (Horovod averaged: amp_agent.py:357-363)
        self.model.adam_step(grad_scale=scale)
        row = self._tr_buf[self._tr_i % self._tr_buf.shape[0]]
        row[:out['scalars'].shape[0]].copy_(out['scalars'])
        self._tr_i += 1
        from .lib import TR_NAMES
        tr = {name: row[j] for j, name in enumerate(TR_NAMES)}
        tr['last_lr'] = self.last_lr
        tr['lr_mul'] = 1.0
        if 'disc_agent_logit' in out:
            tr['disc_agent_logit'] = out['disc_agent_logit']
            tr['disc_demo_logit'] = out['disc_demo_logit']
        self.train_result = tr

    def train_actor_critic(self, input_dict):
        self.calc_gradients(input_dict)
        return self.train_result

    def _pre_update(self, batch_dict):
        pass

    def _post_update(self, batch_dict):
        pass

    def train_epoch(self):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        with torch.no_grad():
            batch_dict = self.play_steps()
        ev[1].record()
        self._pre_update(batch_dict)
        self.set_train()
        self.curr_frames = batch_dict.pop('played_frames')
        self.prepare_dataset(batch_dict)
        nmb = self.mini_epochs_num * len(self.dataset)
        if getattr(self, '_tr_buf', None) is None or self._tr_buf.shape[0] != nmb:
            from .lib import TR_COUNT
            # + the learner's status word + the epoch's episode meter (sum of finished episodes' rewards, of their lengths, their count)
            self._tr_buf = torch.zeros(nmb, TR_COUNT + 4, device=self.ppo_device)
        self._tr_i = 0
        if self._mb_graph_enabled and self._graphs_on and self.ppo_device.type == 'cuda' and self.epoch_num >= 3:
            self._static_dataset()
        for _ in range(self.mini_epochs_num):
            for i in range(len(self.dataset)):
                self._train_minibatch(i)
        self._post_update(batch_dict)
        from .lib import TR_COUNT
        self.model.plane_flag_to(self._tr_buf[:, TR_COUNT])
        # game_rewards / game_lengths of the reference (amp_agent.py:102-105), per epoch instead of over a 100-game window: the meter rides in
        # the epoch's record (every row carries the same three numbers, so the record's row mean is the value) and starts again from zero
        self._tr_buf[:, TR_COUNT + 1:TR_COUNT + 4] = self._episode_meter
        self._episode_meter.zero_()
        ev[2].record()
        self._events = ev
        from .lib import TR_NAMES
        info = {name: self._tr_buf[:, j] for j, name in enumerate(TR_NAMES)}     # per-minibatch series, on device
        return info

    def epoch_times(self):
        """(play_time, update_time, total_time) in seconds from CUDA events (syncs)."""
        ev = self._events
        ev[2].synchronize()
        p, u = ev[0].elapsed_time(ev[1]) / 1e3, ev[1].elapsed_time(ev[2]) / 1e3
        return p, u, p + u

    def update_epoch(self):
        self.epoch_num += 1
        return self.epoch_num

    def _init_train(self):
        pass

    def _sync_stats(self):
        """Horovod sync_stats [recollection of rl_games]: RunningMeanStd buffers are averaged across ranks once per epoch."""
        from .dist_utils import sync_running_stats
        sync_running_stats(self._rms_modules())

    def train(self):
        """common_agent.py:82-155 (logging / checkpoint cadence kept; TensorBoard scalars are the caller's business)."""
        self.init_tensors()
        self.obs = self.env_reset()
        if self.multi_gpu:
            from .dist_utils import broadcast_state
            broadcast_state([self.model.params, self.model.exp_avg, self.model.exp_avg_sq])
            self.model.params_changed()
        self._init_train()
        # SURVEY 8f row 4: no per-epoch host sync -- the epoch's scalars and event timings come back through a pinned ring
        from .async_log import AsyncEpochLog
        from .lib import TR_NAMES
        log = AsyncEpochLog(list(TR_NAMES) + ['plane_status', 'ep_reward_sum', 'ep_length_sum', 'ep_count'], depth=4)
        self.last_mean_rewards = -100500
        self.epoch_log = []                       # [{'epoch', 'frames', 'scalars', 'play_time', 'update_time'}], an epoch or two behind
        total_time = 0.0

        def consume(recs):
            nonlocal total_time
            for r in recs:
                r.pop('series', None)
                # FP16 operand-plane scale status of the epoch (rides in the record: no extra sync).  A miss means the flagged updates
                # were not fp32-accurate: stop right here instead of training on them (ADVICE r1)
                status = int(r['scalars'].pop('plane_status', 0.0))
                if status & 4:
                    raise RuntimeError(f"epoch {r['epoch']}: a peer rank did not reach the gradient barrier of the multi-GPU optimizer step within ~15 s "
                                       "(csrc/peer.cu); that update was skipped -- restore() the last checkpoint")
                if status != 0:
                    raise RuntimeError(f"epoch {r['epoch']}: FP16 operand-plane scale miss -- a tensor's max moved by more than ~2^7 up / ~2^14 down between "
                                       "two consecutive calls; rerun with gemm_backend=1 (restore() the last checkpoint)")
                rs, ls, cnt = (r['scalars'].pop(k, 0.0) for k in ('ep_reward_sum', 'ep_length_sum', 'ep_count'))
                if cnt > 0:       # common_agent.py:125-136 (mean over the episodes that finished in this epoch)
                    r['mean_rewards'], r['mean_lengths'] = rs / cnt, ls / cnt
                    self.mean_rewards = r['mean_rewards']
                total_time += r.get('play_time', 0.0) + r.get('update_time', 0.0)
                r['total_time'] = total_time
                self.epoch_log.append(r)
                if self.rank == 0 and self.print_stats and 'play_time' in r:
                    tot = r['play_time'] + r['update_time']
                    print(f"epoch {r['epoch']}: fps step: {r['frames'] / r['play_time']:.1f} fps total: {r['frames'] / tot:.1f}")
                if self.writer is not None:       # performance/* and losses/* scalars of common_agent.py:119-152,551-564
                    self._write_stats(r)
                if self.rank == 0 and self.algo_observer is not None and hasattr(self.algo_observer, 'after_print_stats'):
                    self.algo_observer.after_print_stats(r['epoch'] * self.batch_size * self.rank_size, r['epoch'], total_time)     # common_agent.py:123

        model_output_file = os.path.join(self.nn_dir, self.config.get('name', self.name))
        while True:
            epoch_num = self.update_epoch()
            self.train_epoch()
            if self.multi_gpu:
                self._sync_stats()
            self.frame += self.curr_frames * self.rank_size
            consume(log.push(epoch_num, self._tr_buf, frames=self.curr_frames, events=tuple(self._events)))
            consume(log.poll())
            if self.rank == 0 and self.save_freq > 0 and epoch_num % self.save_freq == 0:      # common_agent.py:141-147
                self.save(model_output_file)
                if self._save_intermediate:
                    self.save(model_output_file + '_' + str(epoch_num).zfill(8))
            if epoch_num > self.max_epochs:                                                      # common_agent.py:149-152
                consume(log.flush())
                if self.rank == 0:
                    self.save(model_output_file)
                self.total_time = total_time
                return self.last_mean_rewards, epoch_num

    def _write_stats(self, r):
        """TensorBoard emission (common_agent.py:119-152, amp_agent.py:244-262) from an AsyncEpochLog record."""
        w, frame = self.writer, r['epoch'] * self.batch_size * self.rank_size
        if 'play_time' in r:
            tot = r['play_time'] + r['update_time']
            w.add_scalar('performance/total_fps', r['frames'] * self.rank_size / tot, frame)
            w.add_scalar('performance/step_fps', r['frames'] * self.rank_size / r['play_time'], frame)
            w.add_scalar('performance/update_time', r['update_time'], frame)
            w.add_scalar('performance/play_time', r['play_time'], frame)
        w.add_scalar('info/epochs', r['epoch'], frame)
        for k, v in r['scalars'].items():
            w.add_scalar(('info/' if k in ('kl', 'last_lr', 'lr_mul', 'e_clip') else 'losses/') + k, v, frame)
        if 'mean_rewards' in r:            # common_agent.py:125-136
            w.add_scalar('rewards0/frame', r['mean_rewards'], frame)
            w.add_scalar('rewards0/iter', r['mean_rewards'], r['epoch'])
            w.add_scalar('rewards0/time', r['mean_rewards'], r.get('total_time', 0.0))
            w.add_scalar('episode_lengths/frame', r['mean_lengths'], frame)
            w.add_scalar('episode_lengths/iter', r['mean_lengths'], r['epoch'])


class AMPAgent(CommonAgent):
    kind = 'amp'

    def _load_config_params(self, config):
        self._enable_eps_greedy = bool(config['enable_eps_greedy'])
        self._task_reward_w = config['task_reward_w']
        self._disc_reward_w = config['disc_reward_w']
        self._amp_observation_space = self.env_info['amp_observation_space']
        self._amp_batch_size = int(config['amp_batch_size'])
        self._amp_minibatch_size = int(config['amp_minibatch_size'])
        assert self._amp_minibatch_size <= self.minibatch_size
        self._disc_reward_scale = config['disc_reward_scale']
        assert config.get('normalize_amp_input', True)

    def _learner_kwargs(self, config):
        kw = super()._learner_kwargs(config)
        np_ = self._net_params(config)
        for k in ('disc_coef', 'disc_logit_reg', 'disc_grad_penalty', 'disc_weight_decay'):
            kw['hparams'][k] = config[k]
        kw.update(amp_dim=self._amp_observation_space.shape[0], amp_batch=self._amp_minibatch_size, disc_units=tuple(np_['disc']['units']))
        return kw

    def init_tensors(self):
        super().init_tensors()
        H, N, dev = self.horizon_length, self.num_actors, self.ppo_device
        eb = self.experience_buffer
        eb['amp_obs'] = torch.zeros(H, N, self._amp_observation_space.shape[0], device=dev)
        eb['rand_action_mask'] = torch.zeros(H, N, device=dev)
        self._amp_obs_demo_buffer = ReplayBuffer(int(self.config['amp_obs_demo_buffer_size']), dev)
        self._amp_replay_keep_prob = self.config['amp_replay_keep_prob']
        self._amp_replay_buffer = ReplayBuffer(int(self.config['amp_replay_buffer_size']), dev)
        self._build_rand_action_probs()
        self.tensor_list += ['amp_obs', 'rand_action_mask']

    def _build_rand_action_probs(self):
        """amp_agent.py:424-435: p_env = 1 - exp(10 (i/(N-1) - 1)), p_0 = 1, p_{N-1} = 0."""
        n = self.vec_env.env.task.num_envs
        ids = torch.arange(n, dtype=torch.float32, device=self.ppo_device)
        p = 1.0 - torch.exp(10 * (ids / (n - 1.0) - 1.0))
        p[0] = 1.0; p[-1] = 0.0
        if not self._enable_eps_greedy:
            p[:] = 1.0
        self._rand_action_probs = p

    def _rand_action_probs_tensor(self):
        return self._rand_action_probs

    def _extra_buffer_writes(self, n, res, infos):
        self.experience_buffer['amp_obs'][n] = infos['amp_obs']
        self.experience_buffer['rand_action_mask'][n] = res['rand_action_mask']

    def _extra_buffer_writes_device(self, n, infos):
        self.experience_buffer['amp_obs'][n].copy_(infos['amp_obs'])       # (rand_action_mask is written by the sampling kernel)

    def _calc_amp_rewards(self, amp_obs, latents=None):
        """amp_agent.py:563-577 / ase_agent.py:395-411: disc (+enc) trunk over the whole rollout, then the reward kernels."""
        H, N = amp_obs.shape[0], amp_obs.shape[1]
        logits, enc = self.model.eval_disc_enc(amp_obs.reshape(H * N, -1), want_enc=self.kind == 'ase')
        z = None if latents is None else latents.reshape(H * N, -1)
        dr, er, comb = ops.amp_rewards(logits, enc, z, self._disc_reward_scale, getattr(self, '_enc_reward_scale', 1.0),
                                       self.experience_buffer['rewards'].reshape(H * N), self._task_reward_w, self._disc_reward_w,
                                       getattr(self, '_enc_reward_w', 0.0))
        out = {'disc_rewards': dr.reshape(H, N, 1)}
        if er is not None:
            out['enc_rewards'] = er.reshape(H, N, 1)
        return comb.reshape(H, N, 1), out

    def _final_rewards(self):
        return self._calc_amp_rewards(self.experience_buffer['amp_obs'], None)

    def _calc_advs(self, batch_dict):
        return ops.calc_advs(batch_dict['returns'], batch_dict['values'], batch_dict['rand_action_mask'])

    def _init_train(self):
        """amp_agent.py:436-440,520-528: fill the demo buffer."""
        size = self._amp_obs_demo_buffer.get_buffer_size()
        for _ in range(int(math.ceil(size / self._amp_batch_size))):
            self._amp_obs_demo_buffer.store({'amp_obs': self.vec_env.env.fetch_amp_obs_demo(self._amp_batch_size)})

    def _pre_update(self, batch_dict):
        """amp_agent.py:194-202: refresh demos, draw the epoch's demo / replay sample (as indices)."""
        self._amp_obs_demo_buffer.store({'amp_obs': self.vec_env.env.fetch_amp_obs_demo(self._amp_batch_size)})
        n = batch_dict['amp_obs'].shape[0]
        self._demo_idx = self._amp_obs_demo_buffer.sample_indices(n).to(self.ppo_device)
        self._replay_idx = None if self._amp_replay_buffer.get_total_count() == 0 else self._amp_replay_buffer.sample_indices(n).to(self.ppo_device)

    def prepare_dataset(self, batch_dict):
        super().prepare_dataset(batch_dict)
        vd = self.dataset.values_dict
        vd['rand_action_mask'] = batch_dict['rand_action_mask']
        self._amp_obs_flat = batch_dict['amp_obs']

    def _minibatch_pairs(self, i):
        idx = self.dataset.sample_indices(i)
        a = idx[:self._amp_minibatch_size].contiguous()      # only amp_minibatch_size rows are consumed (ase_agent.py:172-181)
        pairs = [(k, v, idx) for k, v in self.dataset.values_dict.items() if v is not None]
        pairs.append(('amp_obs', self._amp_obs_flat, a))
        pairs.append(('amp_obs_demo', self._amp_obs_demo_buffer._data_buf['amp_obs'], self._demo_idx[a]))
        alias = {}
        if self._replay_idx is not None:
            pairs.append(('amp_obs_replay', self._amp_replay_buffer._data_buf['amp_obs'], self._replay_idx[a]))
        else:
            alias['amp_obs_replay'] = 'amp_obs'
        return pairs, alias

    def _post_update(self, batch_dict):
        """amp_agent.py:579-593 _store_replay_amp_obs."""
        amp_obs = batch_dict['amp_obs']
        size = self._amp_replay_buffer.get_buffer_size()
        if self._amp_replay_buffer.get_total_count() > size:
            keep = torch.bernoulli(torch.full((amp_obs.shape[0],), self._amp_replay_keep_prob, device=self.ppo_device)) == 1.0
            amp_obs = amp_obs[keep]
        if amp_obs.shape[0] > size:
            amp_obs = amp_obs[torch.randperm(amp_obs.shape[0], device=self.ppo_device)[:size]]
        if amp_obs.shape[0] > 0:
            self._amp_replay_buffer.store({'amp_obs': amp_obs})


class ASEAgent(AMPAgent):
    kind = 'ase'

    def _load_config_params(self, config):
        super()._load_config_params(config)
        self._latent_dim = config['latent_dim']
        self._latent_steps_min = config.get('latent_steps_min', np.inf)
        self._latent_steps_max = config.get('latent_steps_max', np.inf)
        self._enc_reward_scale = config['enc_reward_scale']
        self._enc_reward_w = config['enc_reward_w']
        assert config.get('enc_weight_decay', 0) == 0 and config.get('enc_grad_penalty', 0) == 0, "0 in the shipped config (ase_humanoid.yaml:108-110)"

    def _learner_kwargs(self, config):
        kw = super()._learner_kwargs(config)
        for k in ('enc_coef', 'amp_diversity_bonus', 'amp_diversity_tar'):
            kw['hparams'][k] = config[k]
        kw.update(latent_dim=self._latent_dim)
        return kw

    def init_tensors(self):
        super().init_tensors()
        H, N, dev = self.horizon_length, self.num_actors, self.ppo_device
        self.experience_buffer['ase_latents'] = torch.zeros(H, N, self._latent_dim, device=dev)
        self._ase_latents = torch.zeros(N, self._latent_dim, device=dev)
        self.tensor_list += ['ase_latents']
        self._latent_reset_steps = torch.zeros(N, dtype=torch.int32, device=dev)
        self._reset_latent_step_count(torch.arange(N, device=dev))

    def _sample_latents(self, n):
        """ase_network_builder.py:221-225."""
        z = torch.randn(n, self._latent_dim, device=self.ppo_device)
        return torch.nn.functional.normalize(z, dim=-1)

    def _new_latents(self, n):
        return self._sample_latents(n)

    def _reset_latents(self, env_ids):
        self._ase_latents[env_ids] = self._sample_latents(len(env_ids))

    def _draw_latent_steps(self, n):
        return torch.randint(self._latent_steps_min, self._latent_steps_max, (n,), dtype=torch.int32, device=self.ppo_device)

    def _reset_latent_step_count(self, env_ids):
        self._latent_reset_steps[env_ids] = self._draw_latent_steps(len(env_ids))

    def env_reset(self, env_ids=None):
        obs = super().env_reset(env_ids)
        if env_ids is None:
            env_ids = torch.arange(self.num_actors, device=self.ppo_device)
        if len(env_ids) > 0:
            self._reset_latents(env_ids)
            self._reset_latent_step_count(env_ids)
        return obs

    def _latents(self):
        return self._ase_latents

    def _pre_action(self):
        """ase_agent.py:366-381 _update_latents."""
        new = self._latent_reset_steps <= self.vec_env.env.task.progress_buf
        ids = new.nonzero(as_tuple=False).flatten()
        if ids.numel() > 0:
            self._reset_latents(ids)
            self._latent_reset_steps[ids] += self._draw_latent_steps(ids.numel())

    def _extra_buffer_writes(self, n, res, infos):
        super()._extra_buffer_writes(n, res, infos)
        self.experience_buffer['ase_latents'][n] = self._ase_latents

    def _extra_buffer_writes_device(self, n, infos):
        super()._extra_buffer_writes_device(n, infos)
        self.experience_buffer['ase_latents'][n].copy_(self._ase_latents)

    def _device_latent_step(self, done_mask, n):
        """env_reset's latent part + _update_latents in one mask-driven kernel (ase_agent.py:329-381)."""
        inj = getattr(self, '_inject', None)
        ops.latent_update(self._ase_latents, self._latent_reset_steps, self.vec_env.env.task.progress_buf, done_mask,
                          self._latent_steps_min, self._latent_steps_max, self._rng, 2,
                          z_in=None if inj is None else inj['z'][n], steps_in=None if inj is None else inj['steps'][n])

    def _final_rewards(self):
        eb = self.experience_buffer
        return self._calc_amp_rewards(eb['amp_obs'], eb['ase_latents'])

    def prepare_dataset(self, batch_dict):
        super().prepare_dataset(batch_dict)
        self.dataset.values_dict['ase_latents'] = batch_dict['ase_latents']


class HRLAgent(CommonAgent):
    """learning/hrl_agent.py: a PPO high-level controller whose 64-d action is the latent of a FROZEN ASE low-level
    controller, stepped `llc_steps` times per high-level step; reward = task_w * task + disc_w * LLC discriminator reward.
    The HLC network applies tanh to mu (hrl_network_builder.py:26-29).  The LLC comes either as a ready ase_b200.Learner
    (config['llc_learner']) or from the reference's pieces: config['llc_net_params'] (+ config['llc_checkpoint'], an
    rl_games .pth such as ase/data/models/ase_llc_reallusion_sword_shield.pth)."""
    kind = 'ppo'
    _mu_activation = 'tanh'

    def __init__(self, base_name, config):
        self._latent_dim = int(config.get('latent_dim', config.get('llc_latent_dim', 64)))
        super().__init__(base_name, config)
        self._task_size = self.vec_env.env.task.get_task_obs_size()
        self._llc_steps = config['llc_steps']
        self._llc_disc_reward_scale = config.get('llc_disc_reward_scale', 2.0)
        self._build_llc(config)

    def _load_config_params(self, config):
        self._task_reward_w = config['task_reward_w']
        self._disc_reward_w = config['disc_reward_w']
        self.actions_num = self._latent_dim            # hrl_agent.py:171-174 _setup_action_space

    def _build_llc(self, config):
        ln = config.get('llc_learner')
        if ln is None:
            np_ = config['llc_net_params']
            amp_dim = self.env_info['amp_observation_space'].shape[0]
            act = self.env_info['action_space'].shape[0]
            ln = Learner('ase', self.obs_shape[0] - self._task_size, act, self.num_actors, amp_dim=amp_dim, latent_dim=self._latent_dim,
                         amp_batch=max(2, self.num_actors), units=tuple(np_['mlp']['units']), disc_units=tuple(np_['disc']['units']),
                         device=self.ppo_device, gemm_backend=config.get('gemm_backend', 2))
            ckpt = config.get('llc_checkpoint')
            if ckpt:
                w = torch.load(ckpt, map_location='cpu', weights_only=True)
                ln.load_state_dict(w['model'])
                ln.set_stats_weights(w)
            else:
                ln.init_reference(seed=1)
        for r in (ln.running_mean_std, ln.value_mean_std, ln.amp_input_mean_std):
            r.eval()
        self._llc = ln

    def init_tensors(self):
        super().init_tensors()
        self.experience_buffer['disc_rewards'] = torch.zeros_like(self.experience_buffer['rewards'])
        self.tensor_list += ['disc_rewards']

    def _compute_llc_action(self, obs, actions):
        """hrl_agent.py:231-240: z = normalize(HLC action); LLC actor mean on the humanoid part of the observation."""
        llc_obs = obs[..., :obs.shape[-1] - self._task_size].contiguous()
        z = torch.nn.functional.normalize(actions, dim=-1)
        mu, _ = self._llc.eval_actor_critic(llc_obs, z, want_value=False)
        return torch.clamp(mu, -1.0, 1.0)

    def env_step(self, actions):
        """hrl_agent.py:45-82."""
        actions = torch.clamp(actions, -1.0, 1.0)
        obs = self.obs['obs']
        rewards = disc_rewards = done_count = terminate_count = 0.0
        for _ in range(self._llc_steps):
            llc_actions = self._compute_llc_action(obs, actions)
            obs, curr_rewards, curr_dones, infos = self.vec_env.step(llc_actions)
            rewards = rewards + curr_rewards
            done_count = done_count + curr_dones.float()
            terminate_count = terminate_count + infos['terminate'].float()
            logits, _ = self._llc.eval_disc_enc(infos['amp_obs'], want_enc=False)
            dr, _, _ = ops.amp_rewards(logits, None, None, self._llc_disc_reward_scale)
            disc_rewards = disc_rewards + dr
        rewards = rewards / self._llc_steps
        disc_rewards = disc_rewards / self._llc_steps
        infos = dict(infos)
        infos['terminate'] = (terminate_count > 0).to(torch.uint8)
        infos['disc_rewards'] = disc_rewards
        return {'obs': obs}, rewards.unsqueeze(1), (done_count > 0).to(torch.uint8), infos

    def _extra_buffer_writes(self, n, res, infos):
        self.experience_buffer['disc_rewards'][n] = infos['disc_rewards']

    def _extra_buffer_writes_device(self, n, infos):
        self.experience_buffer['disc_rewards'][n].copy_(infos['disc_rewards'].reshape(-1, 1))

    def _final_rewards(self):
        """hrl_agent.py:150-152,243-249 _combine_rewards."""
        eb = self.experience_buffer
        return self._task_reward_w * eb['rewards'] + self._disc_reward_w * eb['disc_rewards'], {}
