"""Learner: owns the flat parameter / gradient / Adam arenas (torch tensors), the RunningMeanStd
buffers and the C-side workspace, and exposes the reference's per-minibatch update
(ASEAgent.calc_gradients, learning/ase_agent.py:159-308) as two device calls:
`calc_gradients` (forward + losses + backward) and `adam_step` (optionally after an NCCL all-reduce of
the flat gradient).  Parameters are exposed under the reference's state_dict names as views into the arena,
so shipped checkpoints load/save unchanged (SURVEY.md Appendix B)."""
import ctypes as C
import math
from collections import OrderedDict

import torch

from . import lib as L
from .lib import lib, check
from .ops import RunningMeanStd, _p, _stream

KINDS = {'ppo': L.KIND_PPO, 'amp': L.KIND_AMP, 'ase': L.KIND_ASE}

# hyper-parameter defaults = data/cfg/train/rlg/ase_humanoid.yaml:59-114
DEFAULT_HPARAMS = dict(
    e_clip=0.2, critic_coef=5.0, entropy_coef=0.0, bounds_loss_coef=10.0, disc_coef=5.0, disc_logit_reg=0.01,
    disc_grad_penalty=5.0, disc_weight_decay=1e-4, enc_coef=5.0, amp_diversity_bonus=0.01, amp_diversity_tar=1.0,
    learning_rate=2e-5, beta1=0.9, beta2=0.999, adam_eps=1e-8, rms_eps=1e-5)


def param_names(kind, n_units, n_disc_units, n_style_units):
    """Trainable tensors in model.parameters() order (Adam order) without the frozen `sigma`."""
    names = []
    if kind == 'ase':
        for k in range(n_style_units):
            names += [f'actor_mlp._style_mlp.{2 * k}.weight', f'actor_mlp._style_mlp.{2 * k}.bias']
        names += ['actor_mlp._style_dense.weight', 'actor_mlp._style_dense.bias']
        for k in range(n_units):
            names += [f'actor_mlp._dense_layers.{k}.weight', f'actor_mlp._dense_layers.{k}.bias']
        for k in range(n_units):
            names += [f'critic_mlp._mlp.{2 * k}.weight', f'critic_mlp._mlp.{2 * k}.bias']
    else:
        for k in range(n_units):
            names += [f'actor_mlp.{2 * k}.weight', f'actor_mlp.{2 * k}.bias']
        for k in range(n_units):
            names += [f'critic_mlp.{2 * k}.weight', f'critic_mlp.{2 * k}.bias']
    names += ['value.weight', 'value.bias', 'mu.weight', 'mu.bias']
    if kind != 'ppo':
        for k in range(n_disc_units):
            names += [f'_disc_mlp.{2 * k}.weight', f'_disc_mlp.{2 * k}.bias']
        names += ['_disc_logits.weight', '_disc_logits.bias']
        if kind == 'ase':
            names += ['_enc.weight', '_enc.bias']
    return names


def _aligned_bytes(nbytes, device, align=1024):
    buf = torch.empty(nbytes + align, dtype=torch.uint8, device=device)
    off = (-buf.data_ptr()) % align
    return buf[off:off + nbytes]


class Learner:
    def __init__(self, kind, obs_dim, act_dim, batch, amp_dim=0, latent_dim=0, amp_batch=0, units=(1024, 1024, 512),
                 disc_units=(1024, 1024, 512), style_units=(512, 256), hparams=None, device='cuda', gemm_backend=0,
                 sigma_init=-2.9, mu_activation='None'):
        assert kind in KINDS
        self.kind = kind
        self.device = torch.device(device)
        hp = dict(DEFAULT_HPARAMS); hp.update(hparams or {})
        self.hp = hp
        cfg = L.LearnerConfig()
        cfg.kind = KINDS[kind]
        cfg.obs_dim, cfg.act_dim, cfg.amp_dim, cfg.latent_dim = obs_dim, act_dim, amp_dim if kind != 'ppo' else 0, latent_dim if kind == 'ase' else 0
        cfg.n_units = len(units)
        for i, u in enumerate(units): cfg.units[i] = u
        if kind != 'ppo':
            cfg.n_disc_units = len(disc_units)
            for i, u in enumerate(disc_units): cfg.disc_units[i] = u
        if kind == 'ase':
            cfg.n_style_units = len(style_units)
            for i, u in enumerate(style_units): cfg.style_units[i] = u
        cfg.batch, cfg.amp_batch = batch, amp_batch if kind != 'ppo' else 0
        for k in ('e_clip', 'critic_coef', 'entropy_coef', 'bounds_loss_coef', 'disc_coef', 'disc_logit_reg', 'disc_grad_penalty',
                  'disc_weight_decay', 'enc_coef', 'amp_diversity_bonus', 'amp_diversity_tar', 'beta1', 'beta2', 'adam_eps', 'rms_eps'):
            setattr(cfg, k, float(hp[k]))
        if kind != 'ase':
            cfg.amp_diversity_bonus = 0.0
        cfg.lr = float(hp['learning_rate'])
        cfg.gemm_backend = int(gemm_backend)
        cfg.mu_activation = 2 if mu_activation == 'tanh' else 0     # HRLBuilder.Network.forward: norm_mu = tanh(mu)
        self.cfg = cfg
        self.batch, self.amp_batch = batch, cfg.amp_batch
        self.obs_dim, self.act_dim, self.amp_dim, self.latent_dim = obs_dim, act_dim, cfg.amp_dim, cfg.latent_dim

        n = lib.ase_learner_num_params(C.byref(cfg))
        if n <= 0:
            raise L.AseError(f"bad learner config: {lib.ase_last_error().decode()}")
        names = param_names(kind, len(units), len(disc_units), len(style_units))
        assert len(names) == n, (len(names), n)
        arena = lib.ase_learner_arena_floats(C.byref(cfg))
        dev = self.device
        pad = (arena + 3) // 4 * 4          # the peer-memory optimizer step moves 16 bytes at a time: keep the arenas readable up to a multiple of 4 floats
        self.params = torch.zeros(pad, dtype=torch.float32, device=dev)[:arena]
        self.grads = torch.zeros(pad, dtype=torch.float32, device=dev)[:arena]
        self.exp_avg = torch.zeros(pad, dtype=torch.float32, device=dev)[:arena]
        self.exp_avg_sq = torch.zeros(pad, dtype=torch.float32, device=dev)[:arena]
        self._peer = None                   # AsePeer* when the gradient arena lives in NVLink peer memory (dist_utils.init_peer)
        self._param_slices = []
        self.sigma = torch.full((act_dim,), float(sigma_init), dtype=torch.float32, device=dev)   # frozen logstd parameter
        self.step = 0
        self._views = OrderedDict()
        self._gviews = OrderedDict()
        for i, name in enumerate(names):
            off, rows, cols = C.c_int64(), C.c_int(), C.c_int()
            check(lib.ase_learner_param_desc(C.byref(cfg), i, C.byref(off), C.byref(rows), C.byref(cols)), 'param_desc')
            shape = (cols.value,) if name.endswith('.bias') else (rows.value, cols.value)
            sl = slice(off.value, off.value + rows.value * cols.value)
            self._views[name] = self.params[sl].view(shape)
            self._gviews[name] = self.grads[sl].view(shape)
            self._param_slices.append((name, sl, shape))
        self.running_mean_std = RunningMeanStd(obs_dim, dev, hp['rms_eps'])          # common_agent.py:49
        self.value_mean_std = RunningMeanStd(1, dev, hp['rms_eps'])                  # rl_games A2CBase ('reward_mean_std')
        self.amp_input_mean_std = RunningMeanStd(cfg.amp_dim, dev, hp['rms_eps']) if kind != 'ppo' else None   # amp_agent.py:26

        ws_bytes = lib.ase_learner_workspace_bytes(C.byref(cfg))
        if ws_bytes <= 0:
            raise L.AseError(f"workspace query failed: {lib.ase_last_error().decode()}")
        self._ws = _aligned_bytes(ws_bytes, dev)
        h = C.c_void_p()
        check(lib.ase_learner_create(C.byref(cfg), self._ws.data_ptr(), ws_bytes, C.byref(h)), 'ase_learner_create')
        self._h = h
        self._scalars = torch.zeros(L.TR_COUNT, dtype=torch.float32, device=dev)
        self._agent_logit = torch.zeros(max(2 * cfg.amp_batch, 1), dtype=torch.float32, device=dev)
        self._demo_logit = torch.zeros(max(cfg.amp_batch, 1), dtype=torch.float32, device=dev)
        self._mu = torch.zeros(batch, act_dim, dtype=torch.float32, device=dev)
        self._val = torch.zeros(batch, dtype=torch.float32, device=dev)

    def __del__(self):
        h = getattr(self, '_h', None)
        if h:
            lib.ase_learner_destroy(h)
            self._h = None

    # ------------------------------------------------------------------ parameters / checkpoints
    def named_parameters(self):
        return self._views

    def named_grads(self):
        return self._gviews

    def init_reference(self, seed=0):
        """Reference initialisation: torch default Linear init (kaiming_uniform(a=sqrt5) = U(+-1/sqrt(fan_in))), zero
        biases, _disc_logits U(-1,1), _enc U(-0.1,0.1), _style_dense U(-1,1)
        (amp_network_builder.py:112-120, ase_network_builder.py:196-210,326-336)."""
        g = torch.Generator().manual_seed(seed)
        for name, v in self._views.items():
            if name.endswith('.bias'):
                v.zero_()
                continue
            bound = 1.0 / math.sqrt(v.shape[1])
            if name.startswith('_disc_logits') or name.startswith('actor_mlp._style_dense'):
                bound = 1.0
            elif name.startswith('_enc.'):
                bound = 0.1
            v.copy_(((torch.rand(v.shape, generator=g) * 2 - 1) * bound).to(v.device))
        self.params_changed()

    def params_changed(self):
        """Tell the library the parameter arena was written from outside (the tensor-core backends cache weight planes)."""
        check(lib.ase_learner_params_changed(self._h), 'ase_learner_params_changed')

    def load_named(self, named):
        """named: {reference name without the 'a2c_network.' prefix: tensor}"""
        for k, v in self._views.items():
            v.copy_(named[k].to(v.device).reshape(v.shape))
        if 'sigma' in named:
            self.sigma.copy_(named['sigma'].to(self.device))
        self.params_changed()

    def state_dict(self):
        sd = OrderedDict()
        sd['a2c_network.sigma'] = self.sigma
        for k, v in self._views.items():
            if self.kind == 'ase' and k == '_enc.weight':      # enc.separate False: the encoder trunk IS the discriminator trunk -- the reference's
                for kk, vv in self._views.items():             # state dict lists the same tensors again as _enc_mlp.* between _disc_logits and _enc
                    if kk.startswith('_disc_mlp.'):
                        sd['a2c_network.' + kk.replace('_disc_mlp', '_enc_mlp')] = vv
            sd['a2c_network.' + k] = v
        return sd

    def load_state_dict(self, sd):
        self.load_named({k[len('a2c_network.'):]: v for k, v in sd.items() if '_enc_mlp' not in k})

    def get_stats_weights(self):
        st = {'running_mean_std': self.running_mean_std.state_dict(), 'reward_mean_std': self.value_mean_std.state_dict()}
        if self.amp_input_mean_std is not None:
            st['amp_input_mean_std'] = self.amp_input_mean_std.state_dict()
        return st

    def set_stats_weights(self, w):
        self.running_mean_std.load_state_dict(w['running_mean_std'])
        self.value_mean_std.load_state_dict(w['reward_mean_std'])
        if self.amp_input_mean_std is not None and 'amp_input_mean_std' in w:
            self.amp_input_mean_std.load_state_dict(w['amp_input_mean_std'])

    # ------------------------------------------------------------------ device calls
    def _state(self):
        r, a = self.running_mean_std, self.amp_input_mean_std
        return L.LearnerState(_p(self.params), _p(self.grads), _p(self.exp_avg), _p(self.exp_avg_sq), _p(self.sigma),
                              _p(r.running_mean), _p(r.running_var), _p(r.count),
                              _p(a.running_mean) if a else None, _p(a.running_var) if a else None, _p(a.count) if a else None)

    @staticmethod
    def _c(t, shape=None):
        if t is None:
            return None
        if t.dtype != torch.float32 or not t.is_cuda:
            raise TypeError("minibatch tensors must be CUDA float32")
        t = t if t.is_contiguous() else t.contiguous()
        return t

    def calc_gradients(self, d, new_latents=None, update_rms=True, want_logits=True):
        """d: minibatch dict with the reference's key names (ase_agent.py:162-186).  Fills self.grads and
        returns a dict of device tensors (no host sync)."""
        B, Ba = self.batch, self.amp_batch
        keep = []

        def c(key, rows=None):
            t = d.get(key)
            if t is None:
                return None
            if rows is not None:
                t = t[0:rows]
            t = self._c(t); keep.append(t)
            return t.data_ptr()
        if d['obs'].shape[0] != B:
            raise ValueError(f"minibatch has {d['obs'].shape[0]} rows, learner was built for {B}")
        if self.kind == 'ase' and self.cfg.amp_diversity_bonus != 0 and new_latents is None:
            raise ValueError("ASE learner needs new_latents (the z' of _diversity_loss)")
        nl = None
        if new_latents is not None:
            nl = self._c(new_latents); keep.append(nl)
        mb = L.Minibatch(c('obs'), c('actions'), c('old_logp_actions'), c('advantages'), c('mu'), c('sigma'), c('returns'),
                         c('old_values'), c('rand_action_mask'), c('ase_latents'), _p(nl),
                         c('amp_obs', Ba), c('amp_obs_replay', Ba), c('amp_obs_demo', Ba), int(bool(update_rms)))
        tr = L.TrainResult(_p(self._scalars), _p(self._agent_logit) if (want_logits and Ba) else None,
                           _p(self._demo_logit) if (want_logits and Ba) else None, _p(self._mu), _p(self._val))
        st = self._state()
        check(lib.ase_learner_calc_gradients(self._h, C.byref(st), C.byref(mb), C.byref(tr), _stream()), 'ase_learner_calc_gradients')
        out = {'scalars': self._scalars, 'mus': self._mu, 'values': self._val}
        if Ba:
            out['disc_agent_logit'] = self._agent_logit
            out['disc_demo_logit'] = self._demo_logit
        return out

    def use_grads_arena(self, flat):
        """Accumulate the gradients into `flat` (a float32 CUDA tensor of at least the arena size, e.g. the rank's NVLink peer buffer) from now
        on.  Call before the first calc_gradients (a captured minibatch graph bakes the address in)."""
        n = self.grads.numel()
        assert flat.is_cuda and flat.dtype == torch.float32 and flat.is_contiguous() and flat.numel() >= n
        self._grads_store = flat
        self.grads = flat[:n]
        self.grads.zero_()
        for name, sl, shape in self._param_slices:
            self._gviews[name] = self.grads[sl].view(shape)

    def adam_step(self, grad_scale=1.0):
        """torch.optim.Adam step on the flat arenas.  With a peer buffer attached (multi-GPU, dist_utils.init_peer) the SAME call first sums
        the gradient arenas of all ranks over NVLink peer memory, inside the same kernel (ase_learner_peer_adam_step)."""
        self.step += 1
        st = self._state()
        if self._peer is not None:
            check(lib.ase_learner_peer_adam_step(self._h, self._peer, C.byref(st), self.step, float(grad_scale), _stream()), 'ase_learner_peer_adam_step')
            return
        check(lib.ase_learner_adam_step(self._h, C.byref(st), self.step, float(grad_scale), _stream()), 'ase_learner_adam_step')

    def plane_status(self):
        """gemm_backend 2: raises if a tensor left the window of its predicted FP16 plane scale (include/ase_b200.h,
        ase_learner_plane_status) -- the flagged update would not be fp32-accurate.  One stream synchronisation."""
        f = C.c_int(0)
        check(lib.ase_learner_plane_status(self._h, C.byref(f), _stream()), 'ase_learner_plane_status')
        if f.value & 4:
            raise L.AseError("multi-GPU optimizer step: a peer rank did not reach the gradient barrier within ~15 s (csrc/peer.cu); the update was skipped")
        if f.value:
            raise L.AseError(f"FP16 operand-plane scale miss (flags {f.value}: bit0 overflow, bit1 underflow): a tensor's max moved by more "
                             "than ~2^7 up / ~2^14 down between two consecutive calls; rerun with gemm_backend=1")
        return 0

    def plane_flag_to(self, dst):
        """Write the sticky FP16 plane-scale status (0 = fine) into every element of the 1-D float view `dst`, on the stream (no sync)."""
        check(lib.ase_learner_plane_flag_to(self._h, dst.data_ptr(), dst.shape[0], dst.stride(0), _stream()), 'ase_learner_plane_flag_to')

    def plane_flag_clear(self):
        check(lib.ase_learner_plane_flag_clear(self._h, _stream()), 'ase_learner_plane_flag_clear')

    def train_result(self, out):
        """Host-side view of the last train_result with the reference's key names (one D2H copy)."""
        s = out['scalars'].tolist()
        if self.cfg.gemm_backend == 2:
            self.plane_status()
        return dict(zip(L.TR_NAMES, s))

    def eval_actor_critic(self, obs, latents=None, want_value=True, want_actor=True):
        """Eval-mode actor and/or critic forward (ase_agent.py:117-148,385-393) -> (mu [n,act] or None, normalised value [n,1] or None)."""
        n = obs.shape[0]
        obs = self._c(obs); lat = self._c(latents)
        mu = torch.empty(n, self.act_dim, dtype=torch.float32, device=self.device) if want_actor else None
        val = torch.empty(n, 1, dtype=torch.float32, device=self.device) if want_value else None
        st = self._state()
        for s in range(0, n, self.batch):
            e = min(n, s + self.batch)
            check(lib.ase_learner_eval_actor_critic(self._h, C.byref(st), obs[s:e].data_ptr(), lat[s:e].data_ptr() if lat is not None else None,
                                                    e - s, mu[s:e].data_ptr() if want_actor else None, val[s:e].data_ptr() if want_value else None, _stream()),
                  'ase_learner_eval_actor_critic')
        return mu, val

    def eval_disc_enc(self, amp_obs, want_enc=None):
        """Eval-mode discriminator logits (+ encoder prediction) on [n, amp_dim] (ase_agent.py:395-411)."""
        if want_enc is None:
            want_enc = self.kind == 'ase'
        n = amp_obs.shape[0]
        x = self._c(amp_obs)
        logits = torch.empty(n, 1, dtype=torch.float32, device=self.device)
        enc = torch.empty(n, self.latent_dim, dtype=torch.float32, device=self.device) if want_enc else None
        st = self._state()
        step = 3 * self.amp_batch
        for s in range(0, n, step):
            e = min(n, s + step)
            check(lib.ase_learner_eval_disc_enc(self._h, C.byref(st), x[s:e].data_ptr(), e - s, logits[s:e].data_ptr(),
                                                enc[s:e].data_ptr() if want_enc else None, _stream()), 'ase_learner_eval_disc_enc')
        return logits, enc
