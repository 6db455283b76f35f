"""TEST INFRASTRUCTURE ONLY.  fp64 twin of the evaluation players' run(): learning/common_player.py:25-127 (AMPPlayerContinuous),
ase_players.py:28-98 (latent resets, the global numpy countdown and the colour draws) and hrl_players.py:36-251 (the HLC action, normalised,
as the latent of llc_steps frozen-LLC sub-steps), in the reference's own order with index lists, over ScriptEnv.  Draws are injected:
draws['noise'][k] is the eps of the k-th Normal.sample, draws['z'][k] the [N, Z] table of the k-th _reset_latents call (env i takes row i)."""
import numpy as np
import torch

import ase_oracle as O

# shapes of the player fixtures (oracle/gen_golden_players.py, tests/test_gpu_player.py)
D, AMP, A, Z, TASK = 40, 20, 8, 64, 5
UNITS = [128, 64]
LOW = [-1.0, -2.0, -0.5, 0.0, -3.0, -1.0, 1.0, -0.25]          # a non-unit action box, one component entirely below zero
HIGH = [1.0, 2.0, 1.5, 4.0, -1.0, 0.5, 3.0, 0.25]


def rms(dim, seed):
    g = torch.Generator().manual_seed(seed)
    return {'running_mean': torch.randn(dim, generator=g).double() * 0.3, 'running_var': torch.rand(dim, generator=g).double() + 0.5,
            'count': torch.tensor(1000.0, dtype=torch.float64)}


def params(kind, seed):
    """Reference state-dict names without 'a2c_network.'; mu scaled so head outputs go well beyond +-1."""
    if kind == 'ase':
        P = O.synthetic_params(O.ase_param_shapes(obs=D, z=Z, act=A, amp=AMP, units=UNITS, disc_units=UNITS), seed=seed, sigma_val=-1.0)
    elif kind == 'amp':
        P = O.synthetic_params(O.amp_param_shapes(obs=D, act=A, amp=AMP, units=UNITS, disc_units=UNITS), seed=seed, sigma_val=-1.0)
    elif kind == 'hrl':          # the HLC: a plain PPO network acting in the latent space
        P = O.synthetic_params(O.amp_param_shapes(obs=D, act=Z, amp=0, units=UNITS), seed=seed, sigma_val=-1.0)
    else:                        # 'llc'
        P = O.synthetic_params(O.ase_param_shapes(obs=D - TASK, z=Z, act=A, amp=AMP, units=UNITS, disc_units=UNITS), seed=seed)
    P['mu.weight'] = P['mu.weight'] * 12.0
    return P


def checkpoint(P, obs_rms, amp_rms=None):
    """An rl_games checkpoint: the model under the reference's names (the ASE encoder trunk aliased as _enc_mlp) and the normalisers."""
    sd = {'a2c_network.' + k: v.clone() for k, v in P.items()}
    for k in list(sd):
        if '_disc_mlp' in k and any('_enc.' in kk for kk in sd):
            sd[k.replace('_disc_mlp', '_enc_mlp')] = sd[k]
    w = {'model': sd, 'running_mean_std': obs_rms, 'reward_mean_std': rms(1, 9)}
    if amp_rms is not None:
        w['amp_input_mean_std'] = amp_rms
    return w




def tables(n, seed, T=53, done_p=0.09, obs_dim=40, amp_dim=20):
    """The scripted env of the player fixtures (oracle/gen_golden_players.py): step t returns obs_t[t + 1], rew_t[t], dones_t[t], amp_t[t]
    (t modulo T); a reset sets rows to reset_obs_t[t].  Regenerated from the seed instead of stored."""
    g = torch.Generator().manual_seed(seed)
    dones = (torch.rand(T, n, generator=g) < done_p).to(torch.uint8)
    dones[5, :min(n, 7)] = 1                      # several envs finish on one step
    return {'obs_t': torch.randn(T + 1, n, obs_dim, generator=g) * 2.0, 'reset_obs_t': torch.randn(T, n, obs_dim, generator=g) * 2.0,
            'rew_t': torch.rand(T, n, generator=g) * 3.0 - 1.0, 'dones_t': dones, 'amp_t': torch.randn(T, n, amp_dim, generator=g)}


def latent_tables(rec, n):
    """The recorded sample_latents rows as one [N, Z] table per _reset_latents call (env i takes row i), the form the players inject."""
    out = []
    for rows, ids in zip(rec['latents'], rec['latent_ids']):
        t = torch.zeros(n, rows.shape[1])
        if ids is None:
            t[:] = rows
        else:
            t[ids] = rows
        out.append(t)
    return out


class ScriptEnv:
    """A vec-env that replays tables: step t returns obs_t[t + 1], rew_t[t], dones_t[t] (indices modulo the table length); reset(ids) sets
    the rows of ids (every row for None) to reset_obs_t[t].  Records the actions of every step."""

    def __init__(self, tables, device='cpu', dtype=None):
        self.t = 0
        conv = (lambda x: x.to(device)) if dtype is None else (lambda x: x.to(device=device, dtype=dtype))
        self.obs_t, self.reset_obs_t, self.rew_t = conv(tables['obs_t']), conv(tables['reset_obs_t']), conv(tables['rew_t'])
        self.dones_t = tables['dones_t'].to(device)
        self.amp_t = conv(tables['amp_t'])
        self.T = self.rew_t.shape[0]
        self.cur = self.reset_obs_t[0].clone()
        self.actions = []

    def step(self, actions):
        t = self.t % self.T
        self.actions.append(actions.clone())
        self.cur = self.obs_t[t + 1].clone()
        self.t += 1
        return self.cur, self.rew_t[t].clone(), self.dones_t[t].clone(), {'amp_obs': self.amp_t[t].clone()}

    def reset(self, env_ids=None):
        if env_ids is None:
            self.cur = self.reset_obs_t[self.t % self.T].clone()
        elif len(env_ids) > 0:
            ids = torch.as_tensor(env_ids, dtype=torch.long, device=self.cur.device).reshape(-1)
            self.cur[ids] = self.reset_obs_t[self.t % self.T][ids]
        return self.cur


def _rescale(a, low, high):
    """rl_games rescale_actions."""
    d = (high - low) / 2.0
    m = (high + low) / 2.0
    return a * d + m


def run(kind, P, obs_rms, env, cfg, draws, llc=None, dtype=torch.float64):
    """kind 'amp' / 'ase' / 'hrl'.  P: the network's parameters (reference names without 'a2c_network.'); obs_rms: ase_oracle.RMS;
    cfg: games_num, n_game_life, determenistic, max_steps, low, high [A] and (ASE) latent_dim, latent_steps_min / max, (HRL) llc_steps,
    task_size; llc: (LLC parameters, LLC RMS).  Returns {'lines', 'games_played', 'sum_rewards', 'sum_steps'}; env.actions holds the actions."""
    P = {k: v.to(dtype) for k, v in P.items()}
    low, high = cfg['low'].to(dtype), cfg['high'].to(dtype)
    det = cfg['determenistic']
    N = env.cur.shape[0]
    calls = {'noise': 0, 'z': 0}
    lat = torch.zeros(N, cfg.get('latent_dim', 1), dtype=dtype)
    lines = []

    def draw(name):
        k = calls[name]
        calls[name] = k + 1
        return draws[name][k].to(dtype)

    def reset_latents(ids):                       # ase_players.py:71-80, 143-152 (headless: the colour's three uniforms only)
        z = draw('z')
        ids = torch.arange(N) if ids is None else ids
        lat[ids] = z[ids]
        np.random.uniform(0.0, 1.0, size=3)

    state, countdown = {}, []

    def reset_count():
        state['count'] = np.random.randint(cfg['latent_steps_min'], cfg['latent_steps_max'])
        countdown.append(int(state['count']))

    def env_reset(ids):
        obs = env.reset(ids)
        if kind == 'ase':
            reset_latents(ids)
        return obs

    def head(obs):
        mu = O.eval_actor(P, obs_rms.norm(obs.to(dtype)), lat if kind == 'ase' else None, mu_tanh=kind == 'hrl')
        a = mu if det else mu + torch.exp(P['sigma']) * draw('noise')
        return torch.clamp(a, -1.0, 1.0)

    def step(obs):
        if kind == 'ase':                         # _update_latents
            if state['count'] <= 0:
                reset_latents(None)
                reset_count()
            else:
                state['count'] -= 1
        a = head(obs)
        if kind != 'hrl':
            obs, r, d, _ = env.step(_rescale(a, low, high))
            return obs, r.to(dtype), d
        z = torch.nn.functional.normalize(a, dim=-1)
        Pl, rms_l = {k: v.to(dtype) for k, v in llc[0].items()}, llc[1]
        rewards, done_count = 0.0, 0.0
        for _ in range(cfg['llc_steps']):         # hrl_players.py:169-191
            llc_obs = obs[..., :obs.shape[-1] - cfg['task_size']]
            mu = O.eval_actor(Pl, rms_l.norm(llc_obs.to(dtype)), z)
            obs, r, d, _ = env.step(_rescale(torch.clamp(mu, -1.0, 1.0), low, high))
            rewards = rewards + r.to(dtype)
            done_count = done_count + d.to(dtype)
        return obs, rewards / cfg['llc_steps'], (done_count > 0).to(dtype)

    n_game_life = cfg['n_game_life']
    n_games = cfg['games_num'] * n_game_life
    sum_rewards, sum_steps, games_played = 0, 0, 0
    if kind == 'ase':
        reset_count()
    for _ in range(n_games):
        if games_played >= n_games:
            break
        obs = env_reset(None)
        cr = torch.zeros(N, dtype=dtype)
        steps = torch.zeros(N, dtype=dtype)
        done_indices = []
        for _n in range(cfg['max_steps']):
            obs = env_reset(done_indices)
            obs, r, done = step(obs)
            cr += r
            steps += 1
            done_indices = done.nonzero(as_tuple=False)[:, 0]
            done_count = len(done_indices)
            games_played += done_count
            if done_count > 0:
                cur_rewards = cr[done_indices].sum().item()
                cur_steps = steps[done_indices].sum().item()
                cr = cr * (1.0 - done.to(dtype))
                steps = steps * (1.0 - done.to(dtype))
                sum_rewards += cur_rewards
                sum_steps += cur_steps
                lines.append(('reward:', cur_rewards / done_count, 'steps:', cur_steps / done_count))
                if N == 1 or games_played >= n_games:
                    break
    lines.append((sum_rewards,))
    lines.append(('av reward:', sum_rewards / games_played * n_game_life, 'av steps:', sum_steps / games_played * n_game_life))
    return {'lines': lines, 'games_played': games_played, 'sum_rewards': sum_rewards, 'sum_steps': sum_steps, 'countdown': countdown}


def _rms(sd):
    r = O.RMS(sd['running_mean'].shape[0])
    r.mean, r.var, r.count = sd['running_mean'].clone(), sd['running_var'].clone(), sd['count'].clone()
    return r


def run_fixture(fx, dtype=torch.float64):
    """One run of tests/golden/player_*.pt replayed: the same parameters, script, draws and numpy seed.  -> (run()'s result, the env)."""
    kind, n = fx['kind'], fx['N']
    env = ScriptEnv(tables(n, fx['table_seed']))
    cfg = {k: fx[k] for k in ('games_num', 'determenistic', 'max_steps', 'llc_steps', 'task_size')}
    cfg.update(n_game_life=1, low=fx['low'], high=fx['high'], latent_dim=Z, latent_steps_min=1, latent_steps_max=4)
    draws = {'noise': fx['rec']['normal'], 'z': latent_tables(fx['rec'], n)}
    llc = (params('llc', 31), _rms(rms(D - TASK, 32))) if kind == 'hrl' else None
    np.random.seed(fx['np_seed'])
    return run(kind, params(kind, 11), _rms(rms(D, 12)), env, cfg, draws, llc=llc, dtype=dtype), env
