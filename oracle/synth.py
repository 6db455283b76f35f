"""TEST INFRASTRUCTURE ONLY -- seeded synthetic inputs shared by oracle/gen_golden.py, tests/ and
bench.py's CPU legs (SURVEY.md section 8(d) "Synthetic inputs").  torch CPU generators only, so the same
seed regenerates the same tensors on the GPU box (same image, same torch)."""
import math
import torch
import torch.nn.functional as F

import ase_oracle as O


def rigid_body_state(n, seed=0, bodies=17, dofs=31, edge_cases=False):
    g = torch.Generator().manual_seed(seed)
    pos = torch.randn(n, bodies, 3, generator=g)
    pos[:, 0, 2] = 0.5 + 0.7 * torch.rand(n, generator=g)
    rot = F.normalize(torch.randn(n, bodies, 4, generator=g), dim=-1)
    vel = torch.randn(n, bodies, 3, generator=g)
    ang = torch.randn(n, bodies, 3, generator=g)
    dof_pos = torch.rand(n, dofs, generator=g) * 2 - 1
    dof_vel = torch.randn(n, dofs, generator=g) * 2
    if edge_cases and n >= 8:
        rot[0, :] = torch.tensor([0., 0., 0., 1.])          # identity
        rot[1, 0] = torch.tensor([0., 0., 1., 0.])          # heading = pi
        rot[2, 0] = F.normalize(torch.tensor([1., 0., 0., 1.]), dim=0)   # pitch-free roll
        dof_pos[3, :] = 0.0                                 # zero exp-map -> default-axis branch
        dof_pos[4, 0:3] = torch.tensor([1e-6, 0., 0.])      # |angle| <= 1e-5 branch
        dof_pos[5, 0:3] = torch.tensor([3.5, 0.5, -0.2])    # angle > pi -> normalize_angle wraps
        dof_pos[6, 9] = 4.0                                 # 1-dof joint beyond pi
    return dict(body_pos=pos, body_rot=rot, body_vel=vel, body_ang_vel=ang, dof_pos=dof_pos, dof_vel=dof_vel)


def params(shapes, seed=0):
    p = O.synthetic_params(shapes, seed=seed)
    g = torch.Generator().manual_seed(seed + 1000)
    # push some action means beyond +-1 so bound loss and the diversity clip are exercised
    p['mu.bias'] = (torch.rand(p['mu.bias'].shape, generator=g) * 2 - 1) * 1.3
    return p


def minibatch(st, cfg, B, Ba, seed, kind='ase', obs_dim=253, amp_dim=1400, act=31, zdim=64):
    """One minibatch dict with the reference's key names (ase_agent.py:162-186).  old_logp_actions is
    set near the current policy's neglogp (ratio in ~[0.7,1.4]) so that clipped and unclipped samples,
    both signs of advantage, masked rows and out-of-bound means all occur."""
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(B, obs_dim, generator=g) * 1.5 + 0.3
    z = F.normalize(torch.randn(B, zdim, generator=g), dim=-1) if kind == 'ase' else None
    new_z = F.normalize(torch.randn(B, zdim, generator=g), dim=-1) if kind == 'ase' else None
    with torch.no_grad():
        rms = st.obs_rms.clone(); rms.update(obs)
        mu_cur = O.eval_actor(st.p, rms.norm(obs), z, mu_tanh=cfg.get('mu_tanh', False))
    sig = math.exp(-2.9)
    actions = mu_cur + sig * torch.randn(B, act, generator=g)
    logstd = torch.full((act,), -2.9)
    nlp = O.neglogp(actions, mu_cur, logstd)
    d = dict(old_values=torch.randn(B, 1, generator=g),
             old_logp_actions=nlp + 0.15 * torch.randn(B, generator=g),
             advantages=torch.randn(B, generator=g),
             mu=mu_cur + 0.02 * torch.randn(B, act, generator=g),
             sigma=torch.full((B, act), sig),
             returns=torch.randn(B, 1, generator=g),
             actions=actions, obs=obs)
    if kind != 'ppo':
        d['amp_obs'] = torch.randn(B, amp_dim, generator=g)
        d['amp_obs_replay'] = torch.randn(B, amp_dim, generator=g) * 1.2 - 0.1
        d['amp_obs_demo'] = torch.randn(B, amp_dim, generator=g) * 0.8 + 0.3
        d['rand_action_mask'] = (torch.rand(B, generator=g) < 0.85).float()
    if kind == 'ase':
        d['ase_latents'] = z
    return d, new_z


def rollout_script(fx=None, g=None, N=16, H=8):
    """Normaliser statistics and the per-step observation / AMP tensors of the scripted env behind tests/golden/rollout_ase.pt, drawn
    in this order from one generator (seed 77).  The fixture stores everything the env draws after these.  With a fixture: its three
    tensors; else (rms, obs_t, reset_obs_t, amp_t) drawn from g."""
    if fx is not None:
        N, H = fx['N'], fx['H']
    g = g if g is not None else torch.Generator().manual_seed(77)
    rms = [(torch.randn(dim, generator=g).double() * 0.3, (0.5 + torch.rand(dim, generator=g)).double()) for dim in (253, 1, 1400)]
    obs_t = torch.randn(H + 1, N, 253, generator=g) * 1.5 + 0.3
    reset_obs_t = torch.randn(H + 1, N, 253, generator=g) * 1.5 - 0.2
    amp_t = torch.randn(H, N, 1400, generator=g)
    return dict(obs_t=obs_t, reset_obs_t=reset_obs_t, amp_t=amp_t) if fx is not None else (rms, obs_t, reset_obs_t, amp_t)


HRL_LLC_PARAM_SEED, HRL_HLC_PARAM_SEED = 31, 13


def hrl_llc_params():
    """Seeded weights of the LLC behind tests/golden/rollout_hrl.pt: the ASE network at production widths."""
    return params(O.ase_param_shapes(), seed=HRL_LLC_PARAM_SEED)


def hrl_hlc_params():
    """Seeded weights of the HLC behind tests/golden/rollout_hrl.pt (hrl_humanoid.yaml: obs 258, act 64, units [1024, 512]).  No sigma:
    the network's log-std is the config's constant."""
    p = params(O.amp_param_shapes(obs=258, act=64, amp=0, units=(1024, 512)), seed=HRL_HLC_PARAM_SEED)
    del p['sigma']
    return p


def hrl_rollout_script(fx=None, N=24, H=6, llc_steps=5):
    """Normaliser statistics and per-LLC-step env tables of the scripted env behind tests/golden/rollout_hrl.pt (K = llc_steps * H sub-steps).
    The LLC statistics are the shipped checkpoint's (tests/golden/inference_shipped_stats.pt); the HLC observation statistics extend them by
    the 5 task dims.  Observations lie around the LLC mean with 1.5 x its standard deviations, some rows 40 standard deviations off; AMP
    observations likewise, plus rows pushed 40 standard deviations along the sign of the discriminator's input gradient, whose logits sit
    far beyond the 1e-4 floor of `1 - prob`.  Dones and terminations hit the first, a middle and the last sub-step of an HLC step and the
    rollout's last sub-step."""
    import os
    if fx is not None:
        N, H, llc_steps = fx['N'], fx['H'], fx['llc_steps']
    K = H * llc_steps
    golden = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')
    shipped = torch.load(os.path.join(golden, 'inference_shipped_stats.pt'), weights_only=False)['rms']
    llc_rms = {k: {kk: vv.clone() for kk, vv in v.items()} for k, v in shipped.items()}
    g = torch.Generator().manual_seed(91)
    m, sd = llc_rms['running_mean_std']['running_mean'].float(), llc_rms['running_mean_std']['running_var'].float().sqrt()
    ma, sda = llc_rms['amp_input_mean_std']['running_mean'].float(), llc_rms['amp_input_mean_std']['running_var'].float().sqrt()

    def obs_rows(*shape):
        return torch.cat([m + 1.5 * sd * torch.randn(*shape, 253, generator=g), torch.randn(*shape, 5, generator=g) * 2.0], dim=-1)
    hlc_rms = {'running_mean_std': {'running_mean': torch.cat([llc_rms['running_mean_std']['running_mean'], 0.3 * torch.randn(5, generator=g).double()]),
                                    'running_var': torch.cat([llc_rms['running_mean_std']['running_var'], (0.5 + torch.rand(5, generator=g)).double() * 4.0]),
                                    'count': torch.tensor(1000.0, dtype=torch.float64)},
               'reward_mean_std': {'running_mean': 0.3 * torch.randn(1, generator=g).double(), 'running_var': (0.5 + torch.rand(1, generator=g)).double(),
                                   'count': torch.tensor(1000.0, dtype=torch.float64)}}
    obs_t = obs_rows(K + 1, N)
    reset_obs_t = obs_rows(H + 1, N)
    # LLC inputs (sub-steps 1..4 of an HLC step read the previous sub-step's observation) 40 standard deviations off the mean
    obs_t[3, 5, :253] = m + 40.0 * sd
    obs_t[7, 6, :253] = m - 40.0 * sd
    obs_t[K - 1, 7, :253] = m + 40.0 * sd * torch.sign(torch.randn(253, generator=g))
    amp_t = ma + 1.5 * sda * torch.randn(K, N, 1400, generator=g)
    rew_t = torch.rand(K, N, generator=g)
    dones_t = (torch.rand(K, N, generator=g) < 0.04).to(torch.uint8)
    term_t = (dones_t.bool() & (torch.rand(K, N, generator=g) < 0.5)).to(torch.uint8)
    # a done on the first (env 1), a middle (env 2) and the last (env 3) sub-step of an HLC step, a termination inside an HLC step (env 4),
    # a done on the rollout's last sub-step (env 0)
    dones_t[0 * llc_steps + 0, 1] = 1
    dones_t[1 * llc_steps + 2, 2] = 1
    dones_t[2 * llc_steps + llc_steps - 1, 3] = 1
    dones_t[3 * llc_steps + 1, 4] = 1; term_t[3 * llc_steps + 1, 4] = 1
    dones_t[K - 1, 0] = 1
    # discriminator rows on the 1e-4 floor: normalised input at the +-5 clamp along the sign of d logit / d input at the mean
    P = hrl_llc_params()
    x = torch.zeros(1, 1400, dtype=torch.float64, requires_grad=True)
    O.eval_disc({k: v.double() for k, v in P.items()}, x).sum().backward()
    s = torch.sign(x.grad[0]).float()
    amp_t[2, 9] = ma + 40.0 * sda * s
    amp_t[K - 3, 10] = ma + 40.0 * sda * s
    out = dict(obs_t=obs_t, reset_obs_t=reset_obs_t, amp_t=amp_t, rew_t=rew_t, dones_t=dones_t, term_t=term_t, llc_rms=llc_rms, hlc_rms=hlc_rms)
    if fx is None:
        out.update(N=N, H=H, llc_steps=llc_steps)
    return out


def shipped_stats_inputs(fx, n=96):
    """Inputs of tests/golden/inference_shipped_stats.pt: observations and AMP observations around the stored (shipped) normaliser
    statistics with 1.5 x their standard deviations, plus rows at the mean, 40 standard deviations away and just off the mean; unit
    latents."""
    g = torch.Generator().manual_seed(77)

    def around(st):
        m, sd = st['running_mean'].float(), st['running_var'].float().sqrt()
        x = m + 1.5 * sd * torch.randn(n, m.numel(), generator=g)
        x[0] = m; x[1] = m + 40.0 * sd; x[2] = m - 40.0 * sd; x[3] = m + 1e-3 * torch.randn(m.numel(), generator=g)
        return x
    obs, amp = around(fx['rms']['running_mean_std']), around(fx['rms']['amp_input_mean_std'])
    return dict(obs=obs, amp=amp, z=F.normalize(torch.randn(n, 64, generator=g), dim=-1))
