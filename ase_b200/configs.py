"""Hyper-parameters of the reference's shipped training configs, restated as plain dicts so benchmarks and tests
run where /root/reference is absent.  Values: ase/data/cfg/train/rlg/{ase,amp,hrl}_humanoid.yaml and
ase/data/cfg/humanoid_ase_sword_shield_getup.yaml (numEnvs 4096, line 3)."""
import copy

ASE_HUMANOID = {   # ase_humanoid.yaml
    'net_params': {
        'separate': True,
        'space': {'continuous': {'mu_activation': 'None', 'sigma_activation': 'None', 'mu_init': {'name': 'default'},
                                 'sigma_init': {'name': 'const_initializer', 'val': -2.9}, 'fixed_sigma': True, 'learn_sigma': False}},
        'mlp': {'units': [1024, 1024, 512], 'activation': 'relu'},
        'disc': {'units': [1024, 1024, 512], 'activation': 'relu'},
        'enc': {'units': [1024, 512], 'activation': 'relu', 'separate': False},
    },
    'name': 'Humanoid', 'env_name': 'rlgpu', 'multi_gpu': False, 'ppo': True, 'mixed_precision': False,
    'normalize_input': True, 'normalize_value': True, 'reward_shaper': {'scale_value': 1}, 'normalize_advantage': True,
    'gamma': 0.99, 'tau': 0.95, 'learning_rate': 2e-5, 'lr_schedule': 'constant', 'max_epochs': 100000,
    'save_frequency': 50, 'print_stats': True, 'grad_norm': 1.0, 'entropy_coef': 0.0, 'truncate_grads': False,
    'e_clip': 0.2, 'horizon_length': 32, 'minibatch_size': 16384, 'mini_epochs': 6, 'critic_coef': 5, 'clip_value': False,
    'bounds_loss_coef': 10, 'amp_obs_demo_buffer_size': 200000, 'amp_replay_buffer_size': 200000, 'amp_replay_keep_prob': 0.01,
    'amp_batch_size': 512, 'amp_minibatch_size': 4096, 'disc_coef': 5, 'disc_logit_reg': 0.01, 'disc_grad_penalty': 5,
    'disc_reward_scale': 2, 'disc_weight_decay': 0.0001, 'normalize_amp_input': True, 'enable_eps_greedy': True,
    'latent_dim': 64, 'latent_steps_min': 1, 'latent_steps_max': 150, 'amp_diversity_bonus': 0.01, 'amp_diversity_tar': 1.0,
    'enc_coef': 5, 'enc_weight_decay': 0.0, 'enc_reward_scale': 1, 'enc_grad_penalty': 0,
    'task_reward_w': 0.0, 'disc_reward_w': 0.5, 'enc_reward_w': 0.5,
}

AMP_HUMANOID = {   # amp_humanoid.yaml
    'net_params': {
        'separate': True,
        'space': {'continuous': {'mu_activation': 'None', 'sigma_activation': 'None', 'mu_init': {'name': 'default'},
                                 'sigma_init': {'name': 'const_initializer', 'val': -2.9}, 'fixed_sigma': True, 'learn_sigma': False}},
        'mlp': {'units': [1024, 512], 'activation': 'relu'},
        'disc': {'units': [1024, 512], 'activation': 'relu'},
    },
    'name': 'Humanoid', 'env_name': 'rlgpu', 'multi_gpu': False, 'ppo': True, 'mixed_precision': False,
    'normalize_input': True, 'normalize_value': True, 'reward_shaper': {'scale_value': 1}, 'normalize_advantage': True,
    'gamma': 0.99, 'tau': 0.95, 'learning_rate': 2e-5, 'lr_schedule': 'constant', 'max_epochs': 100000,
    'save_frequency': 50, 'print_stats': True, 'grad_norm': 1.0, 'entropy_coef': 0.0, 'truncate_grads': False,
    'e_clip': 0.2, 'horizon_length': 32, 'minibatch_size': 16384, 'mini_epochs': 6, 'critic_coef': 5, 'clip_value': False,
    'bounds_loss_coef': 10, 'amp_obs_demo_buffer_size': 200000, 'amp_replay_buffer_size': 200000, 'amp_replay_keep_prob': 0.01,
    'amp_batch_size': 512, 'amp_minibatch_size': 4096, 'disc_coef': 5, 'disc_logit_reg': 0.01, 'disc_grad_penalty': 5,
    'disc_reward_scale': 2, 'disc_weight_decay': 0.0001, 'normalize_amp_input': True, 'enable_eps_greedy': False,
    'task_reward_w': 0.0, 'disc_reward_w': 1.0,
}


HRL_HUMANOID = {   # hrl_humanoid.yaml (HumanoidHeading / Location / Reach / Strike task training over a frozen LLC)
    'net_params': {
        'separate': True,
        # the HLC explores wider than the LLC: log-std -2.3 (hrl_humanoid.yaml; the shipped HLC checkpoints store a2c_network.sigma = -2.3)
        'space': {'continuous': {'mu_activation': 'None', 'sigma_activation': 'None', 'mu_init': {'name': 'default'},
                                 'sigma_init': {'name': 'const_initializer', 'val': -2.3}, 'fixed_sigma': True, 'learn_sigma': False}},
        'mlp': {'units': [1024, 512], 'activation': 'relu'},
    },
    'llc_net_params': ASE_HUMANOID['net_params'], 'latent_dim': 64,
    'name': 'Humanoid', 'env_name': 'rlgpu', 'multi_gpu': False, 'ppo': True, 'mixed_precision': False,
    'normalize_input': True, 'normalize_value': True, 'reward_shaper': {'scale_value': 1}, 'normalize_advantage': True,
    'gamma': 0.99, 'tau': 0.95, 'learning_rate': 2e-5, 'lr_schedule': 'constant', 'max_epochs': 100000,
    'save_frequency': 50, 'print_stats': True, 'grad_norm': 1.0, 'entropy_coef': 0.0, 'truncate_grads': False,
    'e_clip': 0.2, 'horizon_length': 32, 'minibatch_size': 16384, 'mini_epochs': 6, 'critic_coef': 5, 'clip_value': False,
    'bounds_loss_coef': 10, 'task_reward_w': 0.9, 'disc_reward_w': 0.1, 'llc_steps': 5,
}


def make(name, **overrides):
    cfg = copy.deepcopy({'ase': ASE_HUMANOID, 'amp': AMP_HUMANOID, 'hrl': HRL_HUMANOID}[name])
    cfg.update(overrides)
    return cfg
