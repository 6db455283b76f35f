"""[recollection of rl_games 1.1.4 common/env_configurations.py] (subset): the env registry BasePlayer.create_env reads and get_env_info."""
configurations = {}


def register(name, config):
    configurations[name] = config


def get_env_info(env):
    result_shapes = {}
    result_shapes['observation_space'] = env.observation_space
    result_shapes['action_space'] = env.action_space
    result_shapes['agents'] = 1
    result_shapes['value_size'] = 1
    if hasattr(env, "get_number_of_agents"):
        result_shapes['agents'] = env.get_number_of_agents()
    if hasattr(env, "value_size"):
        result_shapes['value_size'] = env.value_size
    return result_shapes
