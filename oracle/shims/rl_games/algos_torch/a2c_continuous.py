"""[recollection of rl_games 1.1.4 algos_torch/a2c_continuous.py] -- only what CommonAgent inherits."""
from rl_games.algos_torch import torch_ext
from rl_games.common import a2c_common


class A2CAgent(a2c_common.ContinuousA2CBase):
    def __init__(self, base_name, config):
        raise NotImplementedError("CommonAgent.__init__ calls A2CBase.__init__ directly (common_agent.py:27)")

    def update_epoch(self):
        self.epoch_num += 1
        return self.epoch_num

    def train_actor_critic(self, input_dict):
        self.calc_gradients(input_dict)
        return self.train_result

    def restore(self, fn):
        checkpoint = torch_ext.load_checkpoint(fn)
        self.set_full_state_weights(checkpoint)

    def save(self, fn):
        pass
