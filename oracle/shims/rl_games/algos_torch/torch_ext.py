"""[recollection of rl_games 1.1.4 algos_torch/torch_ext.py] (subset)."""
import numpy as np
import torch
import torch.nn as nn

numpy_to_torch_dtype_dict = {
    np.dtype('bool'): torch.bool, np.dtype('uint8'): torch.uint8, np.dtype('int8'): torch.int8,
    np.dtype('int16'): torch.int16, np.dtype('int32'): torch.int32, np.dtype('int64'): torch.int64,
    np.dtype('float16'): torch.float16, np.dtype('float32'): torch.float32, np.dtype('float64'): torch.float32,
}


def load_checkpoint(filename):
    print("=> loading checkpoint '{}'".format(filename))
    state = torch.load(filename, map_location='cpu', weights_only=False)
    return state


def policy_kl(p0_mu, p0_sigma, p1_mu, p1_sigma, reduce=True):
    c1 = torch.log(p1_sigma / p0_sigma + 1e-5)
    c2 = (p0_sigma ** 2 + (p1_mu - p0_mu) ** 2) / (2.0 * (p1_sigma ** 2 + 1e-5))
    c3 = -1.0 / 2.0
    kl = c1 + c2 + c3
    kl = kl.sum(dim=-1)  # returning mean between all steps of sum between all actions
    if reduce:
        return kl.mean()
    else:
        return kl


def mean_mask(input, mask, sum_mask):
    return (input * mask).sum() / sum_mask


def shape_whc_to_cwh(shape):
    if len(shape) == 3:
        return (shape[2], shape[0], shape[1])
    return shape


def mean_list(val):
    return torch.mean(torch.stack(val))


def get_mean_var_with_masks(values, masks):
    sum_mask = masks.sum()
    values_mask = values * masks
    values_mean = values_mask.sum() / sum_mask
    min_sqr = (((values_mask) ** 2) / sum_mask).sum() - ((values_mask / sum_mask).sum()) ** 2
    values_var = min_sqr * sum_mask / (sum_mask - 1)
    return values_mean, values_var


def get_mean_std_with_masks(values, masks):
    mean, var = get_mean_var_with_masks(values, masks)
    return mean, torch.sqrt(var)


def normalization_with_masks(values, masks):
    values_mean, values_std = get_mean_std_with_masks(values, masks)
    normalized_values = (values - values_mean) / (values_std + 1e-8)
    return normalized_values


class AverageMeter(nn.Module):
    def __init__(self, in_shape, max_size):
        super(AverageMeter, self).__init__()
        self.max_size = max_size
        self.current_size = 0
        self.register_buffer("mean", torch.zeros(in_shape, dtype=torch.float32))

    def update(self, values):
        size = values.size()[0]
        if size == 0:
            return
        new_mean = torch.mean(values.float(), dim=0)
        size = np.clip(size, 0, self.max_size)
        old_size = min(self.max_size - size, self.current_size)
        size_sum = old_size + size
        self.current_size = size_sum
        self.mean = (self.mean * old_size + new_mean * size) / size_sum

    def clear(self):
        self.current_size = 0
        self.mean.fill_(0)

    def __len__(self):
        return self.current_size

    def get_mean(self):
        return self.mean.squeeze(0).cpu().numpy()
