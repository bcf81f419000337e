"""ORACLE / TEST INFRASTRUCTURE ONLY. Minimal stand-in for the un-vendored dependency named by the
package path (mmcv-full==1.5.3 / mmdet==2.25.0, environment.yml:27-28); restates only the
symbols imported at team_code_transfuser/model.py:20-30. parity unpinned (source absent)."""
import math
from torch import nn


def bias_init_with_prob(prior_prob):
    """mmcv.cnn.bias_init_with_prob: bias such that sigmoid(bias) == prior_prob."""
    return float(-math.log((1 - prior_prob) / prior_prob))


def normal_init(module, mean=0, std=1, bias=0):
    if hasattr(module, 'weight') and module.weight is not None:
        nn.init.normal_(module.weight, mean, std)
    if hasattr(module, 'bias') and module.bias is not None:
        nn.init.constant_(module.bias, bias)
