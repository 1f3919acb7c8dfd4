"""Activation modules of the reference's colour MLP (lib/act.py), for DirectMPIGO's act_type='gauss'."""
import torch
import torch.nn as nn


class GaussianActivation(nn.Module):
    """exp(-x^2 / (2 a^2)).  ``a`` is a one-element parameter (state_dict key ``a``), frozen unless ``trainable``.
    The fused marcher reads ``a`` when it builds its device scene (k4_scene_desc.rgbnet_act_param)."""

    def __init__(self, a=1., trainable=False):
        super().__init__()
        self.a = nn.Parameter(torch.full((1,), float(a)), requires_grad=trainable)

    def forward(self, x):
        # the reference's expression, in the same order: the fp32 marcher mode reproduces it operation by operation
        return torch.exp(-x ** 2 / (2 * self.a ** 2))
