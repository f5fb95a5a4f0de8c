"""vima_b200: the VIMA policy forward pass on H100 (sm_90a) kernels behind the reference's `vima` module surface."""
import os

import torch

from .engine import get_precision, refresh_weights, set_precision
from .nn.action import ActionSampler
from .nn.xattn_gpt import SwappedEpisode
from .policy import VIMAFlamingoPolicy, VIMAGatoPolicy, VIMAGPTPolicy, VIMAPolicy

__all__ = ["VIMAPolicy", "VIMAGatoPolicy", "VIMAGPTPolicy", "VIMAFlamingoPolicy", "create_policy_from_ckpt", "set_precision", "get_precision", "refresh_weights", "ActionSampler", "SwappedEpisode"]


def create_policy_from_ckpt(ckpt_path, device):
    """Reference: /root/reference/vima/__init__.py:7-16 -- {"cfg": kwargs, "state_dict": {"policy.<key>": tensor}}."""
    assert os.path.exists(ckpt_path), "Checkpoint path does not exist"
    ckpt = torch.load(ckpt_path, map_location=device)
    policy = VIMAPolicy(**ckpt["cfg"])
    policy.load_state_dict({k.replace("policy.", ""): v for k, v in ckpt["state_dict"].items()}, strict=True)
    policy.to(device)
    policy.eval()
    return policy
