"""Inputs of the TartanVOMatcher fixtures (tests/golden/tartanvo_flow_*.pt): two left images per case from the exactly
rounded generator of the Vanilla fixtures (plain_cases.plain_frontend_inputs: frame t1 = its t2.L, frame t2 = its t2.R, a
shifted copy of the same texture), wrapped as frames with the fields TartanVOMatcher.forward reads."""
from __future__ import annotations

import hashlib
from types import SimpleNamespace

import torch

from tests.golden import plain_cases

CASES = {
    "small": (200, 264),         # margins 4 / 4; pyramid down to 3 x 4
    "kitti": (376, 780),         # KITTI after SmartResizeFrame; margins 28 / 6
    "tartanair": (480, 640),     # width margin 0: the reference's mask is all False
    "euroc": (480, 752),         # margins 16 / 24
}


def frame(image: torch.Tensor) -> SimpleNamespace:
    H, W = image.shape[-2:]
    fx = 320.0
    K = torch.tensor([[[fx, 0.0, W / 2], [0.0, fx, H / 2], [0.0, 0.0, 1.0]]])
    return SimpleNamespace(imageL=image, height=H, width=W, K=K, fx=fx, fy=fx, cx=W / 2, cy=H / 2, frame_baseline=0.25,
                           baseline=torch.tensor([0.25]))


def frames(name: str) -> tuple[SimpleNamespace, SimpleNamespace]:
    H, W = CASES[name]
    _, l2, r2 = plain_cases.plain_frontend_inputs(H, W)
    return frame(l2), frame(r2)


def sha(*tensors: torch.Tensor) -> str:
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.detach().contiguous().float().numpy().tobytes())
    return h.hexdigest()
