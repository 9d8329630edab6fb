"""Seeded inputs of the pose-network fixtures (tests/golden/posenet_*.pt), built from exactly rounded operations only
(randn / rand scaled by powers of two, table look-ups), so that every torch build regenerates the same bits; each
fixture stores the sha256 of its inputs."""
from __future__ import annotations

import torch

from tests.golden.cases import _lognormal_like, sha  # noqa: F401  (sha re-exported for the tests)

# name -> (H, W, fx, fy, cx, cy, baseline, seed)
CASES = {
    "480x640": (480, 640, 320.0, 310.0, 320.0, 240.0, 0.25, 11),        # cx != cy, fx != fy
    "720x1280": (720, 1280, 640.0, 640.0, 640.0, 360.0, 0.25, 12),
    "481x641": (481, 641, 321.0, 320.0, 320.5, 240.5, 0.25, 13),        # odd margins: resize from 449 x 641
    "nonfinite": (480, 640, 320.0, 320.0, 320.0, 240.0, 0.25, 14),      # NaN, +-inf, 0 and negative depth at taps
    "zerodepth": (480, 640, 320.0, 320.0, 320.0, 240.0, 0.25, 15),      # 6 x 6 blocks of zero depth -> +inf network input
}
PREV_POSE = torch.tensor([0.5, -0.25, 1.0, 0.125, -0.25, 0.375, 0.875])   # [t, q_xyzw], not normalised on purpose
SPECIALS = (float("nan"), float("inf"), float("-inf"), 0.0, -2.0)


def special_taps(H: int, W: int) -> list[tuple[int, int, float, bool]]:
    """(row, col, value, whole 2x2 block) positions in the full-resolution depth map of the "nonfinite" case"""
    out = []
    for i, v in enumerate(SPECIALS):
        r, c = 40 + 80 * i, 50 + 110 * i
        out.append((r, c, v, True))           # 2 x 2 block of the special value
        out.append((r + 20, c + 40, v, False))  # single tap: mixes with finite neighbours (inf * 0 -> NaN -> 0)
    return out


def posenet_inputs(name: str) -> dict:
    H, W, fx, fy, cx, cy, bl, seed = CASES[name]
    g = torch.Generator().manual_seed(seed)
    flow = torch.randn(1, 2, H, W, generator=g) * 4.0
    depth = _lognormal_like((1, 1, H, W), g, 2.0)
    if name == "zerodepth":      # the output grid steps ~4 px: some output pixel has all four taps inside each block
        for i in range(4):
            depth[0, 0, 60 + 90 * i:66 + 90 * i, 70 + 130 * i:76 + 130 * i] = 0.0
    if name == "nonfinite":
        for r, c, v, block in special_taps(H, W):
            if block:
                depth[0, 0, r:r + 2, c:c + 2] = v
            else:
                depth[0, 0, r, c] = v
    return {"flow": flow, "depth": depth, "H": H, "W": W, "fx": fx, "fy": fy, "cx": cx, "cy": cy, "baseline": bl,
            "prev_pose": PREV_POSE.clone()}
