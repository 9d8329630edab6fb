"""CPU oracle of the TartanMotionNet prediction (Module/MotionModel.py:101-116): the pose network's input builder
(TartanStereoVOMotion.inference, StereoVO_Interface.py:158-194), the VOFlowRes forward pass (FlowPoseNet.py:35-43,
140-165; config 1, stereo, down_scale, intrinsic) and the composition prev_pose @ se3(motion).Exp() through the pypose
shim. Restated operation by operation with torch CPU ops; the weights are a state dict keyed like VOFlowRes."""
from __future__ import annotations

import os
import sys

import torch
import torch.nn.functional as F

_SHIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pypose_shim")

STAGES = (("layer1", 3), ("layer2", 4), ("layer3", 6), ("layer4", 7), ("layer5", 3))
POSE_NORM = (0.13, 0.13, 0.13, 0.013, 0.013, 0.013)
OUT_H, OUT_W = 112, 160


def crop_resize(x: torch.Tensor) -> torch.Tensor:
    H, W = x.shape[-2:]
    s = min(int(H / OUT_H), int(W / OUT_W))
    th, tw = OUT_H * s, OUT_W * s
    my, mx = (H - th) // 2, (W - tw) // 2            # centerCropTo: narrow(margin, size - 2 * margin)
    x = x.narrow(-2, my, H - 2 * my).narrow(-1, mx, W - 2 * mx)
    return F.interpolate(x, size=(OUT_H, OUT_W), mode="bilinear", align_corners=True)


def network_input(flow: torch.Tensor, depth: torch.Tensor, height: int, width: int, fx: float, fy: float, cx: float,
                  cy: float, baseline: float) -> torch.Tensor:
    """flow (1,2,H,W), depth (1,1,H,W) -> (1,5,112,160)"""
    ys, xs = torch.meshgrid(torch.arange(height), torch.arange(width), indexing="ij")
    intr = torch.stack(((xs.float() - cy + 0.5) / fy, (ys.float() - cx + 0.5) / fx), dim=-1).unsqueeze(0).permute(0, 3, 1, 2)
    return torch.cat((flow_depth_channels(flow, depth, baseline * fx), crop_resize(intr)), dim=1)


def flow_depth_channels(flow: torch.Tensor, depth: torch.Tensor, bl_fx: float) -> torch.Tensor:
    """channels 0..2 of the network input, (1,3,112,160)"""
    depth_r = crop_resize(depth)
    flow_r = crop_resize(flow) * 0.05
    stereo = bl_fx / depth_r
    stereo = torch.nan_to_num(stereo * 0.02, nan=0.0).clamp(min=0.0)
    depth_r = stereo / bl_fx / float(0.02 * 0.25)
    return torch.cat((flow_r, depth_r), dim=1)


def forward(sd: dict[str, torch.Tensor], x: torch.Tensor) -> dict[str, torch.Tensor]:
    """VOFlowRes forward in the dtype of x -> {"fc1": (256,) [trans | rot] after ReLU, "pose": (6,) before pose_norm}"""
    w = {k: v.to(x.dtype) for k, v in sd.items()}
    for i in range(3):
        x = F.relu(F.conv2d(x, w[f"firstconv.{i}.0.weight"], w[f"firstconv.{i}.0.bias"], stride=2 if i == 0 else 1, padding=1))
    for name, blocks in STAGES:
        for b in range(blocks):
            p = f"{name}.{b}."
            stride = 2 if b == 0 else 1
            out = F.relu(F.conv2d(x, w[p + "conv1.0.weight"], w[p + "conv1.0.bias"], stride=stride, padding=1))
            out = F.conv2d(out, w[p + "conv2.weight"], w[p + "conv2.bias"], stride=1, padding=1)
            res = F.conv2d(x, w[p + "downsample.weight"], w[p + "downsample.bias"], stride=2) if b == 0 else x
            x = F.relu(out + res)
    x = x.reshape(1, -1)
    h = {head: F.relu(F.linear(x, w[f"voflow_{head}.0.0.weight"], w[f"voflow_{head}.0.0.bias"])) for head in ("trans", "rot")}
    out = []
    for head in ("trans", "rot"):
        y = F.relu(F.linear(h[head], w[f"voflow_{head}.1.0.weight"], w[f"voflow_{head}.1.0.bias"]))
        out.append(F.linear(y, w[f"voflow_{head}.2.weight"], w[f"voflow_{head}.2.bias"]))
    return {"fc1": torch.cat([h["trans"], h["rot"]], dim=1).reshape(-1), "pose": torch.cat(out, dim=1).reshape(-1)}


def motion(pose: torch.Tensor) -> torch.Tensor:
    return pose * torch.tensor(POSE_NORM, dtype=pose.dtype)


def compose(prev_pose: torch.Tensor, motion_se3: torch.Tensor) -> torch.Tensor:
    """prev_pose @ pp.se3(motion).Exp() (7,) in the dtype of the inputs, with the pypose shim"""
    if _SHIM not in sys.path:
        sys.path.insert(0, _SHIM)
    import pypose as pp
    return (pp.SE3(prev_pose) @ pp.se3(motion_se3).Exp()).tensor()
