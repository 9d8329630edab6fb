"""TartanVO pose network of TartanMotionNet (Module/MotionModel.py:89-116) on the device.

VOFlowRes(config=1, stereo=True, down_scale=True, intrinsic=True) (Module/Network/TartanVOStereo/FlowPoseNet.py:45-165) —
the only part of StereoVONet that `TartanMotionNet.predict` runs — fed by TartanStereoVOMotion.inference
(StereoVO_Interface.py:158-194).

    input builder   macvo_posenet_input: flow / depth maps -> channels 0..2 of the 5 x 112 x 160 input; channels 3..4
                    (the intrinsics layer) depend on the image size and K only and are computed once (`intrinsic_layer`)
    firstconv, layer1, layer2   56x80, 28x40, 14x20 output pixels: cuDNN through torch (plain convolutions)
    layer3 .. layer5, fc1       7x10 pixels and smaller: weight-streaming GEMVs, macvo_posenet_conv (one launch per layer)
    fc2, fc3, x pose_norm, pose composition   macvo_posenet_head (one CTA)
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import ops

# (name, output channels, blocks) of VOFlowRes config 1 with down_scale (layer0 / layer0_2 absent)
STAGES = (("layer1", 64, 3), ("layer2", 128, 4), ("layer3", 128, 6), ("layer4", 256, 7), ("layer5", 256, 3))
DEVICE_STAGES = ("layer3", "layer4", "layer5")          # output 7x10 pixels or smaller -> macvo_posenet_conv
POSE_NORM = (0.13, 0.13, 0.13, 0.013, 0.013, 0.013)       # TartanStereoVONetInterface.pose_norm
CKPT_PREFIX = "module.flowPoseNet."


def state_dict_shapes() -> dict[str, tuple[int, ...]]:
    """tensor name -> shape of VOFlowRes(config=1, stereo=True, down_scale=True, intrinsic=True)"""
    s: dict[str, tuple[int, ...]] = {}
    cin = 5
    for i in range(3):
        s[f"firstconv.{i}.0.weight"], s[f"firstconv.{i}.0.bias"] = (32, cin, 3, 3), (32,)
        cin = 32
    for name, planes, blocks in STAGES:
        for b in range(blocks):
            s[f"{name}.{b}.conv1.0.weight"], s[f"{name}.{b}.conv1.0.bias"] = (planes, cin, 3, 3), (planes,)
            s[f"{name}.{b}.conv2.weight"], s[f"{name}.{b}.conv2.bias"] = (planes, planes, 3, 3), (planes,)
            if b == 0:      # every stage strides by 2 -> a 1x1 stride-2 downsample
                s[f"{name}.0.downsample.weight"], s[f"{name}.0.downsample.bias"] = (planes, cin, 1, 1), (planes,)
            cin = planes
    for head in ("trans", "rot"):
        s[f"voflow_{head}.0.0.weight"], s[f"voflow_{head}.0.0.bias"] = (128, 256 * 6), (128,)
        s[f"voflow_{head}.1.0.weight"], s[f"voflow_{head}.1.0.bias"] = (32, 128), (32,)
        s[f"voflow_{head}.2.weight"], s[f"voflow_{head}.2.bias"] = (3, 32), (3,)
    return s


def synthetic_posenet_state_dict(seed: int = 0) -> dict[str, torch.Tensor]:
    """Deterministic stand-in weights keyed like VOFlowRes's state_dict (no checkpoint exists offline). The residual
    branch's second convolution is scaled down (0.3 / sqrt(fan_in)) so that 25 residual blocks neither grow the activations
    geometrically nor let ReLU silence them; the rest is He-scaled."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, shape in state_dict_shapes().items():
        if name.endswith("bias"):
            out[name] = torch.randn(shape, generator=g) * 0.02
            continue
        fan_in = int(torch.tensor(shape[1:]).prod())
        gain = 0.3 if ".conv2." in name else (1.0 if "downsample" in name or name.startswith("voflow_") and ".2." in name
                                               else 2.0 ** 0.5)
        out[name] = torch.randn(shape, generator=g) * (gain / fan_in ** 0.5)
    return out


def load_checkpoint(path: str) -> dict[str, torch.Tensor]:
    """A TartanVO StereoVONet checkpoint -> the flowPoseNet tensors (`module.` stripped like
    TartanStereoVONetInterface.loadWeight, StereoVO_Interface.py:56-62). Missing tensors raise."""
    raw = torch.load(path, map_location="cpu", weights_only=True)
    sd = {k[len(CKPT_PREFIX):]: v for k, v in raw.items() if k.startswith(CKPT_PREFIX)}
    shapes = state_dict_shapes()
    missing = [k for k in shapes if k not in sd]
    if missing:
        raise KeyError(f"{path}: checkpoint lacks {len(missing)} pose-network tensors, e.g. {CKPT_PREFIX}{missing[0]}")
    for k, shp in shapes.items():
        if tuple(sd[k].shape) != shp:
            raise ValueError(f"{path}: {CKPT_PREFIX}{k} has shape {tuple(sd[k].shape)}, expected {shp}")
    return {k: sd[k] for k in shapes}


def crop_resize(x: torch.Tensor) -> torch.Tensor:
    """TartanStereoVOMotion.cropAndResize to 112 x 160: centre crop (centerCropTo keeps an extra row / column when the
    margin is odd), then bilinear align_corners=True."""
    H, W = x.shape[-2:]
    s = min(H // ops.POSENET_H, W // ops.POSENET_W)
    my, mx = (H - ops.POSENET_H * s) // 2, (W - ops.POSENET_W * s) // 2
    x = x[..., my:H - my, mx:W - mx]
    return F.interpolate(x, size=(ops.POSENET_H, ops.POSENET_W), mode="bilinear", align_corners=True)


def intrinsic_layer(height: int, width: int, fx: float, fy: float, cx: float, cy: float, device) -> torch.Tensor:
    """channels 3..4 of the network input, (1,2,112,160). The reference calls make_device_intrinsic_layer(w, h, ...) with
    (height, width) (StereoVO_Interface.py:176-178, Utility.py:13-18): channel 0 = (x - cy + 0.5) / fy and
    channel 1 = (y - cx + 0.5) / fx — reproduced, not fixed, because the trained weights expect it."""
    ys, xs = torch.meshgrid(torch.arange(height, device=device), torch.arange(width, device=device), indexing="ij")
    a = (ys.float() - cx + 0.5) / fx
    b = (xs.float() - cy + 0.5) / fy
    layer = torch.stack((b, a), dim=-1).unsqueeze(0).permute(0, 3, 1, 2)
    return crop_resize(layer)


class PoseNet:
    """Weights on the device: firstconv / layer1 / layer2 as torch tensors (cuDNN), layer3..layer5 and fc1 as
    macvo_posenet_conv slabs, fc2 / fc3 / pose_norm as the head kernel's blob."""

    def __init__(self, sd: dict[str, torch.Tensor], device):
        self.device = torch.device(device)
        dev = lambda t: t.detach().to(device=self.device, dtype=torch.float32).contiguous()
        self.first = [(dev(sd[f"firstconv.{i}.0.weight"]), dev(sd[f"firstconv.{i}.0.bias"])) for i in range(3)]
        self.stages = []        # per stage: list of blocks {conv1, conv2, downsample}: (weight or slabs, bias, co_tile)
        for name, _, blocks in STAGES:
            on_dev = name in DEVICE_STAGES
            blk = []
            for b in range(blocks):
                layers = {}
                for key, wname in (("conv1", f"{name}.{b}.conv1.0"), ("conv2", f"{name}.{b}.conv2"),
                                   ("downsample", f"{name}.{b}.downsample")):
                    if f"{wname}.weight" not in sd:
                        continue
                    w, bias = sd[f"{wname}.weight"], dev(sd[f"{wname}.bias"])
                    if on_dev:
                        packed, ct = ops.pack_posenet_conv(w)
                        layers[key] = (packed.to(self.device), bias, ct)
                    else:
                        layers[key] = (dev(w), bias, 0)
                blk.append(layers)
            self.stages.append((name, on_dev, blk))
        # fc1 of both heads as one N = 256 GEMV over the flattened (256, 2, 3) map
        w1 = torch.cat([sd["voflow_trans.0.0.weight"], sd["voflow_rot.0.0.weight"]])
        packed, ct = ops.pack_posenet_conv(w1)
        self.fc1 = (packed.to(self.device), dev(torch.cat([sd["voflow_trans.0.0.bias"], sd["voflow_rot.0.0.bias"]])), ct)
        parts = []
        for layer in ("1.0.", "2."):
            for head in ("trans", "rot"):
                parts += [sd[f"voflow_{head}.{layer}weight"].reshape(-1), sd[f"voflow_{head}.{layer}bias"].reshape(-1)]
        parts.append(torch.tensor(POSE_NORM))
        self.head_blob = dev(torch.cat([p.float() for p in parts]))
        if self.head_blob.numel() != ops.posenet_head_floats():
            raise ValueError("pose-network head blob does not match macvo_posenet_head's layout")

    def body(self, inp: torch.Tensor) -> torch.Tensor:
        """(1,5,112,160) network input -> fc1 output (256,) = [trans 128 | rot 128] after ReLU"""
        x = inp
        for i, (w, b) in enumerate(self.first):
            x = F.relu(F.conv2d(x, w, b, stride=2 if i == 0 else 1, padding=1), inplace=True)
        for _, on_dev, blocks in self.stages:
            for b, layers in enumerate(blocks):
                stride = 2 if b == 0 else 1
                if on_dev:
                    ds = layers.get("downsample")
                    res = ops.posenet_conv(x, ds[0], ds[2], ds[1], 1, 2, 0) if ds is not None else x
                    w, bias, ct = layers["conv1"]
                    h = ops.posenet_conv(x, w, ct, bias, 3, stride, 1, relu=True)
                    w, bias, ct = layers["conv2"]
                    x = ops.posenet_conv(h, w, ct, bias, 3, 1, 1, resid=res, relu=True)
                else:       # BasicBlock.forward (FlowPoseNet.py:35-43)
                    w, bias, _ = layers["conv1"]
                    h = F.relu(F.conv2d(x, w, bias, stride=stride, padding=1), inplace=True)
                    w, bias, _ = layers["conv2"]
                    h = F.conv2d(h, w, bias, stride=1, padding=1)
                    ds = layers.get("downsample")
                    h += F.conv2d(x, ds[0], ds[1], stride=2) if ds is not None else x
                    x = F.relu(h, inplace=True)
        w, bias, ct = self.fc1
        return ops.posenet_conv(x.reshape(-1, 1, 1), w, ct, bias, 1, 1, 0, relu=True).reshape(-1)
