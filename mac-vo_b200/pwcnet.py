"""TartanVOMatcher's PWC-Net (Module/Frontend/Matching.py:199-230) on the device.

PWCDCNet_Adapted(md=4, uncertainty=False) (Module/Network/PWCNet/pwc/pwc_model_tartanvo.py:64-297), the forward pass that
StereoVONet.forward_flow runs (StereoVO.py:26-28); it returns flow2 at 1/4 resolution.

    feature pyramid     conv1a .. conv6b, both images as one batch of 2 (shared weights): cuDNN through torch
    per level           macvo_pwc_warp_corr: warp(f2, scale * up_flow) + correlation + LeakyReLU, written straight into
                        the level's dense-block buffer (replaces torch.cat((corr, feat_low1, up_flow, up_feat)))
    dense decoders      conv{l}_0 .. conv{l}_4, predict_flow{l}, deconv{l} / upfeat{l}: cuDNN
    context network     dc_conv1 .. dc_conv7 (dilated): cuDNN
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import ops

MD = 4
ND = (2 * MD + 1) ** 2
DENSE = (128, 128, 96, 64, 32)                          # conv{l}_0 .. conv{l}_4 output channels
DENSE_TOTAL = sum(DENSE)                                 # 448
ENCODER = (("conv1a", 3, 16, 2), ("conv1aa", 16, 16, 1), ("conv1b", 16, 16, 1),
           ("conv2a", 16, 32, 2), ("conv2aa", 32, 32, 1), ("conv2b", 32, 32, 1),
           ("conv3a", 32, 64, 2), ("conv3aa", 64, 64, 1), ("conv3b", 64, 64, 1),
           ("conv4a", 64, 96, 2), ("conv4aa", 96, 96, 1), ("conv4b", 96, 96, 1),
           ("conv5a", 96, 128, 2), ("conv5aa", 128, 128, 1), ("conv5b", 128, 128, 1),
           ("conv6aa", 128, 196, 2), ("conv6a", 196, 196, 1), ("conv6b", 196, 196, 1))
FEAT_CH = {2: 32, 3: 64, 4: 96, 5: 128, 6: 196}
WARP_SCALE = {5: 0.625, 4: 1.25, 3: 2.5, 2: 5.0}         # concate_two_layers' `scale` (pwc_model_tartanvo.py:263-272)
DILATION = (1, 2, 4, 8, 16, 1)                           # dc_conv1 .. dc_conv6
FLOW_NORM = 0.05                                         # TartanStereoVONetInterface.flow_norm
CKPT_PREFIX = "module.flowNet."


def level_input_channels(level: int) -> int:
    """channels entering level l's dense block: the cost volume, plus feat_low1, up_flow and up_feat below level 6"""
    return ND if level == 6 else ND + FEAT_CH[level] + 4


def state_dict_shapes() -> dict[str, tuple[int, ...]]:
    """tensor name -> shape of PWCDCNet_Adapted(md=4, uncertainty=False) (deconv2 exists but forward never runs it)"""
    s: dict[str, tuple[int, ...]] = {}
    for name, cin, cout, _ in ENCODER:
        s[f"{name}.0.weight"], s[f"{name}.0.bias"] = (cout, cin, 3, 3), (cout,)
    for level in (6, 5, 4, 3, 2):
        od = level_input_channels(level)
        cin = od
        for k, cout in enumerate(DENSE):
            s[f"conv{level}_{k}.0.weight"], s[f"conv{level}_{k}.0.bias"] = (cout, cin, 3, 3), (cout,)
            cin += cout
        s[f"predict_flow{level}.weight"], s[f"predict_flow{level}.bias"] = (2, cin, 3, 3), (2,)
        s[f"deconv{level}.weight"], s[f"deconv{level}.bias"] = (2, 2, 4, 4), (2,)
        if level > 2:
            s[f"upfeat{level}.weight"], s[f"upfeat{level}.bias"] = (cin, 2, 4, 4), (2,)
    cin = level_input_channels(2) + DENSE_TOTAL
    for i, cout in enumerate((128, 128, 128, 96, 64, 32)):
        s[f"dc_conv{i + 1}.0.weight"], s[f"dc_conv{i + 1}.0.bias"] = (cout, cin, 3, 3), (cout,)
        cin = cout
    s["dc_conv7.weight"], s["dc_conv7.bias"] = (2, 32, 3, 3), (2,)
    return s


# weight gains of the synthetic stand-in (see synthetic_pwc_state_dict)
SYN_FLOW_GAIN = {6: 40.0, 5: 6.0, 4: 1.5, 3: 0.6, 2: 0.6, 7: 0.6}   # predict_flow{l} (dc_conv7: key 7)
SYN_UPFEAT_GAIN = 0.5


def synthetic_pwc_state_dict(seed: int = 0) -> dict[str, torch.Tensor]:
    """Deterministic stand-in weights keyed like PWCDCNet_Adapted's state_dict (no checkpoint exists offline).
    Convolutions are He-scaled for LeakyReLU (the reference's own kaiming_normal_ init) with small positive biases, so the
    activations neither die nor grow through the pyramid and the dense blocks. The flow heads (predict_flow{l},
    dc_conv7) are scaled so that every level predicts flows of a few pixels at its own resolution: the warps then land
    mostly inside the image with fractional offsets, and some fall outside near the borders. The transposed convolutions
    deconv{l} start as 2x bilinear upsampling of the flow plus noise."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, shape in state_dict_shapes().items():
        if name.endswith("bias"):
            out[name] = torch.randn(shape, generator=g) * 0.02 + (0.01 if ".0." in name else 0.0)
            continue
        if name.startswith("deconv"):
            bil = torch.tensor([0.25, 0.75, 0.75, 0.25])
            k = torch.outer(bil, bil)
            out[name] = torch.eye(2).reshape(2, 2, 1, 1) * k + torch.randn(shape, generator=g) * 0.05
            continue
        fan_in = int(torch.tensor(shape[1:]).prod()) if not name.startswith("upfeat") else shape[0] * 4
        if name.startswith("predict_flow") or name.startswith("dc_conv7"):
            gain = SYN_FLOW_GAIN[7 if name.startswith("dc_conv7") else int(name[12])]
        elif name.startswith("upfeat"):
            gain = SYN_UPFEAT_GAIN
        else:
            gain = (2.0 / (1 + 0.1 ** 2)) ** 0.5
        out[name] = torch.randn(shape, generator=g) * (gain / fan_in ** 0.5)
    return out


def load_checkpoint(path: str) -> dict[str, torch.Tensor]:
    """A TartanVO StereoVONet checkpoint -> the flowNet (PWC-Net) tensors, `module.flowNet.` stripped like
    TartanStereoVONetInterface.loadWeight (StereoVO_Interface.py:56-62). A missing tensor or a wrong shape raises."""
    raw = torch.load(path, map_location="cpu", weights_only=True)
    sd = {k[len(CKPT_PREFIX):]: v for k, v in raw.items() if k.startswith(CKPT_PREFIX)}
    shapes = state_dict_shapes()
    missing = [k for k in shapes if k not in sd]
    if missing:
        raise KeyError(f"{path}: checkpoint lacks {len(missing)} PWC-Net tensors, e.g. {CKPT_PREFIX}{missing[0]}")
    for k, shp in shapes.items():
        if tuple(sd[k].shape) != shp:
            raise ValueError(f"{path}: {CKPT_PREFIX}{k} has shape {tuple(sd[k].shape)}, expected {shp}")
    return {k: sd[k] for k in shapes}


class PWCFlowNet:
    """Weights on the device; `flow2(ims)` runs the network on (2,3,h,w) = [im1; im2] (h, w multiples of 64) and returns
    flow2 (1,2,h/4,w/4). Convolutions go through cuDNN under the process's TF32 flags (which this class does not touch)."""

    def __init__(self, sd: dict[str, torch.Tensor], device):
        self.device = torch.device(device)
        self.w = {k: v.detach().to(device=self.device, dtype=torch.float32).contiguous() for k, v in sd.items()}

    def _conv(self, name: str, x: torch.Tensor, stride: int = 1, dilation: int = 1, out: torch.Tensor | None = None):
        y = F.conv2d(x, self.w[f"{name}.0.weight"], self.w[f"{name}.0.bias"], stride=stride, padding=dilation,
                     dilation=dilation)
        if out is None:
            return F.leaky_relu(y, 0.1, inplace=True)
        return torch._C._nn.leaky_relu(y, 0.1, out=out)

    def _predict(self, name: str, x: torch.Tensor) -> torch.Tensor:
        return F.conv2d(x, self.w[f"{name}.weight"], self.w[f"{name}.bias"], padding=1)

    def _deconv(self, name: str, x: torch.Tensor) -> torch.Tensor:
        return F.conv_transpose2d(x, self.w[f"{name}.weight"], self.w[f"{name}.bias"], stride=2, padding=1)

    def flow2(self, ims: torch.Tensor) -> torch.Tensor:
        x = ims
        pyr = {}
        for name, _, _, stride in ENCODER:
            x = self._conv(name, x, stride=stride)
            if name.endswith("b"):
                pyr[int(name[4])] = x                   # (2, C, h, w): [image 1; image 2]
        x = None
        for level in (6, 5, 4, 3, 2):
            feat = pyr[level]
            h, w = feat.shape[-2:]
            od = level_input_channels(level)
            # The level's dense block is built in place, in the final [c4|c3|c2|c1|c0|corr|feat|up_flow|up_feat] channel
            # order: with batch 1 every suffix of the buffer is a contiguous NCHW tensor, so each convolution reads its
            # input (the suffix written so far) without torch.cat copying the growing tensor five times, and writes
            # (bias + LeakyReLU applied) once into its own slot.
            buf = torch.empty((1, od + DENSE_TOTAL, h, w), dtype=torch.float32, device=self.device)
            base = DENSE_TOTAL
            if level == 6:
                ops.pwc_warp_corr(feat[0:1], feat[1:2], None, 0.0, buf, base)
            else:
                ops.pwc_warp_corr(feat[0:1], feat[1:2], up_flow, WARP_SCALE[level], buf, base)
                c = FEAT_CH[level]
                buf[:, base + ND:base + ND + c].copy_(feat[0:1])
                buf[:, base + ND + c:base + ND + c + 2].copy_(up_flow)
                buf[:, base + ND + c + 2:base + ND + c + 4].copy_(up_feat)
            for k, cout in enumerate(DENSE):
                self._conv(f"conv{level}_{k}", buf[:, base:], out=buf[:, base - cout:base])
                base -= cout
            x = buf
            if level > 2:
                up_flow = self._deconv(f"deconv{level}", self._predict(f"predict_flow{level}", x))
                up_feat = self._deconv(f"upfeat{level}", x)
        flow2 = self._predict("predict_flow2", x)
        for i, d in enumerate(DILATION):
            x = self._conv(f"dc_conv{i + 1}", x, dilation=d)
        return flow2 + self._predict("dc_conv7", x)
