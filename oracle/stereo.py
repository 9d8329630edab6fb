"""CPU oracle of TartanVODepth (Module/Frontend/StereoDepth.py:186-229): StereoCovNet(exp=False, decoder="hourglass")
(Module/Network/StereoCov/{network,StereoNet,decoder}.py, Module/Network/TartanVOStereo/PSM/{submodule,hourglass}.py),
StereoCovNet.inference and padTo.

Restated operation by operation with torch CPU ops, in any floating dtype (float64 included), from a state dict keyed like
StereoCovNet's; BatchNorm runs as eval-mode F.batch_norm (not folded). `head` restates what macvo_stereo_head computes from
the conv_c10 outputs and cat0, with the deconvolution written as its four output phases, so the kernel's tap rule is checked
against F.conv_transpose2d at the same time (test_tartanvo_depth.py)."""
from __future__ import annotations

import torch
import torch.nn.functional as F

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
EPS = 1e-5
FE = "feature.stereo.feature_extraction."


class Net:
    def __init__(self, sd: dict, dtype=torch.float64):
        self.sd, self.dt = sd, dtype

    def t(self, k):
        return self.sd[k].to(self.dt)

    def conv(self, p, x, stride=1, padding=0):
        b = self.t(p + ".bias") if p + ".bias" in self.sd else None
        return F.conv2d(x, self.t(p + ".weight"), b, stride=stride, padding=padding)

    def convbn(self, p, x, stride=1, padding=0):
        y = F.conv2d(x, self.t(p + ".0.weight"), None, stride=stride, padding=padding)
        return F.batch_norm(y, self.t(p + ".1.running_mean"), self.t(p + ".1.running_var"), self.t(p + ".1.weight"),
                            self.t(p + ".1.bias"), False, 0.0, EPS)

    def deconv(self, p, x):
        return F.conv_transpose2d(x, self.t(p + ".weight"), self.t(p + ".bias"), stride=2, padding=1)

    def block(self, p, x, stride):
        out = F.relu(self.convbn(p + ".conv1.0", x, stride, 1))
        out = self.convbn(p + ".conv2", out, 1, 1)
        if p + ".downsample.0.weight" in self.sd:
            x = self.convbn(p + ".downsample", x, stride, 0)
        return out + x

    def residual(self, p, x):
        w = self.sd[p + ".skip_layer.conv.weight"]
        skip = self.conv(p + ".skip_layer.conv", x) if w.shape[0] != w.shape[1] else x
        out = self.conv(p + ".conv1.conv", F.relu(x))
        out = self.conv(p + ".conv2.conv", F.relu(out), padding=1)
        return self.conv(p + ".conv3.conv", F.relu(out)) + skip

    def hourglass(self, p, x, n=2):
        up1 = self.residual(p + ".up1", x)
        low = F.max_pool2d(up1, 2, 2)
        low = self.hourglass(p + ".low2", low, n - 1) if n > 1 else self.residual(p + ".low2", low)
        return up1 + F.interpolate(self.residual(p + ".low3", low), scale_factor=2, mode="bilinear")

    def features(self, x):
        for i, s in ((0, 2), (2, 1), (4, 1)):
            x = F.relu(self.convbn(f"{FE}firstconv.{i}", x, s, 1))
        outs = []
        for name, stride in (("layer1", 1), ("layer2", 2), ("layer3", 1), ("layer4", 1)):
            for i in range(3):
                x = self.block(f"{FE}{name}.{i}", x, stride if i == 0 else 1)
            outs.append(x)
        out0, raw, _, skip = outs
        th, tw = skip.shape[-2:]
        br = []
        for k, s in ((4, 8), (3, 16), (2, 32), (1, 64)):
            b = F.relu(self.convbn(f"{FE}branch{k}.1", F.avg_pool2d(skip, s, s)))
            br.append(F.interpolate(b, (th, tw), mode="bilinear", align_corners=True))
        feat = torch.cat((raw, skip, *br), 1)
        feat = torch.cat((F.interpolate(feat, (2 * th, 2 * tw), mode="bilinear", align_corners=True), out0), 1)
        return self.conv(FE + "lastconv.2", F.relu(self.convbn(FE + "lastconv.0", feat, 1, 1)))

    def encode(self, left, right):
        x = torch.cat((left, right), 1)
        n, c, h, w = x.shape
        x1 = self.features(x.reshape(2 * n, c // 2, h, w)).reshape(n, -1, h // 2, w // 2)
        x = torch.cat((x1, F.interpolate(x, scale_factor=0.5, mode="bilinear")), 1)
        p = "feature.stereo."
        cat0 = self.hourglass(p + "conv_c1", self.conv(p + "conv_c0", x, padding=1))
        x = F.max_pool2d(self.hourglass(p + "conv_c2", cat0), 2)
        th, tw = x.shape[-2:]
        ssp = [F.interpolate(F.relu(self.conv(f"{p}conv_c2_SSP.branch{k}.1", F.avg_pool2d(x, s, s))), (th, tw),
                             mode="bilinear") for k, s in ((4, 8), (3, 16), (2, 32), (1, 64))]
        cat1 = torch.cat((x, *ssp), 1)
        cat2 = F.max_pool2d(self.hourglass(p + "conv_c3", cat1), 2)
        cat3 = F.max_pool2d(self.hourglass(p + "conv_c4", cat2), 2)
        cat4 = F.max_pool2d(F.relu(self.conv(p + "conv_c5", cat3, padding=1)), 2)
        x = F.max_pool2d(F.relu(self.conv(p + "conv_c6", cat4, padding=1)), 2)
        return F.relu(self.conv(p + "conv_c6_2", x, padding=1)), [cat0, cat1, cat2, cat3, cat4]

    def decode(self, p, x, cats):
        cat0, cat1, cat2, cat3, cat4 = cats
        x = torch.cat((F.relu(self.deconv(p + "deconv_c7_2", x)), cat4), 1)
        x = torch.cat((F.relu(self.deconv(p + "deconv_c7", x)), cat3), 1)
        x = torch.cat((self.hourglass(p + "conv_c8", F.relu(self.deconv(p + "deconv_c8", x))), cat2), 1)
        x = torch.cat((self.hourglass(p + "conv_c9", F.relu(self.deconv(p + "deconv_c9", x))), cat1), 1)
        return self.hourglass(p + "conv_c10", F.relu(self.deconv(p + "deconv_c10", x)))

    def head_out(self, p, x, cat0, relu_out: bool):
        x = F.relu(self.deconv(p + "deconv_c11", torch.cat((x, cat0), 1)))
        out = self.conv(p + "conv_c13", F.relu(self.conv(p + "conv_c12", x)))
        return F.relu(out) if relu_out else out


def crop_margins(H: int, W: int):
    """StereoFeature.getCropMargin (network.py:22-31): ((h margin, w margin), (h64, w64))"""
    h64, w64 = H // 64 * 64, W // 64 * 64
    return ((H - h64) // 2, (W - w64) // 2), (h64, w64)


def normalize(img: torch.Tensor) -> torch.Tensor:
    """v2.Normalize (network.py:38): (x - mean) / std per channel"""
    m = torch.tensor(MEAN, dtype=img.dtype).view(1, 3, 1, 1)
    s = torch.tensor(STD, dtype=img.dtype).view(1, 3, 1, 1)
    return (img - m) / s


def inference_from_outputs(disp_out, cov_out, bf: float):
    """StereoFeature's / 0.02 and StereoCovNet.inference (network.py:47, 63-73)"""
    disparity = disp_out / 0.02
    depth = bf / disparity
    d2 = disparity.square()
    return depth, (bf ** 2) * ((cov_out / d2) / d2)


def head_out(sd: dict, p: str, x, cat0, relu_out: bool, dtype=torch.float64, absolute: bool = False):
    """conv_c13(relu(conv_c12(relu(deconv_c11([x | cat0]))))) (+ ReLU) of head `p` at crop resolution (1, 1, 2 h2, 2 w2),
    deconv_c11 written as its four output phases (output 2m + p, kernel tap p + 1 - 2d on input m + d, d in {0, -1} for
    p = 0 and {1, 0} for p = 1). absolute=True: every input, weight and bias by its magnitude and no ReLU, i.e. the sum of
    the magnitudes of the terms, for rounding-error bounds."""
    a = (lambda t: t.abs()) if absolute else (lambda t: t)
    act = (lambda t: t) if absolute else F.relu
    k = a(torch.cat((x, cat0), 1).to(dtype))
    w = a(sd[p + "deconv_c11.weight"].to(dtype))
    _, _, h2, w2 = k.shape
    kp = F.pad(k, (1, 1, 1, 1))
    y = torch.zeros((1, 64, 2 * h2, 2 * w2), dtype=dtype)
    for py in (0, 1):
        for px in (0, 1):
            acc = torch.zeros((1, 64, h2, w2), dtype=dtype)
            for dy in ((0, -1) if py == 0 else (1, 0)):
                for dx in ((0, -1) if px == 0 else (1, 0)):
                    tap = w[:, :, py + 1 - 2 * dy, px + 1 - 2 * dx]                      # (128, 64)
                    acc = acc + torch.einsum("bchw,co->bohw", kp[:, :, 1 + dy:1 + dy + h2, 1 + dx:1 + dx + w2], tap)
            y[:, :, py::2, px::2] = acc + a(sd[p + "deconv_c11.bias"].to(dtype)).view(1, -1, 1, 1)
    y = F.conv2d(act(y), a(sd[p + "conv_c12.weight"].to(dtype)), a(sd[p + "conv_c12.bias"].to(dtype)))
    y = F.conv2d(act(y), a(sd[p + "conv_c13.weight"].to(dtype)), a(sd[p + "conv_c13.bias"].to(dtype)))
    return F.relu(y) if relu_out and not absolute else y


def head(sd: dict, xd, xc, cat0, bf: float, dtype=torch.float64):
    """macvo_stereo_head's result at crop resolution from the conv_c10 outputs and cat0 (1, 64, h2, w2), xc None for the
    disparity head alone: (depth, variance or None), (1, 1, 2 h2, 2 w2)"""
    d = head_out(sd, "feature.stereo.", xd, cat0, False, dtype)
    if xc is None:
        return bf / (d / 0.02), None
    return inference_from_outputs(d, head_out(sd, "decoder.", xc, cat0, True, dtype), bf)


def estimate(sd: dict, imageL, imageR, bf: float, dtype=torch.float64, keep: dict | None = None):
    """TartanVODepth.estimate for (1,3,H,W) images in `dtype`: (depth, cov) (1,1,H,W), NaN outside the centre crop. With
    `keep` a dict, the head inputs (xd, xc, cat0) are stored in it."""
    H, W = imageL.shape[-2:]
    (my, mx), (h64, w64) = crop_margins(H, W)
    assert (H - h64) % 2 == 0 and (W - w64) % 2 == 0, "Can only handle even padding."
    crop = lambda im: normalize(im[..., my:my + h64, mx:mx + w64].to(dtype))
    net = Net(sd, dtype)
    ctx, cats = net.encode(crop(imageL), crop(imageR))
    xd = net.decode("feature.stereo.", ctx, cats)
    xc = net.decode("decoder.", ctx, cats)
    if keep is not None:
        keep.update(xd=xd, xc=xc, cat0=cats[0])
    d = net.head_out("feature.stereo.", xd, cats[0], False)
    c = net.head_out("decoder.", xc, cats[0], True)
    depth, var = inference_from_outputs(d, c, bf)
    out = []
    for t in (depth, var):
        full = torch.full((1, 1, H, W), float("nan"), dtype=t.dtype)
        full[..., my:my + h64, mx:mx + w64] = t
        out.append(full)
    return tuple(out)
