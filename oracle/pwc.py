"""CPU oracle of TartanVOMatcher (Module/Frontend/Matching.py:199-230): the PWCDCNet_Adapted(md=4, uncertainty=False)
forward pass that StereoVONet.forward_flow runs (Module/Network/PWCNet/pwc/pwc_model_tartanvo.py:64-297, StereoVO.py:26-28)
and the matcher's crop / rescale / NaN padding / mask (StereoVO_Interface.py:124-151, Utility/Utils.py:95-113).

Restated operation by operation with torch CPU ops, in any floating dtype (float64 included); the weights are a state dict
keyed like PWCDCNet_Adapted. The reference's correlation exists only as a cupy CUDA kernel; `correlation` restates it from
zero-padded shifts of the channel dot products divided by C.

`warp_fp32_taps` / `warp_exact` state the kernel's rule for the warp (tap positions, weights and mask in fp32, in the
reference's order; non-finite or |position| > 2^24: no tap), with the sampling itself done in any dtype."""
from __future__ import annotations

import torch
import torch.nn.functional as F

MD = 4
ND = (2 * MD + 1) ** 2                                   # 81 displacements
DENSE = (128, 128, 96, 64, 32)                           # dense block growth, conv{l}_0 .. conv{l}_4
ENCODER = (("conv1a", 3, 16, 2), ("conv1aa", 16, 16, 1), ("conv1b", 16, 16, 1),
           ("conv2a", 16, 32, 2), ("conv2aa", 32, 32, 1), ("conv2b", 32, 32, 1),
           ("conv3a", 32, 64, 2), ("conv3aa", 64, 64, 1), ("conv3b", 64, 64, 1),
           ("conv4a", 64, 96, 2), ("conv4aa", 96, 96, 1), ("conv4b", 96, 96, 1),
           ("conv5a", 96, 128, 2), ("conv5aa", 128, 128, 1), ("conv5b", 128, 128, 1),
           ("conv6aa", 128, 196, 2), ("conv6a", 196, 196, 1), ("conv6b", 196, 196, 1))
FEAT_CH = {2: 32, 3: 64, 4: 96, 5: 128, 6: 196}
WARP_SCALE = {5: 0.625, 4: 1.25, 3: 2.5, 2: 5.0}
DILATION = (1, 2, 4, 8, 16, 1)                           # dc_conv1 .. dc_conv6 (padding = dilation)
FLOW_NORM = 0.05                                         # TartanStereoVONetInterface.flow_norm


def _lrelu(x):
    return F.leaky_relu(x, 0.1)


def _conv(sd, name, x, stride=1, dilation=1):
    """conv(): Conv2d(k=3, padding=dilation) + LeakyReLU(0.1)"""
    return _lrelu(F.conv2d(x, sd[f"{name}.0.weight"].to(x.dtype), sd[f"{name}.0.bias"].to(x.dtype), stride=stride,
                           padding=dilation, dilation=dilation))


def _predict(sd, name, x):
    return F.conv2d(x, sd[f"{name}.weight"].to(x.dtype), sd[f"{name}.bias"].to(x.dtype), padding=1)


def _deconv(sd, name, x):
    return F.conv_transpose2d(x, sd[f"{name}.weight"].to(x.dtype), sd[f"{name}.bias"].to(x.dtype), stride=2, padding=1)


def warp(x: torch.Tensor, flo: torch.Tensor) -> torch.Tensor:
    """PWCDCNet_Adapted.warp (pwc_model_tartanvo.py:176-212), literally; the ones tensor takes x's dtype so that float64
    works (the reference's is float32 and only meets float32 grids)"""
    B, C, H, W = x.size()
    xx = torch.arange(0, W).view(1, -1).repeat(H, 1)
    yy = torch.arange(0, H).view(-1, 1).repeat(1, W)
    xx = xx.view(1, 1, H, W).repeat(B, 1, 1, 1)
    yy = yy.view(1, 1, H, W).repeat(B, 1, 1, 1)
    grid = torch.cat((xx, yy), 1).float()
    vgrid = grid + flo
    vgrid[:, 0, :, :] = 2.0 * vgrid[:, 0, :, :].clone() / max(W - 1, 1) - 1.0
    vgrid[:, 1, :, :] = 2.0 * vgrid[:, 1, :, :].clone() / max(H - 1, 1) - 1.0
    vgrid = vgrid.permute(0, 2, 3, 1)
    output = F.grid_sample(x, vgrid, align_corners=True)
    mask = torch.ones(x.size(), dtype=x.dtype)
    mask = F.grid_sample(mask, vgrid, align_corners=True)
    mask[mask < 0.9999] = 0
    mask[mask > 0] = 1
    return output * mask


def correlation(f1: torch.Tensor, f2: torch.Tensor) -> torch.Tensor:
    """FunctionCorrelation (correlation.py:35-102): out[(dy+4)*9 + (dx+4), y, x] = sum_c f1[c,y,x] f2[c,y+dy,x+dx] / C,
    f2 zero outside the image"""
    B, C, H, W = f1.shape
    pad = F.pad(f2, (MD, MD, MD, MD))
    out = f1.new_zeros((B, ND, H, W))
    for dy in range(-MD, MD + 1):
        for dx in range(-MD, MD + 1):
            sh = pad[:, :, MD + dy:MD + dy + H, MD + dx:MD + dx + W]
            out[:, (dy + MD) * (2 * MD + 1) + dx + MD] = (f1 * sh).sum(1) / C
    return out


def warp_fp32_taps(flow: torch.Tensor, scale: float):
    """the kernel's tap rule for flow (B,2,H,W): positions x + scale*flow_x (resp. y), warp()'s normalisation and
    grid_sample's un-normalisation, all in fp32 without contraction. Returns (xw, yn, weights (B,4,H,W) nw/ne/sw/se,
    in-bounds (B,4,H,W) bool, mask (B,1,H,W)) with no tap where a position is non-finite or beyond +-2^24."""
    f = flow.float()
    B, _, H, W = f.shape
    s = torch.tensor(scale, dtype=torch.float32)
    gx = torch.arange(W, dtype=torch.float32).view(1, W).expand(H, W)
    gy = torch.arange(H, dtype=torch.float32).view(H, 1).expand(H, W)
    vx, vy = gx + s * f[:, 0], gy + s * f[:, 1]
    nx = 2.0 * vx / float(max(W - 1, 1)) - 1.0
    ny = 2.0 * vy / float(max(H - 1, 1)) - 1.0
    ix = ((nx + 1.0) / 2.0) * float(W - 1)
    iy = ((ny + 1.0) / 2.0) * float(H - 1)
    ok = (ix.abs() <= 2.0 ** 24) & (iy.abs() <= 2.0 ** 24)
    ix, iy = torch.where(ok, ix, 0.0), torch.where(ok, iy, 0.0)
    xw, yn = ix.floor(), iy.floor()
    xe, ys = xw + 1.0, yn + 1.0
    w = torch.stack(((xe - ix) * (ys - iy), (ix - xw) * (ys - iy), (xe - ix) * (iy - yn), (ix - xw) * (iy - yn)), 1)
    inx = lambda v: (v >= 0) & (v <= W - 1)
    iny = lambda v: (v >= 0) & (v <= H - 1)
    inb = torch.stack((inx(xw) & iny(yn), inx(xe) & iny(yn), inx(xw) & iny(ys), inx(xe) & iny(ys)), 1) & ok.unsqueeze(1)
    m = torch.zeros((B, H, W), dtype=torch.float32)
    for t in range(4):
        m = torch.where(inb[:, t], m + w[:, t], m)
    m = torch.where(m < 0.9999, torch.zeros_like(m), torch.where(m > 0, torch.ones_like(m), m))
    return xw, yn, w, inb, m.unsqueeze(1)


def warp_exact(f2: torch.Tensor, flow: torch.Tensor, scale: float) -> torch.Tensor:
    """g = (sum of the in-bounds taps' weight * f2) * mask with the fp32 taps of warp_fp32_taps, sampled in f2's dtype"""
    B, C, H, W = f2.shape
    xw, yn, w, inb, m = warp_fp32_taps(flow, scale)
    out = torch.zeros_like(f2)
    flat = f2.reshape(B, C, H * W)
    for t, (ox, oy) in enumerate(((0, 0), (1, 0), (0, 1), (1, 1))):
        idx = ((yn + oy).clamp(0, H - 1) * W + (xw + ox).clamp(0, W - 1)).long().reshape(B, 1, H * W).expand(B, C, H * W)
        v = torch.gather(flat, 2, idx).reshape(B, C, H, W)
        term = v * w[:, t:t + 1].to(f2.dtype)
        out = out + torch.where(inb[:, t:t + 1], term, torch.zeros_like(term))
    return out * m.to(f2.dtype)


def warp_corr(f1, f2, flow, scale: float) -> torch.Tensor:
    """what macvo_pwc_warp_corr writes: LeakyReLU_0.1(correlation(f1, warp(f2, scale * flow))), no warp when flow is None"""
    g = f2 if flow is None else warp_exact(f2, flow, scale)
    return _lrelu(correlation(f1, g))


def _dense_block(sd, level, x):
    """multi_scale_conv: x = cat(conv{l}_k(x), x) for k = 0..4"""
    for k in range(5):
        x = torch.cat((_conv(sd, f"conv{level}_{k}", x), x), 1)
    return x


def forward(sd: dict, im1: torch.Tensor, im2: torch.Tensor, corr=correlation, warp_fn=warp) -> dict:
    """PWCDCNet_Adapted.forward (uncertainty=False) on im1, im2 (B,3,h,w), h and w multiples of 64, in their dtype.
    Returns {"flow2": (B,2,h/4,w/4), "corr": {level: LeakyReLU'd cost volume}, "up_flow": {level: up_flow * scale}}."""
    feats = []
    for im in (im1, im2):
        x, pyr = im, {}
        for name, _, _, stride in ENCODER:
            x = _conv(sd, name, x, stride=stride)
            if name.endswith("b"):
                pyr[int(name[4])] = x
        feats.append(pyr)
    c1, c2 = feats
    out = {"corr": {}, "up_flow": {}}
    x = _lrelu(corr(c1[6], c2[6]))
    out["corr"][6] = x
    for level in (6, 5, 4, 3):
        x = _dense_block(sd, level, x)
        flow = _predict(sd, f"predict_flow{level}", x)
        up_flow = _deconv(sd, f"deconv{level}", flow)
        up_feat = _deconv(sd, f"upfeat{level}", x)
        low = level - 1
        out["up_flow"][low] = up_flow * WARP_SCALE[low]
        cv = _lrelu(corr(c1[low], warp_fn(c2[low], up_flow * WARP_SCALE[low])))
        out["corr"][low] = cv
        x = torch.cat((cv, c1[low], up_flow, up_feat), 1)
    x = _dense_block(sd, 2, x)
    flow2 = _predict(sd, "predict_flow2", x)
    for i, d in enumerate(DILATION[:4]):
        x = _conv(sd, f"dc_conv{i + 1}", x, dilation=d)
    for i, d in enumerate(DILATION[4:]):
        x = _conv(sd, f"dc_conv{i + 5}", x, dilation=d)
    out["flow2"] = flow2 + _predict(sd, "dc_conv7", x)
    return out


def crop_margins(H: int, W: int):
    """getCropMargin (StereoVO_Interface.py:107-115): ((h margin, w margin), (h64, w64))"""
    h64, w64 = H // 64 * 64, W // 64 * 64
    return ((H - h64) // 2, (W - w64) // 2), (h64, w64)


def match(sd: dict, img1: torch.Tensor, img2: torch.Tensor, dtype=torch.float32) -> tuple[torch.Tensor, torch.Tensor, dict]:
    """TartanVOMatcher.forward for (1,3,H,W) images: (flow (1,2,H,W) NaN outside the crop, mask, forward dict). The mask
    is built like the reference's, from zeros_like(flow[:, :1]) *before* padTo: (1,1,h64,w64), True on [ph:-ph, pw:-pw]
    (an empty slice, so all False, when a margin is 0)."""
    H, W = img1.shape[-2:]
    (my, mx), (h64, w64) = crop_margins(H, W)
    crop = lambda im: im[..., my:my + h64, mx:mx + w64].to(dtype)
    res = forward(sd, crop(img1), crop(img2))
    flow = F.interpolate(res["flow2"] / FLOW_NORM, scale_factor=4.0, mode="nearest")
    ph, pw = (H - h64) // 2, (W - w64) // 2
    assert (H - h64) % 2 == 0 and (W - w64) % 2 == 0, "Can only handle even padding."
    mask = torch.zeros((1, 1, h64, w64), dtype=torch.bool)
    mask[..., ph:-ph, pw:-pw] = True
    full = torch.full((1, 2, H, W), float("nan"), dtype=flow.dtype)
    full[..., ph:ph + h64, pw:pw + w64] = flow
    return full, mask, res
