"""TartanVODepth's network (Module/Frontend/StereoDepth.py:186-229) on the device.

StereoCovNet(exp=False, decoder="hourglass") (Module/Network/StereoCov/network.py:50-73): StereoNet7 (StereoNet.py:69-197)
predicts the disparity, HourglassDecoder (decoder.py:8-75) its covariance from the same encoder context.

    encoder         feature_extraction (both images as one batch of 2), conv_c0 .. conv_c6_2: cuDNN through torch, eval-mode
                    BatchNorm folded into the preceding convolution once at load
    decoders        deconv_c7_2 .. conv_c10, one per head (disparity: StereoNet7's own layers, covariance: HourglassDecoder's),
                    sharing the encoder's context and skip tensors: cuDNN
    heads           [conv_c10 output | cat0] -> deconv_c11 -> ReLU -> conv_c12 -> ReLU -> conv_c13 (-> ReLU on the covariance
                    head) for both decoders, then StereoCovNet.inference and padTo: macvo_stereo_head (csrc/stereo_head.cu) when
                    cuDNN may use TF32, else the same steps as torch ops
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import ops

IMG_MEAN = (0.485, 0.456, 0.406)                     # network.py:38 (v2.Normalize after v2.CenterCrop)
IMG_STD = (0.229, 0.224, 0.225)
NORMALIZE_FACTOR = 0.02                              # StereoFeature.normalize_factor (network.py:17)
BN_EPS = 1e-5
MIN_CROP = 256                                       # feature_extraction.branch1's 64x64 average pooling at 1/4 resolution
FE = "feature.stereo.feature_extraction."
DISP = "feature.stereo."                             # StereoNet7's own decoder layers: the disparity head
COV = "decoder."                                     # HourglassDecoder: the covariance head
# feature_extraction(last_planes=64, bigger=True, middleblock=3) (submodule.py:69-108): (planes, blocks, stride) per layer
FE_LAYERS = (("layer1", 32, 3, 1), ("layer2", 64, 3, 2), ("layer3", 128, 3, 1), ("layer4", 128, 3, 1))
FE_POOLS = ((4, 8), (3, 16), (2, 32), (1, 64))      # branch k: AvgPool2d(s), in torch.cat order (submodule.py:152)
SSP_POOLS = ((4, 8), (3, 16), (2, 32), (1, 64))     # SSP (StereoNet.py:21-66), same order
# decoder transposed convolutions (k=4, s=2, p=1): name, in, out (StereoNet.py:100-127, decoder.py:20-43)
DECONVS = (("deconv_c7_2", 512, 512), ("deconv_c7", 896, 320), ("deconv_c8", 576, 192), ("deconv_c9", 384, 128),
           ("deconv_c10", 256, 64), ("deconv_c11", 128, 64))
# decoder hourglasses: name, channels (Hourglass(2, f, 0))
DEC_HOURGLASSES = (("conv_c8", 192), ("conv_c9", 128), ("conv_c10", 64))


# ---------------------------------------------------------------------------------------------------------------------------
# state dict layout
# ---------------------------------------------------------------------------------------------------------------------------
def _convbn_shapes(s, p, cin, cout, k):
    s[f"{p}.0.weight"] = (cout, cin, k, k)
    for t in ("weight", "bias", "running_mean", "running_var"):
        s[f"{p}.1.{t}"] = (cout,)
    s[f"{p}.1.num_batches_tracked"] = ()


def _conv_shapes(s, p, cin, cout, k, bias=True):
    s[f"{p}.weight"] = (cout, cin, k, k)
    if bias:
        s[f"{p}.bias"] = (cout,)


def _residual_shapes(s, p, cin, cout):
    """hourglass.py Residual(inp, out): conv1 1x1 -> out/2, conv2 3x3, conv3 1x1 -> out, skip_layer 1x1 (always built)"""
    h = cout // 2
    _conv_shapes(s, f"{p}.conv1.conv", cin, h, 1)
    _conv_shapes(s, f"{p}.conv2.conv", h, h, 3)
    _conv_shapes(s, f"{p}.conv3.conv", h, cout, 1)
    _conv_shapes(s, f"{p}.skip_layer.conv", cin, cout, 1)


def _hourglass_shapes(s, p, n, f, increase=0):
    nf = f + increase
    _residual_shapes(s, f"{p}.up1", f, nf)
    if n > 1:
        _hourglass_shapes(s, f"{p}.low2", n - 1, nf)
    else:
        _residual_shapes(s, f"{p}.low2", nf, nf)
    _residual_shapes(s, f"{p}.low3", nf, nf)


def _decoder_shapes(s, p):
    for name, cin, cout in DECONVS:
        s[f"{p}{name}.weight"], s[f"{p}{name}.bias"] = (cin, cout, 4, 4), (cout,)
    for name, f in DEC_HOURGLASSES:
        _hourglass_shapes(s, f"{p}{name}", 2, f)
    _conv_shapes(s, f"{p}conv_c12", 64, 16, 1)
    _conv_shapes(s, f"{p}conv_c13", 16, 1, 1)


def state_dict_shapes() -> dict[str, tuple[int, ...]]:
    """tensor name -> shape of StereoCovNet(exp=False, decoder="hourglass").state_dict()"""
    s: dict[str, tuple[int, ...]] = {}
    _convbn_shapes(s, FE + "firstconv.0", 3, 32, 3)
    _convbn_shapes(s, FE + "firstconv.2", 32, 32, 3)
    _convbn_shapes(s, FE + "firstconv.4", 32, 32, 3)
    cin = 32
    for name, planes, blocks, stride in FE_LAYERS:
        for i in range(blocks):
            _convbn_shapes(s, f"{FE}{name}.{i}.conv1.0", cin if i == 0 else planes, planes, 3)
            _convbn_shapes(s, f"{FE}{name}.{i}.conv2", planes, planes, 3)
            if i == 0 and (stride != 1 or cin != planes):
                _convbn_shapes(s, f"{FE}{name}.{i}.downsample", cin, planes, 1)
        cin = planes
    for k, _ in FE_POOLS:
        _convbn_shapes(s, f"{FE}branch{k}.1", 128, 32, 1)
    _convbn_shapes(s, FE + "lastconv.0", 352, 128, 3)
    _conv_shapes(s, FE + "lastconv.2", 128, 64, 1, bias=False)
    p = DISP
    _conv_shapes(s, p + "conv_c0", 134, 64, 3)
    _hourglass_shapes(s, p + "conv_c1", 2, 64)
    _hourglass_shapes(s, p + "conv_c2", 2, 64)
    for k, _ in SSP_POOLS:
        _conv_shapes(s, f"{p}conv_c2_SSP.branch{k}.1", 64, 16, 1)
    _hourglass_shapes(s, p + "conv_c3", 2, 128, 64)
    _hourglass_shapes(s, p + "conv_c4", 2, 192, 64)
    _conv_shapes(s, p + "conv_c5", 256, 384, 3)
    _conv_shapes(s, p + "conv_c6", 384, 512, 3)
    _conv_shapes(s, p + "conv_c6_2", 512, 512, 3)
    _decoder_shapes(s, DISP)
    _decoder_shapes(s, COV)
    return s


# weight gains of the synthetic stand-in (see synthetic_stereo_state_dict)
SYN_HEAD_BIAS = {DISP: 0.3, COV: 0.4}              # conv_c13 bias: disparity 0.3 / 0.02 = 15 px, covariance 0.4
SYN_HEAD_GAIN = 0.002                               # conv_c13 weight std
SYN_RESIDUAL_GAIN = 0.15                            # last convolution of a residual branch (He gain x this)
SYN_SKIP_GAIN = 0.5                                 # 1x1 skip convolutions
SYN_DECODER_GAIN = 0.5                              # transposed convolutions and conv_c12


def synthetic_stereo_state_dict(seed: int = 0) -> dict[str, torch.Tensor]:
    """Deterministic stand-in weights keyed like StereoCovNet's state_dict (no checkpoint exists offline).
    Convolutions are He-scaled for ReLU over their fan-in and halved on the residual branches, so the hourglasses neither
    die nor blow up; BatchNorm layers get non-trivial running statistics and affine terms, so the fold at load time is
    exercised. The last 1x1 convolutions of both heads get a positive bias and small weights: the disparity is mostly
    positive, a few to a few tens of pixels after / 0.02, and the covariance head is positive on most pixels."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, shape in state_dict_shapes().items():
        if name.endswith("num_batches_tracked"):
            out[name] = torch.tensor(100, dtype=torch.long)
        elif name.endswith("running_mean"):
            out[name] = torch.randn(shape, generator=g) * 0.1
        elif name.endswith("running_var"):
            out[name] = 1.0 + 0.5 * torch.rand(shape, generator=g)
        elif name.endswith("conv_c13.weight"):
            out[name] = torch.randn(shape, generator=g) * SYN_HEAD_GAIN
        elif name.endswith("conv_c13.bias"):
            out[name] = torch.full(shape, SYN_HEAD_BIAS[DISP if name.startswith(DISP) else COV])
        elif len(shape) == 1 and ".1.weight" in name:                   # BatchNorm gamma
            out[name] = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif name.endswith("bias"):
            out[name] = torch.randn(shape, generator=g) * 0.02
        else:
            fan_in = shape[1] * shape[2] * shape[3] if "deconv" not in name else shape[0] * 4
            gain = 2.0 ** 0.5
            if ".conv3.conv" in name or ".conv2.0" in name:
                gain *= SYN_RESIDUAL_GAIN                              # the last layer of a residual branch
            elif ".skip_layer." in name or name.endswith("lastconv.2.weight"):
                gain *= SYN_SKIP_GAIN
            elif "deconv" in name or "conv_c12" in name:
                gain *= SYN_DECODER_GAIN
            out[name] = torch.randn(shape, generator=g) * (gain / fan_in ** 0.5)
    return out


def load_checkpoint(path: str) -> dict[str, torch.Tensor]:
    """A TartanVO_depth_cov.pth-style checkpoint -> the StereoCovNet tensors, a `module.` prefix stripped like
    StereoCovNet.load_ddp_state_dict (network.py:75-82). A missing tensor or a wrong shape raises."""
    raw = torch.load(path, map_location="cpu", weights_only=True)
    sd = {(k[7:] if k.startswith("module.") else k): v for k, v in raw.items()}
    shapes = state_dict_shapes()
    missing = [k for k in shapes if k not in sd]
    if missing:
        raise KeyError(f"{path}: checkpoint lacks {len(missing)} StereoCovNet tensors, e.g. {missing[0]}")
    for k, shp in shapes.items():
        if tuple(sd[k].shape) != shp:
            raise ValueError(f"{path}: {k} has shape {tuple(sd[k].shape)}, expected {shp}")
    return {k: sd[k] for k in shapes}


def fold_batchnorm(sd: dict[str, torch.Tensor]) -> dict[str, torch.Tensor]:
    """eval-mode BatchNorm `A.1` folded into its convolution `A.0` (every convbn and downsample of feature_extraction):
    A.weight = w * gamma / sqrt(var + eps), A.bias = beta - mean * gamma / sqrt(var + eps), computed in float64"""
    bns = [k[:-len(".1.running_mean")] for k in sd if k.endswith(".1.running_mean")]
    out = {k: v for k, v in sd.items() if not any(k.startswith((f"{a}.0.", f"{a}.1.")) for a in bns)}
    for a in bns:
        inv = sd[f"{a}.1.weight"].double() / (sd[f"{a}.1.running_var"].double() + BN_EPS).sqrt()
        out[f"{a}.weight"] = (sd[f"{a}.0.weight"].double() * inv.view(-1, 1, 1, 1)).float()
        out[f"{a}.bias"] = (sd[f"{a}.1.bias"].double() - sd[f"{a}.1.running_mean"].double() * inv).float()
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# heads: deconv_c11 as four dense GEMMs
# ---------------------------------------------------------------------------------------------------------------------------
def head_taps(parity: int) -> tuple[tuple[int, int], tuple[int, int]]:
    """ConvTranspose2d(k=4, s=2, p=1) along one axis: output 2m + parity takes inputs m + d at kernel tap k for
    (d, k) in the returned pair (k = parity + 1 - 2 d): parity 0 -> (m, 1), (m-1, 3); parity 1 -> (m+1, 0), (m, 2)"""
    ds = (0, -1) if parity == 0 else (1, 0)
    return tuple((d, parity + 1 - 2 * d) for d in ds)


def arrange_head(w11: torch.Tensor) -> torch.Tensor:
    """deconv_c11.weight (128 in, 64 out, 4, 4) -> the kernel's B operand, tf32-rounded: (4 channel chunks, 4 phases,
    4 taps, 64 out, 32 in), phase = 2 py + px, tap = 2 ty + tx over head_taps(py) x head_taps(px)"""
    w = w11.detach().float()
    blocks = torch.empty(4, 4, 4, 64, 32, dtype=torch.float32)
    for py in (0, 1):
        for px in (0, 1):
            for ty, (_, ky) in enumerate(head_taps(py)):
                for tx, (_, kx) in enumerate(head_taps(px)):
                    wt = w[:, :, ky, kx].t()                            # (64 out, 128 in)
                    blocks[:, 2 * py + px, 2 * ty + tx] = wt.reshape(64, 4, 32).permute(1, 0, 2)
    return ops.round_tf32(blocks.contiguous())


# ---------------------------------------------------------------------------------------------------------------------------
# the network
# ---------------------------------------------------------------------------------------------------------------------------
class StereoCovNetDevice:
    """Folded weights on the device. `encode(images)` runs (2,3,h,w) = [left; right], normalised and cropped (h, w
    multiples of 64), and returns the context and the skip tensors; `decode(prefix, ...)` one decoder up to conv_c10;
    `head_torch` the rest of a head as torch ops. Convolutions go through cuDNN under the process's TF32 flags, which this
    class does not touch."""

    def __init__(self, sd: dict[str, torch.Tensor], device):
        self.device = torch.device(device)
        self.w = {k: v.detach().to(device=self.device, dtype=torch.float32).contiguous()
                  for k, v in fold_batchnorm(sd).items() if not k.endswith("num_batches_tracked")}
        # macvo_stereo_head's operands per head: deconv_c11 as GEMM blocks, and b11 | w12 | b12 | w13 | b13 in one blob
        self.head = {p: (arrange_head(self.w[p + "deconv_c11.weight"].cpu()).to(self.device),
                         torch.cat([self.w[p + n].reshape(-1) for n in ("deconv_c11.bias", "conv_c12.weight", "conv_c12.bias",
                                                                        "conv_c13.weight", "conv_c13.bias")]).contiguous())
                     for p in (DISP, COV)}

    def _conv(self, name, x, stride=1, padding=0, relu=False):
        y = F.conv2d(x, self.w[f"{name}.weight"], self.w.get(f"{name}.bias"), stride=stride, padding=padding)
        return F.relu(y, inplace=True) if relu else y

    def _deconv(self, name, x):
        return F.relu(F.conv_transpose2d(x, self.w[f"{name}.weight"], self.w[f"{name}.bias"], stride=2, padding=1),
                      inplace=True)

    def _layer(self, p, x, blocks, stride):
        """BasicBlock x blocks (submodule.py:20-43): no ReLU after the residual sum"""
        for i in range(blocks):
            s = stride if i == 0 else 1
            out = self._conv(f"{p}.{i}.conv1.0", x, stride=s, padding=1, relu=True)
            out = self._conv(f"{p}.{i}.conv2", out, padding=1)
            res = self._conv(f"{p}.{i}.downsample", x, stride=s) if f"{p}.{i}.downsample.weight" in self.w else x
            x = out + res
        return x

    def _residual(self, p, x):
        """hourglass.py Residual: the ReLU before conv1 is not in place, x itself is the identity skip"""
        w = self.w[f"{p}.skip_layer.conv.weight"]
        skip = self._conv(f"{p}.skip_layer.conv", x) if w.shape[0] != w.shape[1] else x
        out = self._conv(f"{p}.conv1.conv", F.relu(x), relu=True)
        out = self._conv(f"{p}.conv2.conv", out, padding=1, relu=True)
        return self._conv(f"{p}.conv3.conv", out) + skip

    def _hourglass(self, p, x, n=2):
        up1 = self._residual(f"{p}.up1", x)
        low = F.max_pool2d(up1, 2, 2)
        low = self._hourglass(f"{p}.low2", low, n - 1) if n > 1 else self._residual(f"{p}.low2", low)
        low = self._residual(f"{p}.low3", low)
        # nn.Upsample(scale_factor=2, mode='bilinear'): align_corners=False (hourglass.py:69)
        return up1 + F.interpolate(low, scale_factor=2, mode="bilinear")

    def _features(self, x):
        """feature_extraction(last_planes=64, bigger=True, middleblock=3).forward (submodule.py:127-159)"""
        for i in (0, 2, 4):
            x = self._conv(f"{FE}firstconv.{i}", x, stride=2 if i == 0 else 1, padding=1, relu=True)
        out0 = self._layer(FE + "layer1", x, 3, 1)
        raw = self._layer(FE + "layer2", out0, 3, 2)
        skip = self._layer(FE + "layer4", self._layer(FE + "layer3", raw, 3, 1), 3, 1)
        th, tw = skip.shape[-2:]
        # the branches upsample with align_corners=True (submodule.py:137-150), as does the x2 of `bigger` (:155)
        br = [F.interpolate(self._conv(f"{FE}branch{k}.1", F.avg_pool2d(skip, s, s), relu=True), (th, tw),
                            mode="bilinear", align_corners=True) for k, s in FE_POOLS]
        feat = torch.cat((raw, skip, *br), 1)
        feat = torch.cat((F.interpolate(feat, (2 * th, 2 * tw), mode="bilinear", align_corners=True), out0), 1)
        x = self._conv(FE + "lastconv.0", feat, padding=1, relu=True)
        return self._conv(FE + "lastconv.2", x)

    def encode(self, images: torch.Tensor):
        """StereoNet7.forward up to hourglass_context (StereoNet.py:138-171) -> (context, [cat0 .. cat4])"""
        _, _, h, w = images.shape
        x6 = images.reshape(1, 6, h, w)                         # torch.cat((tenOne, tenTwo), dim=1) (network.py:44-46)
        x1 = self._features(images).reshape(1, 128, h // 2, w // 2)    # both images as one batch of 2 (StereoNet.py:141)
        x2 = F.interpolate(x6, scale_factor=0.5, mode="bilinear")       # align_corners=False (StereoNet.py:145)
        x = self._conv(DISP + "conv_c0", torch.cat((x1, x2), 1), padding=1)     # no activation (StereoNet.py:149)
        cat0 = self._hourglass(DISP + "conv_c1", x)
        x = F.max_pool2d(self._hourglass(DISP + "conv_c2", cat0), 2)
        th, tw = x.shape[-2:]
        # SSP upsamples with align_corners=False (StereoNet.py:49-62)
        ssp = [F.interpolate(self._conv(f"{DISP}conv_c2_SSP.branch{k}.1", F.avg_pool2d(x, s, s), relu=True), (th, tw),
                             mode="bilinear") for k, s in SSP_POOLS]
        cat1 = torch.cat((x, *ssp), 1)
        cat2 = F.max_pool2d(self._hourglass(DISP + "conv_c3", cat1), 2)
        cat3 = F.max_pool2d(self._hourglass(DISP + "conv_c4", cat2), 2)
        cat4 = F.max_pool2d(self._conv(DISP + "conv_c5", cat3, padding=1, relu=True), 2)
        x = F.max_pool2d(self._conv(DISP + "conv_c6", cat4, padding=1, relu=True), 2)
        ctx = self._conv(DISP + "conv_c6_2", x, padding=1, relu=True)
        return ctx, [cat0, cat1, cat2, cat3, cat4]

    def decode(self, p: str, ctx: torch.Tensor, cats: list) -> torch.Tensor:
        """deconv_c7_2 .. conv_c10 of one decoder (StereoNet.py:173-189, decoder.py:48-64) -> (1, 64, h/2, w/2)"""
        cat0, cat1, cat2, cat3, cat4 = cats
        x = torch.cat((self._deconv(p + "deconv_c7_2", ctx), cat4), 1)
        x = torch.cat((self._deconv(p + "deconv_c7", x), cat3), 1)
        x = torch.cat((self._hourglass(p + "conv_c8", self._deconv(p + "deconv_c8", x)), cat2), 1)
        x = torch.cat((self._hourglass(p + "conv_c9", self._deconv(p + "deconv_c9", x)), cat1), 1)
        return self._hourglass(p + "conv_c10", self._deconv(p + "deconv_c10", x))

    def head_torch(self, p: str, x: torch.Tensor, cat0: torch.Tensor) -> torch.Tensor:
        """the rest of a head: cat, deconv_c11, ReLU, conv_c12, ReLU, conv_c13; the disparity head has no final activation
        (StereoNet.py:195), the covariance head ends in ReLU (decoder.py:73-74, exp=False)"""
        x = self._deconv(p + "deconv_c11", torch.cat((x, cat0), 1))
        out = self._conv(p + "conv_c13", self._conv(p + "conv_c12", x, relu=True))
        return F.relu(out) if p == COV else out


def depth_torch(disp_out: torch.Tensor, cov_out: torch.Tensor | None, bf: float):
    """StereoFeature's / 0.02 (network.py:47) and StereoCovNet.inference (network.py:63-73) in its own operation order:
    -> (depth, depth variance or None)"""
    disparity = disp_out / NORMALIZE_FACTOR
    depth = bf / disparity
    if cov_out is None:
        return depth, None
    disparity_2 = disparity.square()
    return depth, (bf ** 2) * ((cov_out / disparity_2) / disparity_2)
