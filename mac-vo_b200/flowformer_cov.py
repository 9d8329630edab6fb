"""FlowFormerCov frontend network — host-side PyTorch plumbing around the two hot-path kernels.

This is a from-scratch, weight-compatible (same `state_dict` keys, SURVEY.md Appendix A) functional
re-implementation of the reference network

    Module/Network/FlowFormerCov/flownet.py:18-44      (forward / inference)
    Module/Network/FlowFormer/core/twins_svt.py:19-37   (Twins-SVT-L, 2 stages)
    Module/Network/FlowFormer/core/encoder.py:12-295    (PatchEmbed, cost perceiver, MemoryEncoder)
    Module/Network/FlowFormer/core/twins.py:22-243      (context-conditioned Twins blocks)
    Module/Network/FlowFormerCov/covhead.py:60-140      (12-iteration flow + covariance decoder)
    Module/Network/FlowFormer/core/gma.py, gru.py, attention.py

Plain GEMMs and convolutions go through torch (cuBLAS / cuDNN — library GEMMs); everything memory-bound on a CUDA
fp32 run goes through our own kernels (`csrc/nn_kernels.cu`, `csrc/decoder_fused.cu`: LayerNorm, PatchEmbed conv1,
the attention family incl. the K/V-free perceiver input layer, the SepConvGRU glue on NHWC `[h|x]` state buffers); CPU
tensors and half-precision runs keep the torch ops (`_native()`), which is also how the class is checked against the
reference network's golden outputs on the CPU. The two operators `BASELINE.json: north_star` names are NOT torch ops here:

* `corr_fn(f1, f2) -> (B, 1, H1, W1, H1, W1)`   all-pairs correlation volume (encoder.py:256-275)
* `lookup_fn(cost_maps, coords) -> (B, 81, H1, W1)`  9x9 window lookup (decoder.py:141-153)

By default both bind to the sm_90a CUDA kernels behind the C-ABI (`ops.corr_build`, `ops.corr_lookup`)
and fail loudly when the library / a GPU is missing. Tests inject the CPU oracle instead; a CUDA network always looks up
with `ops.corr_lookup`.

Restructuring relative to the reference (same arithmetic per output, fewer launches / bytes):
* weights live in a flat dict keyed by the checkpoint names, the forward pass is functional;
* eval mode only returns the last prediction, so the convex upsampling and both 576-channel mask
  heads run once (after the last refinement) instead of 12 times;
* z and r gates of each separable GRU share their input -> one conv with concatenated filters;
* sine position encodings that do not depend on the input are built once per resolution;
* projections whose input is `cat([x, context]) + position` are split by linearity: the context / position half is a
  per-(image % 2, position) term computed once per layer on 2 x N tokens and added inside the attention kernel;
* independent branches (context encoder vs feature path, flow GRU vs covariance GRU, the two motion-encoder
  branches) run on forked streams, which the frontend's CUDA graph captures as parallel branches.
"""
from __future__ import annotations

import math
import os
import zlib
from typing import Callable

import torch
import torch.nn.functional as F

Tensor = torch.Tensor

# cfg constants: Module/Network/FlowFormer/configs/submission.py:16-32
LATENT_TOKENS = 8
LATENT_DIM = 128
QUERY_DIM = 64
COST_INPUT_DIM = 64
VERT_C_DIM = 64
ENCODER_DEPTH = 3


# ----------------------------------------------------------------------------------------------
# parameter table (name -> shape, init kind); keys equal the reference checkpoint's
# ----------------------------------------------------------------------------------------------
def _svt_spec(prefix: str) -> list[tuple[str, tuple[int, ...], str]]:
    out: list[tuple[str, tuple[int, ...], str]] = []
    dims, heads, srs, patch, cin = (128, 256), (4, 8), (8, 4), (4, 2), (3, 128)
    for s, (C, sr, ps, ci) in enumerate(zip(dims, srs, patch, cin)):
        p = f"{prefix}.svt."
        out += [(p + f"patch_embeds.{s}.proj.weight", (C, ci, ps, ps), "w"), (p + f"patch_embeds.{s}.proj.bias", (C,), "b"),
                (p + f"patch_embeds.{s}.norm.weight", (C,), "one"), (p + f"patch_embeds.{s}.norm.bias", (C,), "zero")]
        for j in range(2):
            b = p + f"blocks.{s}.{j}."
            out += [(b + "norm1.weight", (C,), "one"), (b + "norm1.bias", (C,), "zero")]
            if j == 0:
                out += [(b + "attn.qkv.weight", (3 * C, C), "w"), (b + "attn.qkv.bias", (3 * C,), "b")]
            else:
                out += [(b + "attn.q.weight", (C, C), "w"), (b + "attn.q.bias", (C,), "b"),
                        (b + "attn.kv.weight", (2 * C, C), "w"), (b + "attn.kv.bias", (2 * C,), "b")]
            out += [(b + "attn.proj.weight", (C, C), "w"), (b + "attn.proj.bias", (C,), "b")]
            if j == 1:
                out += [(b + "attn.sr.weight", (C, C, sr, sr), "w"), (b + "attn.sr.bias", (C,), "b"),
                        (b + "attn.norm.weight", (C,), "one"), (b + "attn.norm.bias", (C,), "zero")]
            out += [(b + "norm2.weight", (C,), "one"), (b + "norm2.bias", (C,), "zero"),
                    (b + "mlp.fc1.weight", (4 * C, C), "w"), (b + "mlp.fc1.bias", (4 * C,), "b"),
                    (b + "mlp.fc2.weight", (C, 4 * C), "w"), (b + "mlp.fc2.bias", (C,), "b")]
        out += [(p + f"pos_block.{s}.proj.0.weight", (C, 1, 3, 3), "w"), (p + f"pos_block.{s}.proj.0.bias", (C,), "b")]
    return out


def _attn_layer_spec(p: str, qdim: int, tdim: int, proj_in: int) -> list[tuple[str, tuple[int, ...], str]]:
    return [(p + "norm1.weight", (qdim,), "one"), (p + "norm1.bias", (qdim,), "zero"),
            (p + "norm2.weight", (qdim,), "one"), (p + "norm2.bias", (qdim,), "zero"),
            (p + "q.weight", (qdim, qdim), "w"), (p + "q.bias", (qdim,), "b"),
            (p + "k.weight", (qdim, tdim), "w"), (p + "k.bias", (qdim,), "b"),
            (p + "v.weight", (qdim, tdim), "w"), (p + "v.bias", (qdim,), "b"),
            (p + "proj.weight", (qdim, proj_in), "w"), (p + "proj.bias", (qdim,), "b"),
            (p + "ffn.0.weight", (qdim, qdim), "w"), (p + "ffn.0.bias", (qdim,), "b"),
            (p + "ffn.3.weight", (qdim, qdim), "w"), (p + "ffn.3.bias", (qdim,), "b")]


def _gru_spec(p: str) -> list[tuple[str, tuple[int, ...], str]]:
    out = []
    for g in "zrq":
        out += [(p + f"conv{g}1.weight", (128, 512, 1, 5), "w"), (p + f"conv{g}1.bias", (128,), "b")]
    for g in "zrq":
        out += [(p + f"conv{g}2.weight", (128, 512, 5, 1), "w"), (p + f"conv{g}2.bias", (128,), "b")]
    return out


def param_spec() -> list[tuple[str, tuple[int, ...], str]]:
    """All 428 tensors of the reference `FlowFormerCov.state_dict()` (SURVEY.md Appendix A)."""
    D = LATENT_DIM
    s = _svt_spec("memory_encoder.feat_encoder")
    s += [("memory_encoder.channel_convertor.weight", (256, 256, 1, 1), "w")]
    c = "memory_encoder.cost_perceiver_encoder."
    s += [(c + "latent_tokens", (1, LATENT_TOKENS, D), "randn")]
    pe = c + "patch_embed."
    s += [(pe + "proj.0.weight", (16, 1, 6, 6), "w"), (pe + "proj.0.bias", (16,), "b"),
          (pe + "proj.2.weight", (32, 16, 6, 6), "w"), (pe + "proj.2.bias", (32,), "b"),
          (pe + "proj.4.weight", (64, 32, 6, 6), "w"), (pe + "proj.4.bias", (64,), "b"),
          (pe + "ffn_with_coord.0.weight", (D, D, 1, 1), "w"), (pe + "ffn_with_coord.0.bias", (D,), "b"),
          (pe + "ffn_with_coord.2.weight", (D, D, 1, 1), "w"), (pe + "ffn_with_coord.2.bias", (D,), "b"),
          (pe + "norm.weight", (D,), "one"), (pe + "norm.bias", (D,), "zero")]
    s += _attn_layer_spec(c + "input_layer.", D, D, D)
    for i in range(ENCODER_DEPTH):
        s += _attn_layer_spec(c + f"encoder_layers.{i}.", D, D, D)
    for i in range(ENCODER_DEPTH):
        for blk in ("local_block", "global_block"):
            b = c + f"vertical_encoder_layers.{i}.{blk}."
            s += [(b + "norm1.weight", (D,), "one"), (b + "norm1.bias", (D,), "zero"),
                  (b + "attn.context_proj.weight", (VERT_C_DIM, 256), "w"), (b + "attn.context_proj.bias", (VERT_C_DIM,), "b"),
                  (b + "attn.q.weight", (D, D + VERT_C_DIM), "w"), (b + "attn.q.bias", (D,), "b")]
            kin = D + VERT_C_DIM if blk == "local_block" else D
            s += [(b + "attn.k.weight", (D, kin), "w"), (b + "attn.k.bias", (D,), "b"),
                  (b + "attn.v.weight", (D, D), "w"), (b + "attn.v.bias", (D,), "b"),
                  (b + "attn.proj.weight", (D, D), "w"), (b + "attn.proj.bias", (D,), "b")]
            if blk == "global_block":
                s += [(b + "attn.sr_key.weight", (D, D + VERT_C_DIM, 4, 4), "w"), (b + "attn.sr_key.bias", (D,), "b"),
                      (b + "attn.sr_value.weight", (D, D, 4, 4), "w"), (b + "attn.sr_value.bias", (D,), "b"),
                      (b + "attn.norm.weight", (D,), "one"), (b + "attn.norm.bias", (D,), "zero")]
            s += [(b + "norm2.weight", (D,), "one"), (b + "norm2.bias", (D,), "zero"),
                  (b + "mlp.fc1.weight", (4 * D, D), "w"), (b + "mlp.fc1.bias", (4 * D,), "b"),
                  (b + "mlp.fc2.weight", (D, 4 * D), "w"), (b + "mlp.fc2.bias", (D,), "b")]
    m = "memory_decoder."
    s += [(m + "delta", (1, 9, 9, 2), "delta"),
          (m + "flow_token_encoder.0.weight", (QUERY_DIM, 81, 1, 1), "w"), (m + "flow_token_encoder.0.bias", (QUERY_DIM,), "b"),
          (m + "flow_token_encoder.2.weight", (QUERY_DIM, QUERY_DIM, 1, 1), "w"), (m + "flow_token_encoder.2.bias", (QUERY_DIM,), "b"),
          (m + "proj.weight", (256, 256, 1, 1), "w"), (m + "proj.bias", (256,), "b")]
    s += _attn_layer_spec(m + "decoder_layer.cross_attend.", QUERY_DIM, D, 2 * QUERY_DIM)
    e = m + "update_block.encoder."
    s += [(e + "convc1.weight", (256, 81 + QUERY_DIM, 1, 1), "w"), (e + "convc1.bias", (256,), "b"),
          (e + "convc2.weight", (192, 256, 3, 3), "w"), (e + "convc2.bias", (192,), "b"),
          (e + "convf1.weight", (128, 2, 7, 7), "w"), (e + "convf1.bias", (128,), "b"),
          (e + "convf2.weight", (64, 128, 3, 3), "w"), (e + "convf2.bias", (64,), "b"),
          (e + "conv.weight", (126, 256, 3, 3), "w"), (e + "conv.bias", (126,), "b")]
    s += _gru_spec(m + "update_block.gru.")
    s += [(m + "update_block.flow_head.conv1.weight", (256, 128, 3, 3), "w"), (m + "update_block.flow_head.conv1.bias", (256,), "b"),
          (m + "update_block.flow_head.conv2.weight", (2, 256, 3, 3), "w"), (m + "update_block.flow_head.conv2.bias", (2,), "b"),
          (m + "update_block.mask.0.weight", (256, 128, 3, 3), "w"), (m + "update_block.mask.0.bias", (256,), "b"),
          (m + "update_block.mask.2.weight", (576, 256, 1, 1), "w"), (m + "update_block.mask.2.bias", (576,), "b"),
          (m + "update_block.aggregator.gamma", (1,), "gamma"),
          (m + "update_block.aggregator.to_v.weight", (128, 128, 1, 1), "w"),
          (m + "att.to_qk.weight", (256, 128, 1, 1), "w")]
    s += _gru_spec(m + "cov_update.gru.")
    h = m + "cov_update.cov_head."
    s += [(h + "conv1.weight", (256, 128, 3, 3), "w"), (h + "conv1.bias", (256,), "b"),
          (h + "conv2.weight", (128, 256, 3, 3), "w"), (h + "conv2.bias", (128,), "b"),
          (h + "conv3.weight", (64, 128, 3, 3), "w"), (h + "conv3.bias", (64,), "b"),
          (h + "conv4.weight", (2, 64, 3, 3), "w"), (h + "conv4.bias", (2,), "b"),
          (m + "cov_update.mask.0.weight", (256, 128, 3, 3), "w"), (m + "cov_update.mask.0.bias", (256,), "b"),
          (m + "cov_update.mask.2.weight", (576, 256, 1, 1), "w"), (m + "cov_update.mask.2.bias", (576,), "b")]
    s += _svt_spec("context_encoder")
    return s


def synthetic_state_dict(seed: int = 0) -> dict[str, Tensor]:
    """Deterministic stand-in for the released checkpoint (absent: no network, SURVEY.md §8c).

    Every tensor is drawn from its own generator seeded by (seed, crc32(key)), so the values do not
    depend on module construction order and can be loaded into the reference model as well
    (`tests/golden/make_golden.py`) — that is how the golden fixtures are tied to these weights.
    Weights ~ U(+-1/sqrt(fan_in)) (torch's default conv/linear init), norms (1, 0), GMA gamma 0.5
    (the reference initialises it to 0, which would leave the aggregation path untested).
    """
    sd: dict[str, Tensor] = {}
    for key, shape, kind in param_spec():
        g = torch.Generator().manual_seed((seed * 1000003 + zlib.crc32(key.encode())) % (2 ** 31))
        if kind == "one":
            t = torch.ones(shape)
        elif kind == "zero":
            t = torch.zeros(shape)
        elif kind == "randn":
            t = torch.randn(shape, generator=g)
        elif kind == "gamma":
            t = torch.full(shape, 0.5)
        elif kind == "delta":
            t = window_delta()
        else:
            fan_in = 1
            for d in shape[1:]:
                fan_in *= d
            if kind == "b":  # bias: fan_in unknown from its own shape; same +-1/sqrt(.) family
                fan_in = max(shape[0], 16)
            bound = 1.0 / math.sqrt(fan_in)
            t = (torch.rand(shape, generator=g) * 2 - 1) * bound
        sd[key] = t
    return sd


def window_delta() -> Tensor:
    """`MemoryDecoder.delta` buffer (decoder.py:124-129): delta[0,i,j] = (i-4, j-4)."""
    r = torch.linspace(-4, 4, 9)
    return torch.stack(torch.meshgrid(r, r, indexing="ij"), dim=-1).view(1, 9, 9, 2)


# ----------------------------------------------------------------------------------------------
# small functional helpers
# ----------------------------------------------------------------------------------------------
def coords_grid(batch: int, ht: int, wd: int, device, dtype) -> Tensor:
    """(B, 2, H, W) with channel 0 = x, 1 = y  (core/utils.py:36-43)."""
    ys, xs = torch.meshgrid(torch.arange(ht, device=device, dtype=dtype),
                            torch.arange(wd, device=device, dtype=dtype), indexing="ij")
    return torch.stack((xs, ys), dim=0).unsqueeze(0).repeat(batch, 1, 1, 1)


def sine_embed(xy: Tensor, dim: int) -> Tensor:
    """LinearPositionEmbeddingSine (core/attention.py:71-101): cat(sin x f, cos x f, sin y f, cos y f)."""
    freq = torch.arange(dim // 4, device=xy.device, dtype=xy.dtype) * (1 / 200) * torch.pi
    ax = xy[..., -2:-1] * freq
    ay = xy[..., -1:] * freq
    return torch.cat([torch.sin(ax), torch.cos(ax), torch.sin(ay), torch.cos(ay)], dim=-1)


def _f32(x: Tensor) -> Tensor:
    """The reference's `.float()` interface casts (flownet.py:28-29, covhead.py:121-131). A float64 run of this class — the
    ground truth of the parity ladder, tests/golden/make_golden.py — stays float64 end to end."""
    return x if x.dtype == torch.float64 else x.float()


def _sdpa(q: Tensor, k: Tensor, v: Tensor) -> Tensor:
    return F.scaled_dot_product_attention(q, k, v, attn_mask=None, dropout_p=0.0, is_causal=False)


class FlowFormerCovNet:
    """Functional FlowFormerCov. `inference(image1, image2) -> (flow, cov)` like flownet.py:37-44."""

    def __init__(self, state_dict: dict[str, Tensor], device, enc_dtype=torch.float32, dec_dtype=torch.float32,
                 decoder_depth: int = 12,
                 corr_fn: Callable[[Tensor, Tensor], Tensor] | None = None,
                 lookup_fn: Callable[[Tensor, Tensor], Tensor] | None = None):
        self.device = torch.device(device)
        self.enc_dtype, self.dec_dtype, self.depth = enc_dtype, dec_dtype, decoder_depth
        # TF32 mode only: the 128-channel transformer MLPs as one fused kernel (MACVO_B200_MLP_TC=0: cuBLAS GEMMs + GELU + add)
        self.mlp_tensor_cores = os.environ.get("MACVO_B200_MLP_TC", "1") != "0"
        self._ops = None
        if corr_fn is None or lookup_fn is None or self.device.type == "cuda":
            from . import ops  # binds to the CUDA library; raises if it cannot be loaded
            if self.device.type == "cuda" and lookup_fn is not None and lookup_fn is not ops.corr_lookup:
                raise ValueError("a CUDA FlowFormerCovNet looks up with ops.corr_lookup (its decoder reads the lookup rows "
                                 "directly); inject a lookup_fn only into a CPU network")
            corr_fn = corr_fn or ops.corr_build
            lookup_fn = lookup_fn or ops.corr_lookup
            self._ops = ops if self.device.type == "cuda" else None
        self.corr_fn, self.lookup_fn = corr_fn, lookup_fn
        self.load_state_dict(state_dict)
        self._cache: dict = {}
        self.taps: dict | None = None      # set to {} to record per-stage intermediates (parity ladder; eager runs only)

    def _tap(self, name: str, t: Tensor) -> None:
        if self.taps is not None:
            self.taps.setdefault(name, []).append(t.detach().clone())

    # ---- weights -------------------------------------------------------------------------------
    def load_state_dict(self, ckpt: dict[str, Tensor]) -> None:
        """Accepts the reference checkpoint layout incl. DDP `module.` prefixes (flownet.py:46-53)."""
        ckpt = {(k[7:] if k.startswith("module.") else k): v for k, v in ckpt.items()}
        W: dict[str, Tensor] = {}
        missing = []
        for key, shape, _ in param_spec():
            if key not in ckpt:
                missing.append(key)
                continue
            t = ckpt[key]
            assert tuple(t.shape) == shape, f"{key}: expected {shape}, got {tuple(t.shape)}"
            if key.startswith("memory_decoder."):
                dt = self.dec_dtype
                if key.startswith("memory_decoder.proj.") and dt != torch.float64:
                    dt = torch.float32  # MemoryDecoder.proj is not cast (covhead.py:52-58 omits it)
            else:
                dt = self.enc_dtype
            t = t.detach().to(device=self.device, dtype=dt).contiguous()
            if t.dim() == 4:        # conv filters: NHWC so that cuDNN runs its tensor-core kernels without layout round trips
                t = t.contiguous(memory_format=torch.channels_last)
            W[key] = t
        if missing:
            raise KeyError(f"checkpoint misses {len(missing)} tensors, e.g. {missing[:3]}")
        self.W = W
        # fused GRU gate filters (z|r share their input)
        for p in ("memory_decoder.update_block.gru.", "memory_decoder.cov_update.gru."):
            for o in "12":
                W[p + f"convzr{o}.weight"] = torch.cat([W[p + f"convz{o}.weight"], W[p + f"convr{o}.weight"]], 0).contiguous(
                    memory_format=torch.channels_last)
                W[p + f"convzr{o}.bias"] = torch.cat([W[p + f"convz{o}.bias"], W[p + f"convr{o}.bias"]], 0).contiguous()
        # channel-padded motion-encoder filters for the fused token path (csrc/decoder_token.cu): convc1 reads the 160-channel
        # rows [cost_global 64 | cost_forward 81 | 0 x 15]; `conv` writes 128 channels whose last two (zero filters, zero bias
        # -> relu(0) = 0) receive the flow afterwards, which removes the 126+2 concat and cuDNN's channel re-padding passes
        e = "memory_decoder.update_block.encoder."
        w1 = W[e + "convc1.weight"]
        W[e + "convc1p.weight"] = F.pad(w1, (0, 0, 0, 0, 0, 160 - w1.shape[1])).contiguous(memory_format=torch.channels_last)
        W[e + "convc1p.bias"] = W[e + "convc1.bias"]
        W[e + "convp.weight"] = F.pad(W[e + "conv.weight"], (0, 0, 0, 0, 0, 0, 0, 2)).contiguous(memory_format=torch.channels_last)
        W[e + "convp.bias"] = F.pad(W[e + "conv.bias"], (0, 2)).contiguous()

    def state_dict(self) -> dict[str, Tensor]:
        return {k: self.W[k] for k, _, _ in param_spec()}

    def _lin(self, x: Tensor, p: str) -> Tensor:
        return F.linear(x, self.W[p + ".weight"], self.W.get(p + ".bias"))

    def _conv(self, x: Tensor, p: str, stride=1, padding=0, groups=1) -> Tensor:
        """conv2d on channels-last activations: maps stay (B, H, W, C)-strided between the convolutions, so a
        1x1 conv is a plain GEMM and `tokens <-> map` reshapes are free views."""
        if not x.is_contiguous(memory_format=torch.channels_last):
            x = x.contiguous(memory_format=torch.channels_last)
        return F.conv2d(x, self.W[p + ".weight"], self.W.get(p + ".bias"), stride=stride, padding=padding, groups=groups)

    def _conv_relu(self, x: Tensor, p: str, stride=1, padding=0) -> Tensor:
        """relu(conv2d(x) + bias): one cuDNN fused conv-bias-activation launch on the GPU path."""
        if self._ops is not None and x.is_cuda:
            if not x.is_contiguous(memory_format=torch.channels_last):
                x = x.contiguous(memory_format=torch.channels_last)
            pair = lambda v: (v, v) if isinstance(v, int) else tuple(v)
            return torch.cudnn_convolution_relu(x, self.W[p + ".weight"], self.W.get(p + ".bias"), pair(stride), pair(padding), (1, 1), 1)
        return F.relu(self._conv(x, p, stride=stride, padding=padding))

    def _ln(self, x: Tensor, p: str, eps: float = 1e-5) -> Tensor:
        if self._native(x) and x.shape[-1] in self._ops.LAYER_NORM_CHANNELS:
            return self._ops.layer_norm(x, self.W[p + ".weight"], self.W[p + ".bias"], eps)
        return F.layer_norm(x, (x.shape[-1],), self.W[p + ".weight"], self.W[p + ".bias"], eps)

    def _add_ln(self, x: Tensor, y: Tensor, p: str, eps: float = 1e-5) -> tuple[Tensor, Tensor]:
        """(x + y, LayerNorm(x + y)): the residual add in front of every norm2, fused into the LayerNorm pass"""
        if self._native(x) and x.shape[-1] in (128, 256, 512) and x.shape == y.shape:
            return self._ops.add_layer_norm(x, y, self.W[p + ".weight"], self.W[p + ".bias"], eps)
        s = x + y
        return s, self._ln(s, p, eps)

    def _native(self, x: Tensor) -> bool:
        """fp32 CUDA activations go through csrc/nn_kernels.cu; half-precision ones (MACVO_Fast) and the CPU
        golden-parity runs of this class keep the torch ops."""
        return self._ops is not None and x.is_cuda and x.dtype == torch.float32

    def _attn(self, q: Tensor, k: Tensor, v: Tensor, heads: int) -> Tensor:
        """softmax(q k^T / sqrt(d)) v on (B|1, Nq, C), (B, Nk, C), (B, Nk, C) token matrices -> (B, Nq, C)."""
        B, J, C = k.shape
        d = C // heads
        if self._native(k) and (d in (16, 32) or (d == 8 and q.shape[1] <= 8 and (heads == 8 or q.shape[1] == 1))) and (J + 31) // 32 * 32 * (2 * d + 16) * 4 <= 200 * 1024:
            return self._ops.small_attention(q, k, v, heads)
        I = q.shape[1]
        qh = q.reshape(q.shape[0], I, heads, d).permute(0, 2, 1, 3).expand(B, -1, -1, -1)
        kh = k.reshape(B, J, heads, d).permute(0, 2, 1, 3)
        vh = v.reshape(B, J, heads, d).permute(0, 2, 1, 3)
        if I * J <= 4096:      # tiny products: explicit matmul-softmax-matmul beats the SDPA kernels
            a = (torch.matmul(qh, kh.transpose(-1, -2)) * (d ** -0.5)).softmax(dim=-1)
            o = torch.matmul(a, vh)
        else:
            o = _sdpa(qh, kh, vh)
        return o.permute(0, 2, 1, 3).reshape(B, I, C)

    def _memo(self, key, fn):
        if key not in self._cache:
            self._cache[key] = fn()
        return self._cache[key]

    # ---- Twins-SVT-L, first two stages (core/twins_svt.py:19-37, Twins/svt_large.py) -------------
    def svt(self, x: Tensor, prefix: str) -> Tensor:
        B = x.shape[0]
        for s, (heads, sr, ps) in enumerate(((4, 8, 4), (8, 4, 2))):
            p = f"{prefix}.svt."
            x = self._conv(x, p + f"patch_embeds.{s}.proj", stride=ps)
            C, H, W = x.shape[1:]
            x = self._ln(x.flatten(2).transpose(1, 2), p + f"patch_embeds.{s}.norm")
            b0, b1 = p + f"blocks.{s}.0.", p + f"blocks.{s}.1."
            # block 0: locally-grouped attention (7x7 windows, zero padded after the norm)
            x, xn = self._add_ln(x, self._svt_local_attn(self._ln(x, b0 + "norm1", 1e-6), (H, W), b0 + "attn.", heads), b0 + "norm2", 1e-6)
            x = self._mlp_residual(x, xn, b0 + "mlp.", "fc1", "fc2")
            # PEG: depthwise 3x3 + identity
            t = x.transpose(1, 2).reshape(B, C, H, W)          # channels-last view of the token matrix
            t = self._conv(t, p + f"pos_block.{s}.proj.0", padding=1, groups=C) + t
            x = t.flatten(2).transpose(1, 2)
            # block 1: globally sub-sampled attention
            x, xn = self._add_ln(x, self._svt_global_attn(self._ln(x, b1 + "norm1", 1e-6), (H, W), b1 + "attn.", heads, sr), b1 + "norm2", 1e-6)
            x = self._mlp_residual(x, xn, b1 + "mlp.", "fc1", "fc2")
            x = x.reshape(B, H, W, C).permute(0, 3, 1, 2)      # (B, C, H, W) logical, channels-last in memory
        return x

    def _mlp_residual(self, x: Tensor, xn: Tensor, p: str, fc1: str, fc2: str) -> Tensor:
        """x + fc2(GELU(fc1(xn))); in TF32 mode at 128 channels one kernel (csrc/mlp_tc.cu) that keeps the hidden activation on
        chip, with its weights rounded to tf32 once"""
        w1 = self.W[p + fc1 + ".weight"]
        if (self.mlp_tensor_cores and self._native(x) and torch.backends.cuda.matmul.allow_tf32 and x.shape[-1] == 128
                and w1.shape[0] in self._ops.MLP_TC_HIDDEN and x.is_contiguous() and xn.is_contiguous()):
            w1t, w2t = self._memo(("mlp_tc", p), lambda: (self._ops.round_tf32(w1), self._ops.round_tf32(self.W[p + fc2 + ".weight"])))
            return self._ops.mlp_tc(xn, x, w1t, self.W[p + fc1 + ".bias"], w2t, self.W[p + fc2 + ".bias"])
        return x + self._lin(F.gelu(self._lin(xn, p + fc1)), p + fc2)

    @staticmethod
    def _to_windows(x: Tensor, ws: int) -> tuple[Tensor, tuple[int, int, int, int]]:
        """(B, H, W, C) -> (B*nh*nw, ws*ws, C), zero padded on the right / bottom."""
        B, H, W, C = x.shape
        pr, pb = (ws - W % ws) % ws, (ws - H % ws) % ws
        x = F.pad(x, (0, 0, 0, pr, 0, pb))
        nh, nw = (H + pb) // ws, (W + pr) // ws
        x = x.reshape(B, nh, ws, nw, ws, C).transpose(2, 3).reshape(B * nh * nw, ws * ws, C)
        return x, (B, nh, nw, C)

    @staticmethod
    def _from_windows(x: Tensor, meta: tuple[int, int, int, int], ws: int, H: int, W: int) -> Tensor:
        B, nh, nw, C = meta
        x = x.reshape(B, nh, nw, ws, ws, C).transpose(2, 3).reshape(B, nh * ws, nw * ws, C)
        return x[:, :H, :W, :].reshape(B, H * W, C)

    def _svt_local_attn(self, x: Tensor, size, p: str, heads: int, ws: int = 7) -> Tensor:
        B, N, C = x.shape
        H, W = size
        xw, meta = self._to_windows(x.view(B, H, W, C), ws)
        wq, bq = self.W[p + "qkv.weight"], self.W[p + "qkv.bias"]          # rows [q | k | v] (svt_large.py:111)
        q, k, v = (F.linear(xw, wq[i * C:(i + 1) * C], bq[i * C:(i + 1) * C]) for i in range(3))
        o = self._attn(q, k, v, heads)
        return self._lin(self._from_windows(o, meta, ws, H, W), p + "proj")

    def _svt_global_attn(self, x: Tensor, size, p: str, heads: int, sr: int) -> Tensor:
        B, N, C = x.shape
        q = self._lin(x, p + "q")
        t = self._conv(x.permute(0, 2, 1).reshape(B, C, *size), p + "sr", stride=sr)
        t = self._ln(t.reshape(B, C, -1).permute(0, 2, 1), p + "norm")
        wkv, bkv = self.W[p + "kv.weight"], self.W[p + "kv.bias"]          # rows [k | v] (svt_large.py:161)
        o = self._attn(q, F.linear(t, wkv[:C], bkv[:C]), F.linear(t, wkv[C:], bkv[C:]), heads)
        return self._lin(o, p + "proj")

    # ---- cost perceiver encoder (core/encoder.py:194-244) -------------------------------------
    def patch_embed(self, cost_maps: Tensor) -> Tensor:
        """(M, 1, H2, W2) -> (M, h*w, 128) tokens  (PatchEmbed, core/encoder.py:12-55)."""
        p = "memory_encoder.cost_perceiver_encoder.patch_embed."
        M, _, H2, W2 = cost_maps.shape
        if self._native(cost_maps) and (H2 + 7) // 8 * 8 * ((W2 + 7) // 8 * 8) <= 96 * 160:
            if torch.backends.cudnn.allow_tf32:
                # conv1 written space-to-depth -> proj.2 (6x6 / s2 over 16 channels, half-empty K blocks in the implicit GEMM)
                # runs as the equivalent 3x3 / s1 convolution over 64 channels
                x = self._ops.patch_embed_conv1(cost_maps, self.W[p + "proj.0.weight"], self.W[p + "proj.0.bias"], s2d=True)
                w2 = self._memo(("pe_w2_s2d", x.device), lambda: self._ops.space_to_depth_filter(self.W[p + "proj.2.weight"])
                                .contiguous(memory_format=torch.channels_last))
                x = torch.cudnn_convolution_relu(x, w2, self.W[p + "proj.2.bias"], (1, 1), (1, 1), (1, 1), 1)
            else:
                x = self._ops.patch_embed_conv1(cost_maps, self.W[p + "proj.0.weight"], self.W[p + "proj.0.bias"])
                x = self._conv_relu(x, p + "proj.2", stride=2, padding=2)
        else:
            x = F.pad(cost_maps, (0, (8 - W2 % 8) % 8, 0, (8 - H2 % 8) % 8))
            x = self._conv_relu(x, p + "proj.0", stride=2, padding=2)
            x = self._conv_relu(x, p + "proj.2", stride=2, padding=2)
        native = self._native(x)
        # proj.4 has no activation after it, so its bias b4 only enters through ffn_with_coord.0: W0x (x + b4) — on the
        # native path it is folded into the per-position term and the conv runs bias-free (saves a 0.13 ms bias pass)
        x = F.conv2d(x if x.is_contiguous(memory_format=torch.channels_last) else x.contiguous(memory_format=torch.channels_last),
                     self.W[p + "proj.4.weight"], None if native else self.W[p + "proj.4.bias"], stride=2, padding=2)
        h, w = x.shape[2:]

        # ffn_with_coord.0 acts on cat([x, sine(patch centre)]): the position half does not depend on the input,
        # so it is folded into a per-position bias once per resolution and the concat disappears.
        w0, b0 = self.W[p + "ffn_with_coord.0.weight"], self.W[p + "ffn_with_coord.0.bias"]

        def coord_term():
            xy = coords_grid(1, h, w, x.device, x.dtype) * 8 + 4
            enc = sine_embed(xy.view(1, 2, -1).permute(0, 2, 1), COST_INPUT_DIM)          # (1, hw, 64)
            term = F.linear(enc, w0[:, COST_INPUT_DIM:, 0, 0], b0)                         # (1, hw, 128)
            if native:
                term = term + F.linear(self.W[p + "proj.4.bias"], w0[:, :COST_INPUT_DIM, 0, 0])
            return term.contiguous()
        term = self._memo(("pe", h, w, x.dtype, x.device, native), coord_term)
        t = x.permute(0, 2, 3, 1).reshape(M, h * w, COST_INPUT_DIM)                        # tokens (free view in NHWC)
        w2 = self.W[p + "ffn_with_coord.2.weight"][:, :, 0, 0]
        if native and torch.backends.cuda.matmul.allow_tf32:
            # linear, add_rows_relu_, linear, LayerNorm in one kernel (csrc/patch_tokens_tc.cu) with the same bits
            w0t, w2t = self._memo(("pe_tc", x.device), lambda: (self._ops.round_tf32(w0[:, :COST_INPUT_DIM, 0, 0]),
                                                                self._ops.round_tf32(w2)))
            return self._ops.patch_tokens_tc(t, w0t, term[0], w2t, self.W[p + "ffn_with_coord.2.bias"],
                                             self.W[p + "norm.weight"], self.W[p + "norm.bias"])
        t = F.linear(t, w0[:, :COST_INPUT_DIM, 0, 0])
        t = self._ops.add_rows_relu_(t, term[0]) if native else F.relu(t + term)
        t = F.linear(t, w2, self.W[p + "ffn_with_coord.2.bias"])
        return self._ln(t, p + "norm")

    def _latent_layer(self, x: Tensor, p: str) -> Tensor:
        """SelfAttentionLayer over the 8 latent tokens of each source pixel (core/encoder.py:97-140)."""
        y = self._ln(x, p + "norm1")
        a = self._attn(self._lin(y, p + "q"), self._lin(y, p + "k"), self._lin(y, p + "v"), 8)
        x, xn = self._add_ln(x, self._lin(a, p + "proj"), p + "norm2")
        return self._mlp_residual(x, xn, p, "ffn.0", "ffn.3")

    def _context_tokens(self, context: Tensor, p: str, reps: int) -> Tensor:
        """context_proj of the context map, tiled like `context.repeat(B//b, 1, 1, 1)` (twins.py:55-58):
        row i of the (B*8)-batch sees context[i % b] — a reference quirk that is kept."""
        b, _, H, W = context.shape
        c = self._lin(context.flatten(2).permute(0, 2, 1), p + "context_proj").view(b, H, W, -1)
        return c.repeat(reps, 1, 1, 1)

    def _vert_local_attn_native(self, x: Tensor, size, context: Tensor, p: str, ws: int, heads: int) -> Tensor:
        """Same function as `_vert_local_attn` with the projections split by linearity:
            q = Wq (cat[x, ctx] + enc) + bq = Wq[:, :C] x  +  (Wq[:, C:] ctx + Wq enc + bq)
        The second term only depends on (image index % 2, position): it is built once per layer on 2 x Hp x Wp tokens and
        added inside the attention kernel; x goes through ONE [q|k|v] GEMM whose output the kernel reads in place. Removes the
        192-channel concat, its window copy, the encoding add and two thirds of the GEMM launches (core/twins.py:46-114)."""
        Bt, N, C = x.shape
        H, W = size
        b = context.shape[0]
        wq, wk = self.W[p + "q.weight"], self.W[p + "k.weight"]
        enc = self._memo(("win", ws, C + VERT_C_DIM, x.dtype, x.device), lambda: sine_embed(
            coords_grid(1, ws, ws, x.device, x.dtype).view(1, 2, -1).permute(0, 2, 1), C + VERT_C_DIM))      # (1, 49, 192)
        cproj = self._lin(context.flatten(2).permute(0, 2, 1), p + "context_proj").view(b, H, W, -1)            # (b, H, W, 64)
        cw, meta = self._to_windows(cproj, ws)                                                                 # (b*nwin, 49, 64), zero padded
        w_qk_c = torch.cat([wq[:, C:], wk[:, C:]], 0)                                                          # (2C, 64)
        w_qk = torch.cat([wq, wk], 0)
        b_qk = torch.cat([self.W[p + "q.bias"], self.W[p + "k.bias"]], 0)
        terms = F.linear(cw, w_qk_c) + F.linear(enc, w_qk, b_qk)                                               # (b*nwin, 49, 2C)
        q_add, k_add = terms[..., :C].contiguous(), terms[..., C:].contiguous()
        w_x = self._memo(("vloc_w", p), lambda: torch.cat([wq[:, :C], wk[:, :C], self.W[p + "v.weight"]], 0).contiguous())
        b_x = self._memo(("vloc_b", p), lambda: torch.cat([torch.zeros(2 * C, device=x.device, dtype=x.dtype), self.W[p + "v.bias"]], 0))
        xw, meta = self._to_windows(x.view(Bt, H, W, C), ws)                                                   # (Bt*nwin, 49, C)
        qkv = F.linear(xw, w_x, b_x)
        # window n = image * nwin + wi; images repeat the b contexts cyclically -> additive slice = n % (b * nwin)
        o = self._ops.fused_qkv_attention(qkv, heads, q_add, k_add)
        return self._lin(self._from_windows(o, meta, ws, H, W), p + "proj")

    def _vert_local_attn(self, x: Tensor, size, context: Tensor, p: str, ws: int = 7, heads: int = 8) -> Tensor:
        if self._native(x) and (x.shape[-1] // heads) in (16, 32):
            return self._vert_local_attn_native(x, size, context, p, ws, heads)
        Bt, N, C = x.shape
        H, W = size
        ctx = self._context_tokens(context, p, Bt // context.shape[0])
        xg = x.view(Bt, H, W, C)
        xw, meta = self._to_windows(xg, ws)
        qkw, _ = self._to_windows(torch.cat([xg, ctx], dim=-1), ws)
        enc = self._memo(("win", ws, C + VERT_C_DIM, x.dtype, x.device), lambda: sine_embed(
            coords_grid(1, ws, ws, x.device, x.dtype).view(1, 2, -1).permute(0, 2, 1), C + VERT_C_DIM))
        qkw = qkw + enc
        o = self._attn(self._lin(qkw, p + "q"), self._lin(qkw, p + "k"), self._lin(xw, p + "v"), heads)
        return self._lin(self._from_windows(o, meta, ws, H, W), p + "proj")

    def _vert_global_attn_native(self, x: Tensor, size, context: Tensor, p: str, sr: int, heads: int) -> Tensor:
        """`_vert_global_attn` for H, W multiples of sr, projections split by linearity like the local variant:
        q = Wq[:, :C] x + T_q[image % b], and the strided key conv sr_key(cat[x, ctx]) = conv_x(x) + conv_c(ctx)[image % b]
        (core/twins.py:120-183). No 192-channel concat, no encoding add over the full map."""
        Bt, N, C = x.shape
        H, W = size
        b = context.shape[0]
        Cq = C + VERT_C_DIM
        wq = self.W[p + "q.weight"]
        cproj = self._lin(context.flatten(2).permute(0, 2, 1), p + "context_proj")                              # (b, N, 64)
        enc_full = self._memo(("full", H, W, Cq, x.dtype, x.device), lambda: sine_embed(
            coords_grid(1, H, W, x.device, x.dtype).view(1, 2, -1).permute(0, 2, 1), Cq))
        q_add = (F.linear(cproj, wq[:, C:]) + F.linear(enc_full, wq, self.W[p + "q.bias"])).contiguous()        # (b, N, C)
        q = F.linear(x, wq[:, :C])
        xg = x.view(Bt, H, W, C).permute(0, 3, 1, 2)
        wsk = self.W[p + "sr_key.weight"]
        wk_x = self._memo(("vglob_wkx", p), lambda: wsk[:, :C].contiguous(memory_format=torch.channels_last))
        wk_c = self._memo(("vglob_wkc", p), lambda: wsk[:, C:].contiguous(memory_format=torch.channels_last))
        k_ctx = F.conv2d(cproj.view(b, H, W, -1).permute(0, 3, 1, 2), wk_c, self.W[p + "sr_key.bias"], stride=sr)  # (b, C, h, w)
        k_in = F.conv2d(xg, wk_x, None, stride=sr).permute(0, 2, 3, 1)                                          # (Bt, h, w, C) rows
        M = k_in.shape[1] * k_in.shape[2]
        k_in = (k_in.reshape(Bt // b, b, M, C) + k_ctx.permute(0, 2, 3, 1).reshape(1, b, M, C)).view(Bt, M, C)  # image i: ctx i % b
        v_in = self._conv(xg, p + "sr_value", stride=sr).reshape(Bt, C, -1).permute(0, 2, 1)
        v_in, k_in = self._ln(v_in, p + "norm"), self._ln(k_in, p + "norm")
        enc_sub = self._memo(("sub", H // sr, W // sr, sr, C, x.dtype, x.device), lambda: sine_embed(
            coords_grid(1, H // sr, W // sr, x.device, x.dtype).view(1, 2, -1).permute(0, 2, 1) * sr, C))
        o = self._ops.attention_with_terms(q, self._lin(k_in + enc_sub, p + "k"), self._lin(v_in, p + "v"), heads, q_add)
        return self._lin(o, p + "proj")

    def _vert_global_attn(self, x: Tensor, size, context: Tensor, p: str, sr: int = 4, heads: int = 8) -> Tensor:
        if self._native(x) and size[0] % sr == 0 and size[1] % sr == 0 and (x.shape[-1] // heads) in (16, 32):
            return self._vert_global_attn_native(x, size, context, p, sr, heads)
        Bt, N, C = x.shape
        H, W = size
        ctx = self._context_tokens(context, p, Bt // context.shape[0])
        xg = x.view(Bt, H, W, C)
        qk = torch.cat([xg, ctx], dim=-1)
        pr, pb = (sr - W % sr) % sr, (sr - H % sr) % sr
        xg, qk = F.pad(xg, (0, 0, 0, pr, 0, pb)), F.pad(qk, (0, 0, 0, pr, 0, pb))
        Hp, Wp = H + pb, W + pr
        Cq = C + VERT_C_DIM
        enc_full = self._memo(("full", Hp, Wp, Cq, x.dtype, x.device), lambda: sine_embed(
            coords_grid(1, Hp, Wp, x.device, x.dtype).view(1, 2, -1).permute(0, 2, 1), Cq))
        q = self._lin(qk.reshape(Bt, Hp * Wp, Cq) + enc_full, p + "q")
        v_in = self._conv(xg.permute(0, 3, 1, 2), p + "sr_value", stride=sr).reshape(Bt, C, -1).permute(0, 2, 1)
        k_in = self._conv(qk.permute(0, 3, 1, 2), p + "sr_key", stride=sr).reshape(Bt, C, -1).permute(0, 2, 1)
        v_in, k_in = self._ln(v_in, p + "norm"), self._ln(k_in, p + "norm")
        enc_sub = self._memo(("sub", Hp // sr, Wp // sr, sr, C, x.dtype, x.device), lambda: sine_embed(
            coords_grid(1, Hp // sr, Wp // sr, x.device, x.dtype).view(1, 2, -1).permute(0, 2, 1) * sr, C))
        o = self._attn(q, self._lin(k_in + enc_sub, p + "k"), self._lin(v_in, p + "v"), heads)
        o = o.view(Bt, Hp, Wp, C)[:, :H, :W, :].reshape(Bt, N, C)
        return self._lin(o, p + "proj")

    def _vert_block(self, x: Tensor, size, context: Tensor, p: str, local: bool) -> Tensor:
        attn = self._vert_local_attn if local else self._vert_global_attn
        x, xn = self._add_ln(x, attn(self._ln(x, p + "norm1"), size, context, p + "attn."), p + "norm2")
        return self._mlp_residual(x, xn, p + "mlp.", "fc1", "fc2")

    def cost_perceiver(self, cost_volume: Tensor, context: Tensor) -> tuple[Tensor, Tensor]:
        c = "memory_encoder.cost_perceiver_encoder."
        B, heads, H1, W1, H2, W2 = cost_volume.shape
        assert heads == 1
        cost_maps = cost_volume.view(B * H1 * W1, 1, H2, W2)     # contiguous view: heads == 1
        tokens = self.patch_embed(cost_maps)                     # (B*N, hw, 128)
        # input_layer: 8 learned latents cross-attend to each pixel's patch tokens (encoder.py:150-191)
        p = c + "input_layer."
        lat = self.W[c + "latent_tokens"]                        # (1, 8, 128)
        M = tokens.shape[0]
        q = self._lin(self._ln(lat, p + "norm1"), p + "q")       # (1, 8, 128): shared by every source pixel
        if self._native(tokens) and torch.backends.cuda.matmul.allow_tf32 and LATENT_DIM == 128 and LATENT_TOKENS == 8:
            # K and V are never built: scores and pooling run on the token rows themselves (csrc/nn_kernels.cu)
            a = self._ops.latent_pool(tokens, q[0], self.W[p + "k.weight"], self.W[p + "v.weight"], self.W[p + "v.bias"])
        else:
            a = self._attn(q, self._lin(tokens, p + "k"), self._lin(tokens, p + "v"), 8)
        x = lat + self._lin(a, p + "proj")
        x = self._mlp_residual(x, self._ln(x, p + "norm2"), p, "ffn.0", "ffn.3")
        short_cut = x
        N = H1 * W1
        self._join_context()                                      # first use of the context map
        for i in range(ENCODER_DEPTH):
            x = self._latent_layer(x, c + f"encoder_layers.{i}.")
            x = x.view(B, N, LATENT_TOKENS, -1).permute(0, 2, 1, 3).reshape(B * LATENT_TOKENS, N, -1)
            v_ = c + f"vertical_encoder_layers.{i}."
            x = self._vert_block(x, (H1, W1), context, v_ + "local_block.", True)
            x = self._vert_block(x, (H1, W1), context, v_ + "global_block.", False)
            x = x.view(B, LATENT_TOKENS, N, -1).permute(0, 2, 1, 3).reshape(B * N, LATENT_TOKENS, -1)
        return x + short_cut, cost_maps

    def memory_encoder(self, img1: Tensor, img2: Tensor, context: Tensor, shared: tuple[int, int] | None = None) -> tuple[Tensor, Tensor]:
        """shared = (i, j): image2[j] IS image1[i] (the frontend batches [t2.L, t1.L] against [t2.R, t2.L], Frontend.py:284-285,
        so t2.L would be encoded twice in the same call): that image goes through the feature encoder once."""
        B = img1.shape[0]
        if shared is None:
            feats = self.svt(torch.cat([img1, img2], dim=0), "memory_encoder.feat_encoder")
            feats = self._conv(feats, "memory_encoder.channel_convertor")
            f1, f2 = feats[:B], feats[B:]
        else:
            i, j = shared
            if not (0 <= i < B and 0 <= j < B):
                raise ValueError(f"shared={shared}: image indices must lie in [0, {B})")
            keep = [k for k in range(B) if k != j]
            feats = self.svt(torch.cat([img1] + [img2[k:k + 1] for k in keep], dim=0), "memory_encoder.feat_encoder")
            feats = self._conv(feats, "memory_encoder.channel_convertor")
            f1 = feats[:B]
            f2 = torch.empty_like(f1)                                       # same (channels_last) layout as f1
            for pos, k in enumerate(keep):
                f2[k:k + 1].copy_(feats[B + pos:B + pos + 1])
            f2[j:j + 1].copy_(feats[i:i + 1])
            if self.taps is not None:
                feats = torch.cat([f1, f2], dim=0)
        self._tap("feats", feats)
        cost_volume = self.corr_fn(f1, f2).to(feats.dtype)                 # encoder.py:289-290
        self._tap("corr_rows", cost_volume.reshape(B, -1, cost_volume.shape[-2] * cost_volume.shape[-1])[:, ::97])
        out = self.cost_perceiver(cost_volume, context)
        self._tap("cost_memory", out[0])
        return out

    # ---- decoder (covhead.py:60-140) -----------------------------------------------------------
    def _gru(self, h: Tensor, x: Tensor, p: str) -> Tensor:
        for o, pad in (("1", (0, 2)), ("2", (2, 0))):
            hx = torch.cat([h, x], dim=1)
            zr = torch.sigmoid(self._conv(hx, p + f"convzr{o}", padding=pad))
            z, r = zr[:, :128], zr[:, 128:]
            q = torch.tanh(self._conv(torch.cat([r * h, x], dim=1), p + f"convq{o}", padding=pad))
            h = (1 - z) * h + z * q
        return h

    def _gru_native(self, hx: Tensor, rhx: Tensor, z: Tensor, p: str, h_dense: Tensor, shape) -> None:
        """SepConvGRU (gru.py:22-43) on the NHWC [h|x] / [r*h|x] buffers: 2 convs + 2 fused kernels per pass."""
        B, H, W = shape
        hx_map, rhx_map = (t.view(B, H, W, 512).permute(0, 3, 1, 2) for t in (hx, rhx))
        for o, pad in (("1", (0, 2)), ("2", (2, 0))):
            zr = F.conv2d(hx_map, self.W[p + f"convzr{o}.weight"], None, padding=pad)      # biases folded into the gate kernels
            self._ops.gru_gates(zr.permute(0, 2, 3, 1), hx, z, rhx, self.W[p + f"convzr{o}.bias"])
            q = F.conv2d(rhx_map, self.W[p + f"convq{o}.weight"], None, padding=pad)
            self._ops.gru_blend(q.permute(0, 2, 3, 1), z, hx, h_dense if o == "2" else None, self.W[p + f"convq{o}.bias"])

    def _make_decoder_tc(self, B: int, H: int, W: int, device):
        """Buffers (fp16 padded pixel rows, csrc/rows_layout.cuh) and packed filters of the tensor-core decoder iteration
        (csrc/conv_tc.cu): motion encoder, value projection, flow head, covariance head."""
        from types import SimpleNamespace
        ops, m = self._ops, "memory_decoder."
        e, ub, cu = m + "update_block.encoder.", m + "update_block.", m + "cov_update."
        rows, P = ops.rows_count(B, H, W), B * H * W
        u16 = lambda c: torch.zeros(rows, c, dtype=torch.float16, device=device)
        t = SimpleNamespace(shape=(B, H, W))
        t.tok16, t.c1, t.cp, t.f1, t.mf16 = u16(192), u16(256), u16(256), u16(128), u16(128)
        t.fh, t.ch1, t.ch2, t.ch3 = u16(256), u16(256), u16(128), u16(64)
        t.f0 = torch.zeros(P, 128, dtype=torch.float16, device=device)            # im2col rows of the flow (dense)
        t.v16 = torch.zeros(P, 128, dtype=torch.float16, device=device)
        t.mf32 = torch.zeros(P, 128, dtype=torch.float32, device=device)
        t.d_flow, t.d_cov = (torch.zeros(P, 2, dtype=torch.float32, device=device) for _ in range(2))
        pk = lambda name, cin=None: ops.pack_conv_filter(self.W[name + ".weight"], self.W.get(name + ".bias"), cin, device)
        t.convc1 = pk(e + "convc1p", 192)
        t.convc2, t.convf2, t.conv = pk(e + "convc2"), pk(e + "convf2"), pk(e + "conv")
        wf1 = self.W[e + "convf1.weight"]                                          # (128, 2, 7, 7) -> 1x1 over the 98 im2col columns
        t.convf1 = ops.pack_conv_filter(wf1.permute(0, 2, 3, 1).reshape(wf1.shape[0], 98, 1, 1), self.W[e + "convf1.bias"], 128, device)
        t.to_v = pk(ub + "aggregator.to_v")
        t.fh1, t.fh2 = pk(ub + "flow_head.conv1"), pk(ub + "flow_head.conv2")
        t.chw = [pk(cu + f"cov_head.conv{i}") for i in (1, 2, 3, 4)]
        return t

    @staticmethod
    def convex_upsample(flow: Tensor, mask: Tensor) -> Tensor:
        """`upsample_flow` (decoder.py:131-139): softmax over the 9 neighbours, 8x."""
        N, C, H, W = flow.shape
        mask = mask.reshape(N, 9, 8, 8, H, W).softmax(dim=1)
        up = F.unfold(8 * flow, (3, 3), padding=1).view(N, C, 9, H, W)
        out = (mask.unsqueeze(1) * up.unsqueeze(-3).unsqueeze(-3)).sum(dim=2)
        return out.permute(0, 1, 4, 2, 5, 3).reshape(N, C, 8 * H, 8 * W)

    def _decoder_mode(self, ctx: Tensor) -> str:
        """How the refinement loop runs: "tf32" (fp32 CUDA net with TF32 matmuls AND convolutions allowed: every iteration on
        our kernels, the tensor-core ones included), "strict" (fp32 CUDA net otherwise: token kernel + cuDNN fp32 convolutions
        + the SepConvGRU glue kernels), "torch" (CPU golden runs, half-precision `native` runs: torch ops)."""
        if not (self._native(ctx) and self.dec_dtype == torch.float32):
            return "torch"
        if torch.backends.cuda.matmul.allow_tf32 and torch.backends.cudnn.allow_tf32:
            return "tf32"
        return "strict"

    def memory_decoder(self, cost_memory: Tensor, context: Tensor, cost_maps: Tensor) -> tuple[Tensor, Tensor]:
        m, dd = "memory_decoder.", self.dec_dtype
        cost_memory = cost_memory.to(dd)
        B, _, H1, W1 = context.shape
        coords0 = coords_grid(B, H1, W1, context.device, context.dtype)
        coords1, ccoords1 = coords0.clone(), coords0.clone()
        ctx = self._conv(context, m + "proj")
        net = ctx[:, :128].tanh().to(dd)
        cnet = net.clone()
        inp = ctx[:, 128:].relu().to(dd)
        mode = self._decoder_mode(ctx)
        # GMA attention, once per frame (gma.py:39-82): softmax over the N x N similarity
        qk = self._conv(inp, m + "att.to_qk")
        qv = (qk[:, :128] * (128 ** -0.5)).flatten(2).transpose(1, 2)            # (B, N, 128)
        scores = torch.matmul(qv, qk[:, 128:].flatten(2))                        # (B, N, N)
        # the N x N GMA attention matrix (184 MB at 640x480) is re-read by every iteration's aggregation GEMM, which is
        # bound by that read: when TF32 matmuls are allowed it is kept in fp16 (values in [0, 1]; no precision below TF32's)
        half_attention = mode != "torch" and torch.backends.cuda.matmul.allow_tf32
        if half_attention and scores.shape[-1] % 4 == 0 and scores.shape[-1] <= 8192:
            attention = self._ops.softmax_rows_f16(scores)         # softmax + fp16 in one pass over the scores
        else:
            attention = scores.softmax(dim=-1)
            if half_attention:
                attention = attention.to(torch.float16)
        ca = m + "decoder_layer.cross_attend."
        key = self._lin(cost_memory, ca + "k")
        value = self._lin(cost_memory, ca + "v")
        refine = {"tf32": self._refine_tf32, "strict": self._refine_strict, "torch": self._refine_torch}[mode]
        coords1, ccoords1, net, cnet = refine(coords0, coords1, ccoords1, net, cnet, inp, attention, key, value, cost_maps)
        # the reference evaluates both mask heads + upsampling every iteration but (eval mode) returns
        # only the last one (covhead.py:137-140) -> evaluate once
        ub, cu = m + "update_block.", m + "cov_update."
        if mode != "torch":     # scale + softmax + unfold + weighted sum + pixel shuffle in one kernel per map
            up_logits = self._conv(self._conv_relu(net, ub + "mask.0", padding=1), ub + "mask.2")
            cov_logits = self._conv(self._conv_relu(cnet, cu + "mask.0", padding=1), cu + "mask.2")
            return (self._ops.convex_upsample(coords1 - coords0, up_logits, 0.25),
                    self._ops.convex_upsample(ccoords1 - coords0, cov_logits, 0.25))
        up_mask = _f32(0.25 * self._conv(F.relu(self._conv(net, ub + "mask.0", padding=1)), ub + "mask.2"))
        cov_mask = _f32(0.25 * self._conv(F.relu(self._conv(cnet, cu + "mask.0", padding=1)), cu + "mask.2"))
        return self.convex_upsample(coords1 - coords0, up_mask), self.convex_upsample(ccoords1 - coords0, cov_mask)

    def _refine_tf32(self, coords0, coords1, ccoords1, net, cnet, inp, attention, key, value, cost_maps):
        """The whole iteration on our kernels: lookup, token kernel, motion encoder / value projection / heads on the
        tensor-core convolution kernel (fp16 rows between the layers), both SepConvGRU units on their tensor-core kernel (fp16
        operands, fp32 state; csrc/gru_conv_tc.cu); the one library call left is the GMA aggregation GEMM over the fp16
        `attention`."""
        m = "memory_decoder."
        ub, cu = m + "update_block.", m + "cov_update."
        ops = self._ops
        B, _, H1, W1 = coords0.shape
        N, dev = H1 * W1, coords0.device
        P, shp = B * N, (B, H1, W1)
        side = self._memo(("side_stream", dev), lambda: torch.cuda.Stream(dev))
        side2 = self._memo(("side_stream2", dev), lambda: torch.cuda.Stream(dev))
        as_map = lambda t: t.view(B, H1, W1, -1).permute(0, 3, 1, 2)                   # channels_last logical map

        def make_gru():
            names = [f"conv{g}{o}" for g in ("zr", "q") for o in ("1", "2")]
            ws = [{n: self.W[pre + "gru." + n + ".weight"] for n in names} for pre in (ub, cu)]
            bs = [{n: self.W[pre + "gru." + n + ".bias"] for n in names} for pre in (ub, cu)]
            return ops.SepConvGruTC(ws, bs, B, H1, W1, dev)
        gru = self._memo(("gru_tc", B, H1, W1, dev), make_gru)
        t = self._memo(("decoder_tc", B, H1, W1, dev), lambda: self._make_decoder_tc(B, H1, W1, dev))
        gru.set_context(inp.permute(0, 2, 3, 1).reshape(P, 128).contiguous())
        net_rows = net.permute(0, 2, 3, 1).reshape(P, 128).contiguous()
        gru.set_state(0, net_rows)
        gru.set_state(1, net_rows)
        net_d, cnet_d = gru.h
        token_blob = self._memo(("token_blob", dev), lambda: ops.decoder_token_blob(self.W, m))
        key, value = key.contiguous(), value.contiguous()
        gamma = self.W[ub + "aggregator.gamma"]
        cov_done = None
        for _ in range(self.depth):
            main = torch.cuda.current_stream()
            fork = torch.cuda.Event()
            fork.record(main)
            with torch.cuda.stream(side):                                                # flow branch of the motion encoder
                side.wait_event(fork)
                ops.flow_im2col(coords1, coords0, t.f0, t.mf32, t.mf16)
                ops.conv_tc(t.f0, t.convf1[0], t.convf1[1], 128, 1, True, shp, in_dense=True, out16=t.f1)
                ops.conv_tc(t.f1, t.convf2[0], t.convf2[1], 64, 3, True, shp, out16=t.cp, out16_offset=192)
                joinf = torch.cuda.Event()
                joinf.record(side)
            cf = ops.corr_lookup(cost_maps, coords1, rows=True)                          # (P, 81)
            ops.decoder_token(cf, coords1, key, value, token_blob, out16_rows=t.tok16)   # rows [global | forward | 0] in fp16
            ops.conv_tc(t.tok16, t.convc1[0], t.convc1[1], 256, 1, True, shp, out16=t.c1)
            ops.conv_tc(t.c1, t.convc2[0], t.convc2[1], 192, 3, True, shp, out16=t.cp)
            main.wait_event(joinf)
            ops.conv_tc(t.cp, t.conv[0], t.conv[1], 126, 3, True, shp, out16=t.mf16, out32=t.mf32)   # + flow in channels 126, 127
            ops.conv_tc(t.mf16, t.to_v[0], None, 128, 1, False, shp, out16=t.v16, out16_dense=True)
            agg = torch.bmm(attention, t.v16.view(B, N, 128), out_dtype=torch.float32)   # GMA aggregation (gma.py:84-130)
            if cov_done is not None:            # the previous iteration's covariance head still reads the covariance unit's state rows
                main.wait_event(cov_done)
            # one launch chain per GRU unit on two streams; the covariance unit's chain ends in `unit1_done`, which only the
            # covariance head waits for
            unit1_done = gru.step(t.mf32, agg.view(P, 128), gamma)
            # The covariance head (4 chained convolutions, covhead.py:20-58) feeds only the covariance coordinates: it runs on
            # its own stream and is joined right before the NEXT iteration's GRU update, so it overlaps the next lookup / token
            # kernel / motion encoder instead of extending this iteration (they depend on the flow head only).
            with torch.cuda.stream(side2):
                side2.wait_event(unit1_done)
                ops.conv_tc(gru.h_rows[0][1], t.chw[0][0], t.chw[0][1], 256, 3, True, shp, out16=t.ch1)
                ops.conv_tc(t.ch1, t.chw[1][0], t.chw[1][1], 128, 3, False, shp, out16=t.ch2)
                ops.conv_tc(t.ch2, t.chw[2][0], t.chw[2][1], 64, 3, True, shp, out16=t.ch3)
                ops.conv_tc(t.ch3, t.chw[3][0], t.chw[3][1], 2, 3, False, shp, add_to_map=ccoords1)   # ccoords1 += delta (in the epilogue)
                cov_done = torch.cuda.Event()
                cov_done.record(side2)
            ops.conv_tc(gru.h_rows[0][0], t.fh1[0], t.fh1[1], 256, 3, True, shp, out16=t.fh)
            ops.conv_tc(t.fh, t.fh2[0], t.fh2[1], 2, 3, False, shp, add_to_map=coords1)               # coords1 += delta_flow
            if self.taps is not None:
                main.wait_event(cov_done)
            net, cnet = as_map(net_d), as_map(cnet_d)
            self._tap("flow_iter", coords1 - coords0)
            self._tap("cov_iter", ccoords1 - coords0)
        if cov_done is not None:
            torch.cuda.current_stream().wait_event(cov_done)
        return coords1, ccoords1, net, cnet

    def _refine_strict(self, coords0, coords1, ccoords1, net, cnet, inp, attention, key, value, cost_maps):
        """fp32 everywhere the flags ask for it: lookup and token kernel rows into cuDNN's convolutions, SepConvGRU as cuDNN
        convolutions + the glue kernels of csrc/decoder_fused.cu on NHWC `[h | x]` state buffers. `attention` is fp16 when
        TF32 matmuls are allowed (the aggregation then reads it like the tf32 mode does), fp32 otherwise."""
        m, dd = "memory_decoder.", torch.float32
        ub, cu, e = m + "update_block.", m + "cov_update.", m + "update_block.encoder."
        ops = self._ops
        B, _, H1, W1 = coords0.shape
        P, dev = B * H1 * W1, coords0.device
        side = self._memo(("side_stream", dev), lambda: torch.cuda.Stream(dev))
        as_map = lambda t: t.view(B, H1, W1, -1).permute(0, 3, 1, 2)                   # channels_last logical map
        inp_rows = inp.permute(0, 2, 3, 1).reshape(P, 128).contiguous()
        net_rows = net.permute(0, 2, 3, 1).reshape(P, 128).contiguous()
        # recurrent state in NHWC [h | x] buffers (csrc/decoder_fused.cu): x = [inp | mf | mf + gamma*agg]
        bufs = [torch.empty(P, 512, dtype=dd, device=dev) for _ in range(4)]   # hx, rhx (flow) / hx, rhx (cov)
        for bf in bufs:
            bf[:, 128:256] = inp_rows
        bufs[0][:, :128] = net_rows
        bufs[2][:, :128] = bufs[0][:, :128]
        zbuf, zbuf2 = torch.empty(P, 128, dtype=dd, device=dev), torch.empty(P, 128, dtype=dd, device=dev)
        net_d, cnet_d = torch.empty(P, 128, dtype=dd, device=dev), torch.empty(P, 128, dtype=dd, device=dev)
        token_blob = self._memo(("token_blob", dev), lambda: ops.decoder_token_blob(self.W, m))
        key, value = key.contiguous(), value.contiguous()
        gamma = self.W[ub + "aggregator.gamma"]
        for _ in range(self.depth):
            flow = coords1 - coords0
            # pixels-major rows end to end: lookup kernel -> ONE token kernel (token MLP, LayerNorm + sine embedding, q
            # projection, per-pixel 8x8 cross attention, output projection, FFN) writing the motion encoder's input rows
            cf = ops.corr_lookup(cost_maps, coords1, rows=True)                          # (P, 81)
            corr = ops.decoder_token(cf, coords1, key, value, token_blob)                # (P, 160) = [global | forward | 0]
            corr = corr.view(B, H1, W1, 160).permute(0, 3, 1, 2)                         # channels_last view
            # motion encoder (gru.py:45-64), its flow branch on the side stream
            main = torch.cuda.current_stream()
            fork = torch.cuda.Event()
            fork.record(main)
            with torch.cuda.stream(side):
                side.wait_event(fork)
                flo = self._conv_relu(self._conv_relu(flow, e + "convf1", padding=3), e + "convf2", padding=1)
                joinf = torch.cuda.Event()
                joinf.record(side)
            cor = self._conv_relu(self._conv_relu(corr, e + "convc1p"), e + "convc2", padding=1)
            main.wait_event(joinf)
            # 128-channel conv output (last two channels zero), flow written into them in place
            mf = self._conv_relu(torch.cat([cor, flo], dim=1), e + "convp", padding=1)
            mf.permute(0, 2, 3, 1)[..., 126:] = flow.permute(0, 2, 3, 1)
            # GMA aggregation (gma.py:84-130)
            mf = mf.contiguous(memory_format=torch.channels_last)
            v = self._conv(mf, ub + "aggregator.to_v").flatten(2).transpose(1, 2)   # (B, N, 128)
            if attention.dtype == torch.float16:      # fp16 operands (11-bit mantissa >= TF32's 10), fp32 accumulate AND output
                agg = torch.bmm(attention, v.to(torch.float16), out_dtype=torch.float32)
            else:
                agg = torch.matmul(attention, v)                                    # (B, N, 128) = pixels-major
            # the flow branch (GRU + flow head) and the covariance branch (GRU + cov head) only share their input:
            # at 60x80 each conv fills about two thirds of the 132 SMs, so the two run on forked streams (fork/join is
            # captured into the CUDA graph as parallel branches)
            ops.gru_input(mf.permute(0, 2, 3, 1), agg, gamma, bufs)
            main = torch.cuda.current_stream()
            fork = torch.cuda.Event()
            fork.record(main)
            with torch.cuda.stream(side):
                side.wait_event(fork)
                self._gru_native(bufs[2], bufs[3], zbuf2, cu + "gru.", cnet_d, (B, H1, W1))
                cnet = as_map(cnet_d)
                h = cu + "cov_head."
                t = self._conv(self._conv_relu(cnet, h + "conv1", padding=1), h + "conv2", padding=1)
                d_cov = self._conv(self._conv_relu(t, h + "conv3", padding=1), h + "conv4", padding=1)
                join = torch.cuda.Event()
                join.record(side)
            self._gru_native(bufs[0], bufs[1], zbuf, ub + "gru.", net_d, (B, H1, W1))
            net = as_map(net_d)
            d_flow = self._conv(self._conv_relu(net, ub + "flow_head.conv1", padding=1), ub + "flow_head.conv2", padding=1)
            main.wait_event(join)
            coords1 = coords1 + d_flow
            ccoords1 = ccoords1 + d_cov
            self._tap("flow_iter", coords1 - coords0)
            self._tap("cov_iter", ccoords1 - coords0)
        return coords1, ccoords1, net, cnet

    def _refine_torch(self, coords0, coords1, ccoords1, net, cnet, inp, attention, key, value, cost_maps):
        """torch ops in the decoder dtype, `lookup_fn` for the window lookup: the CPU golden runs (float32 / float64) and the
        half-precision `native` runs."""
        m, dd = "memory_decoder.", self.dec_dtype
        ub, cu, e = m + "update_block.", m + "cov_update.", m + "update_block.encoder."
        ca = m + "decoder_layer.cross_attend."
        B, _, H1, W1 = coords0.shape
        P = B * H1 * W1
        gamma = self.W[ub + "aggregator.gamma"]
        for _ in range(self.depth):
            flow = (coords1 - coords0).to(dd)
            cost_forward = self.lookup_fn(cost_maps, coords1).to(dd)         # fp32 lookup (covhead.py:91-93)
            query = self._conv(F.gelu(self._conv(cost_forward, m + "flow_token_encoder.0")), m + "flow_token_encoder.2")
            query = query.permute(0, 2, 3, 1).reshape(P, QUERY_DIM)          # rows = pixels (2-D: plain GEMMs below)
            # cross attention of each pixel's query to its 8 cost-memory tokens (decoder.py:56-76)
            enc = sine_embed(coords1.to(dd).permute(0, 2, 3, 1).reshape(P, 2), QUERY_DIM)
            qin = self._ln(query, ca + "norm1") + enc
            q = self._lin(qin, ca + "q")
            a = self._attn(q.unsqueeze(1), key, value, 8).squeeze(1)
            g = query + self._lin(torch.cat([a, query], dim=1), ca + "proj")
            g = g + self._lin(F.gelu(self._lin(self._ln(g, ca + "norm2"), ca + "ffn.0")), ca + "ffn.3")
            cost_global = g.view(B, H1, W1, QUERY_DIM).permute(0, 3, 1, 2)
            corr = torch.cat([cost_global, cost_forward], dim=1)
            # motion encoder (gru.py:45-64)
            cor = self._conv_relu(self._conv_relu(corr, e + "convc1"), e + "convc2", padding=1)
            flo = self._conv_relu(self._conv_relu(flow, e + "convf1", padding=3), e + "convf2", padding=1)
            mf = torch.cat([self._conv_relu(torch.cat([cor, flo], dim=1), e + "conv", padding=1), flow], dim=1)
            # GMA aggregation (gma.py:84-130)
            mf = mf.contiguous(memory_format=torch.channels_last)
            v = self._conv(mf, ub + "aggregator.to_v").flatten(2).transpose(1, 2)   # (B, N, 128)
            agg = torch.matmul(attention, v)                                    # (B, N, 128) = pixels-major
            inp_cat = torch.cat([inp, mf, mf + gamma * agg.transpose(1, 2).reshape(B, 128, H1, W1)], dim=1)
            net = self._gru(net, inp_cat, ub + "gru.")
            cnet = self._gru(cnet, inp_cat, cu + "gru.")
            d_flow = self._conv(self._conv_relu(net, ub + "flow_head.conv1", padding=1), ub + "flow_head.conv2", padding=1)
            h = cu + "cov_head."
            t = self._conv(self._conv_relu(cnet, h + "conv1", padding=1), h + "conv2", padding=1)
            d_cov = self._conv(self._conv_relu(t, h + "conv3", padding=1), h + "conv4", padding=1)
            coords1 = coords1 + _f32(d_flow)
            ccoords1 = ccoords1 + _f32(d_cov)
            self._tap("flow_iter", coords1 - coords0)
            self._tap("cov_iter", ccoords1 - coords0)
        return coords1, ccoords1, net, cnet

    # ---- top level (flownet.py:18-44) -----------------------------------------------------------
    @torch.inference_mode()
    def forward(self, image1: Tensor, image2: Tensor, shared: tuple[int, int] | None = None) -> tuple[Tensor, Tensor]:
        image1 = ((2 * image1) - 1.0).to(self.enc_dtype)
        image2 = ((2 * image2) - 1.0).to(self.enc_dtype)
        self._ctx_join = None
        if self._ops is not None and image1.is_cuda:
            # the context encoder (a chain of small kernels on 2 images) is independent of the feature encoder, the
            # correlation volume and PatchEmbed: it runs on a forked stream and is joined where the cost perceiver first
            # needs the context (its vertical layers)
            main = torch.cuda.current_stream()
            side = self._memo(("side_stream", image1.device), lambda: torch.cuda.Stream(image1.device))
            fork = torch.cuda.Event()
            fork.record(main)
            with torch.cuda.stream(side):
                side.wait_event(fork)
                context = self.svt(image1, "context_encoder")
                self._ctx_join = torch.cuda.Event()
                self._ctx_join.record(side)
            context.record_stream(main)
        else:
            context = self.svt(image1, "context_encoder")
        if self.taps is not None:
            self._join_context()
            self._tap("context", context)
        cost_memory, cost_maps = self.memory_encoder(image1, image2, context, shared)
        self._join_context()
        return self.memory_decoder(cost_memory, _f32(context), _f32(cost_maps))

    def _join_context(self) -> None:
        if getattr(self, "_ctx_join", None) is not None:
            torch.cuda.current_stream().wait_event(self._ctx_join)
            self._ctx_join = None

    @torch.inference_mode()
    def inference(self, image1: Tensor, image2: Tensor, shared: tuple[int, int] | None = None) -> tuple[Tensor, Tensor]:
        """(B,3,H,W) x2 in [0,1] -> flow (B,2,H,W), cov = exp(2 log sigma) (B,2,H,W); shared = (i, j) promises that image2[j] is
        image1[i] (it is then encoded once, see `memory_encoder`)."""
        H, W = image1.shape[-2:]
        ph, pw = (-H) % 8, (-W) % 8
        pad = [pw // 2, pw - pw // 2, ph // 2, ph - ph // 2]       # InputPadder 'sintel' (core/utils.py:4-24)
        if ph or pw:
            image1, image2 = F.pad(image1, pad, mode="replicate"), F.pad(image2, pad, mode="replicate")
        flow, logsig = self.forward(image1, image2, shared)
        if ph or pw:
            flow = flow[..., pad[2]:flow.shape[-2] - pad[3], pad[0]:flow.shape[-1] - pad[1]]
            logsig = logsig[..., pad[2]:logsig.shape[-2] - pad[3], pad[0]:logsig.shape[-1] - pad[1]]
        return flow, torch.exp(logsig * 2)
