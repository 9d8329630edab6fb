"""Argument checks of every ops wrapper on the device, with the library replaced by a stub that records calls: host-only
size queries go to the real library, every other entry point is recorded and returns 0 without running anything. A missing
check therefore shows up as a recorded call, never as a launch. Device 1 is simulated on one GPU by making ops report it as
the current device while every operand stays on cuda:0."""
import ctypes as C
import types

import pytest
import torch

from tests.test_cabi_load import HOST_ONLY, NEEDS_CUDA_BUFFERS

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


class _StubLibrary:
    def __init__(self, ops, real):
        self.ops, self.real, self.calls = ops, real, []

    def __getattr__(self, name):
        if self.ops.EXPORTS[name][0] is C.c_size_t:        # pure host size queries
            return getattr(self.real, name)
        return lambda *args: self.calls.append(name) or 0


@pytest.fixture
def ops(monkeypatch):
    from macvo_b200 import build, ops
    build.build(verbose=False)
    stub = _StubLibrary(ops, ops.load_library())
    monkeypatch.setattr(ops, "_lib", stub)
    monkeypatch.setattr(ops, "stub", stub, raising=False)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", True)      # stereo_head runs only under TF32
    return ops


def z(*shape, dtype=torch.float32):
    return torch.zeros(*shape, dtype=dtype, device=DEV)


def f64(*shape):
    return z(*shape, dtype=torch.float64)


def strided(t):
    """the same shape and dtype, not contiguous"""
    return torch.zeros(*t.shape, 2, dtype=t.dtype, device=t.device)[..., 0]


def _gru(ops):
    names = {"convzr1": (256, 512, 1, 5), "convq1": (128, 512, 1, 5), "convzr2": (256, 512, 5, 1), "convq2": (128, 512, 5, 1)}
    return ops.SepConvGruTC([{n: torch.zeros(s) for n, s in names.items()}], [{n: torch.zeros(s[0]) for n, s in names.items()}],
                            1, 2, 2, DEV)


def _device_calls(ops):
    """one valid call per public wrapper (and per SepConvGruTC method that launches), every operand on cuda:0"""
    pgo = lambda: [f64(5, 3), f64(5, 2), f64(5), f64(5, 3), f64(5)]
    intr = (1.0, 1.0, 1.0, 1.0, 1.0)
    score = lambda: ops.ScoreBuffers(4, 4, DEV, 5)
    cand = lambda: ops.CandidateList(4, 4, DEV)
    exchange = types.SimpleNamespace(ptrs=(C.c_void_p * 1)(), world=1, rank=0)
    rows = lambda c: z(ops.rows_count(1, 2, 2), c, dtype=torch.float16)
    maps = lambda: [z(1, 1, 4, 4) for _ in range(4)]

    def depth_aware_score():
        s = score()
        s.flow_quality, s.cand_vals2 = z(4, 4), z(16)
        return s

    def counted(n):
        c = cand()
        c.host[0] = n
        c.n.fill_(n)
        return c

    return {
        "corr_build": lambda: ops.corr_build(z(1, 64, 4, 4), z(1, 64, 4, 4)),
        "corr_lookup": lambda: ops.corr_lookup(z(16, 1, 4, 4), z(1, 2, 4, 4)),
        "dense_postproc": lambda: ops.dense_postproc(z(2, 2, 4, 4), z(2, 2, 4, 4), 80.0, score=score()),
        "score_only": lambda: ops.score_only(z(1, 3, 4, 4), score()),
        "score_depth_aware": lambda: ops.score_depth_aware(z(1, 3, 4, 4), z(1, 1, 4, 4), z(1, 1, 4, 4), score()),
        "select_candidates_depth": lambda: ops.select_candidates_depth(depth_aware_score(), z(1, 1, 4, 4), z(1, 1, 4, 4),
                                                                       z(1, 1, 4, 4), 4, 10.0, 1.0, 1.0, None, None, cand()),
        "select_candidates": lambda: ops.select_candidates(score(), 4, 1.0, z(1, 1, 4, 4, dtype=torch.bool), cand()),
        "select_mapping_candidates": lambda: ops.select_mapping_candidates(z(1, 1, 4, 4), z(1, 1, 4, 4), 4, 10.0, 1.0, cand()),
        "sample_from_counts": lambda: ops.sample_from_counts([(counted(3), 2)]),
        "sample_candidates": lambda: ops.sample_candidates(counted(3), 2),
        "sample_candidates_many": lambda: ops.sample_candidates_many([(counted(3), 2)]),
        "retrieve_pixels": lambda: ops.retrieve_pixels(z(5, 2, dtype=torch.int64), z(1, 1, 4, 4)),
        "match_covariance": lambda: ops.match_covariance(z(5, 2, dtype=torch.int64), z(1, 1, 4, 4), z(5, 3), 1.0, 1.0, 1.0, 1.0),
        "pgo_solve": lambda: ops.pgo_solve(*pgo(), intr, f64(7)),
        "pgo_solve_graph": lambda: ops.pgo_solve_graph("disp", pgo()[0], intr, f64(7), *pgo()[1:]),
        "pgo_accumulate": lambda: ops.pgo_accumulate(*pgo(), intr, f64(7)),
        "pgo_solve_sharded": lambda: ops.pgo_solve_sharded(pgo(), intr, f64(7), exchange, k_total=z(1, dtype=torch.int32)),
        "motion_interpolate_": lambda: ops.motion_interpolate_(z(3, 7), z(3, dtype=torch.bool)),
        "cov_sanity_filter": lambda: ops.cov_sanity_filter(f64(3, 3, 3), f64(3, 3, 3)),
        "cov_modify": lambda: ops.cov_modify(f64(3, 3, 3), ["diagonalize"]),
        "observe_pack": lambda: ops.observe_pack(ops.ObservationBuffers(8, DEV), z(5, 2, dtype=torch.int64), z(1, 2, 4, 4),
                                                 z(1, 3, 4, 4), *maps(), 1, (1, 1, 1, 1), (1, 1, 1, 1), f64(7), f64(7),
                                                 ext=dict(depth_cov0=z(1, 1, 4, 4))),
        "pgo_solve_counted": lambda: ops.pgo_solve_counted(ops.ObservationBuffers(8, DEV), intr, f64(7), f64(8)),
        "layer_norm": lambda: ops.layer_norm(z(4, 128), z(128), z(128)),
        "add_layer_norm": lambda: ops.add_layer_norm(z(4, 128), z(4, 128), z(128), z(128)),
        "mlp_tc": lambda: ops.mlp_tc(z(4, 128), z(4, 128), z(128, 128), z(128), z(128, 128), z(128)),
        "patch_tokens_tc": lambda: ops.patch_tokens_tc(z(4, 64), z(128, 64), z(2, 128), z(128, 128), z(128), z(128), z(128)),
        "patch_embed_conv1": lambda: ops.patch_embed_conv1(z(2, 1, 8, 8), z(16, 1, 6, 6), z(16)),
        "small_attention": lambda: ops.small_attention(z(2, 4, 128), z(2, 4, 128), z(2, 4, 128), 8),
        "gru_input": lambda: ops.gru_input(z(8, 128), z(8, 128), z(1), [z(8, 512)]),
        "gru_gates": lambda: ops.gru_gates(z(8, 256), z(8, 512), z(8, 128), z(8, 512)),
        "gru_blend": lambda: ops.gru_blend(z(8, 128), z(8, 128), z(8, 512), None),
        "conv_tc": lambda: ops.conv_tc(rows(64), z(32, 64, dtype=torch.float16), None, 32, 1, False, (1, 2, 2), out32=z(4, 32)),
        "flow_im2col": lambda: ops.flow_im2col(z(1, 2, 2, 2), z(1, 2, 2, 2), z(4, 128, dtype=torch.float16), z(4, 128), rows(128)),
        "pack_rows": lambda: ops.pack_rows(z(4, 64), rows(64), 0, (1, 2, 2)),
        "SepConvGruTC.set_context": lambda: _gru(ops).set_context(z(4, 128)),
        "SepConvGruTC.set_state": lambda: _gru(ops).set_state(0, z(4, 128)),
        "SepConvGruTC.step": lambda: _gru(ops).step(z(4, 128), z(4, 128), z(1)),
        "convex_upsample": lambda: ops.convex_upsample(z(1, 2, 4, 4), z(1, 576, 4, 4)),
        "softmax_rows_f16": lambda: ops.softmax_rows_f16(z(4, 8)),
        "decoder_token": lambda: ops.decoder_token(z(4, 81), z(1, 2, 2, 2), z(4, 8, 64), z(4, 8, 64), z(10)),
        "add_rows_relu_": lambda: ops.add_rows_relu_(z(2, 80, 128), z(80, 128)),
        "fused_qkv_attention": lambda: ops.fused_qkv_attention(z(2, 49, 384), 8),
        "attention_with_terms": lambda: ops.attention_with_terms(z(2, 4, 128), z(2, 4, 128), z(2, 4, 128), 8),
        "latent_pool": lambda: ops.latent_pool(z(2, 80, 128), z(8, 128), z(128, 128), z(128, 128), z(128)),
        "posenet_input": lambda: ops.posenet_input(z(1, 2, 112, 160), z(1, 1, 112, 160), 1.0, z(1, 5, 112, 160)),
        "posenet_conv": lambda: ops.posenet_conv(z(8, 4, 4), z(32 * 8 * 9), 1, z(32), 3, 1, 1),
        "posenet_head": lambda: ops.posenet_head(z(256), z(ops.posenet_head_floats()), f64(7), z(6), f64(7)),
        "pwc_warp_corr": lambda: ops.pwc_warp_corr(z(1, 4, 4, 4), z(1, 4, 4, 4), None, 1.0, z(1, 81, 4, 4), 0),
        "stereo_head": lambda: ops.stereo_head(z(1, 64, 2, 3), None, z(1, 64, 2, 3), z(4, 4, 4, 64, 32),
                                               z(ops.STEREO_HEAD_SMALL), None, None, 1.0, (0, 0), z(1, 1, 4, 6), None),
    }


def _refused(ops, call):
    """the call raises MacvoB200Error before any entry point is called or counted"""
    n0, calls0 = ops.LAUNCHES[0], len(ops.stub.calls)
    with pytest.raises(ops.MacvoB200Error) as e:
        call()
    assert len(ops.stub.calls) == calls0 and ops.LAUNCHES[0] == n0
    return str(e.value)


def test_every_wrapper_has_a_device_case(ops):
    import inspect
    public = {n for n, f in vars(ops).items() if inspect.isfunction(f) and f.__module__ == ops.__name__ and not n.startswith("_")}
    assert public - HOST_ONLY == {n for n in _device_calls(ops) if "." not in n}
    assert NEEDS_CUDA_BUFFERS <= set(_device_calls(ops))


def test_every_wrapper_refuses_operands_on_another_device(ops, monkeypatch):
    """each call is accepted with cuda:0 current (so the refusal below is the device check, not another one) and refused,
    with nothing recorded or counted, when ops reports device 1 as current"""
    for name, call in _device_calls(ops).items():
        n0 = ops.LAUNCHES[0]
        del ops.stub.calls[:]
        call()
        assert ops.stub.calls and ops.LAUNCHES[0] > n0, name
        with monkeypatch.context() as m:
            m.setattr(ops, "_device", lambda: 1)
            msg = _refused(ops, call)
        assert "current device is cuda:1" in msg, (name, msg)


@pytest.mark.parametrize("which", ["pose_io", "stats"])
def test_pgo_solve_counted_checks_pose_and_stats(ops, which):
    buf = ops.ObservationBuffers(8, DEV)
    good = dict(pose_io=f64(7), stats=f64(8))
    ops.pgo_solve_counted(buf, (1.0,) * 5, **good)
    t = good[which]
    for bad in (t.cpu(), t.float(), strided(t), f64(t.numel() + 1)):
        _refused(ops, lambda: ops.pgo_solve_counted(buf, (1.0,) * 5, **dict(good, **{which: bad})))


@pytest.mark.parametrize("which", ["pose_io", "stats", "k_total"])
def test_pgo_solve_sharded_checks_pose_stats_and_count(ops, which):
    exchange = types.SimpleNamespace(ptrs=(C.c_void_p * 1)(), world=1, rank=0)
    shard = [f64(5, 3), f64(5, 2), f64(5), f64(5, 3), f64(5)]
    good = dict(pose_io=f64(7), stats=f64(8), k_total=z(1, dtype=torch.int32))
    ops.pgo_solve_sharded(shard, (1.0,) * 5, None, exchange, **good)
    t = good[which]
    bads = [t.cpu(), t.double() if which == "k_total" else t.float(), z(t.numel() + 1, dtype=t.dtype)]
    if t.numel() > 1:
        bads.append(strided(t))
    for bad in bads:
        _refused(ops, lambda: ops.pgo_solve_sharded(shard, (1.0,) * 5, None, exchange, **dict(good, **{which: bad})))


def test_pgo_accumulate_checks_graph_columns_cluster_and_flag(ops):
    """every graph type launches with its own columns; a missing column, a cluster size outside 0..8 or a bad flag buffer
    is refused before the launch"""
    pos, uv, disp, uvc, dc = f64(5, 3), f64(5, 2), f64(5), f64(5, 3), f64(5)
    icp = dict(pc_obs=f64(5, 3), obs_cov=f64(5, 3, 3), pts_cov=f64(5, 3, 3))
    intr = (1.0,) * 5
    calls = {"disp": lambda **kw: ops.pgo_accumulate(pos, uv, disp, uvc, dc, intr, f64(7), **kw),
             "reproj": lambda **kw: ops.pgo_accumulate(pos, uv, None, uvc, None, intr, f64(7), graph_type="reproj", **kw),
             "icp": lambda **kw: ops.pgo_accumulate(pos, None, None, None, None, intr, f64(7), graph_type="icp",
                                                    **dict(icp, **kw))}
    for gt, call in calls.items():
        del ops.stub.calls[:]
        call(cluster=0, singular_flag=f64(1))
        call(cluster=8)
        assert ops.stub.calls == ["macvo_pgo_accumulate_graph"] * 2, gt
        for bad in (dict(cluster=-1), dict(cluster=9), dict(singular_flag=f64(2)), dict(singular_flag=z(1)),
                    dict(singular_flag=f64(1).cpu())):
            _refused(ops, lambda: call(**bad))
    _refused(ops, lambda: ops.pgo_accumulate(pos, None, disp, uvc, dc, intr, f64(7)))
    _refused(ops, lambda: ops.pgo_accumulate(pos, uv, None, None, None, intr, f64(7), graph_type="reproj"))
    _refused(ops, lambda: ops.pgo_accumulate(pos, None, None, None, None, intr, f64(7), graph_type="icp",
                                             **dict(icp, pts_cov=None)))
    _refused(ops, lambda: calls["icp"](obs_cov=f64(5, 3, 3).cpu()))


@pytest.mark.parametrize("which", ["rows", "mf32", "mf16_rows"])
def test_flow_im2col_checks_its_outputs(ops, which):
    good = dict(rows=z(4, 128, dtype=torch.float16), mf32=z(4, 128),
                mf16_rows=z(ops.rows_count(1, 2, 2), 128, dtype=torch.float16))
    ops.flow_im2col(z(1, 2, 2, 2), z(1, 2, 2, 2), **good)
    t = good[which]
    bads = [t.cpu(), t.double(), strided(t)] + ([z(5, 128)] if which == "mf32" else [])
    for bad in bads:
        _refused(ops, lambda: ops.flow_im2col(z(1, 2, 2, 2), z(1, 2, 2, 2), **dict(good, **{which: bad})))


def test_pack_rows_checks_dst(ops):
    dst = z(ops.rows_count(1, 2, 2), 64, dtype=torch.float16)
    ops.pack_rows(z(4, 64), dst, 0, (1, 2, 2))
    ops.pack_rows(z(1, 2, 2, 64), dst, 0, (1, 2, 2))          # any contiguous (.., C) rows of B*H*W pixels
    for bad in (dst.cpu(), dst.float(), strided(dst)):
        _refused(ops, lambda: ops.pack_rows(z(4, 64), bad, 0, (1, 2, 2)))
