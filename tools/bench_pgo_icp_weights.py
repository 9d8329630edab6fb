"""Cost of the icp graph's block weights in csrc/pgo.cu: one linearisation (macvo_pgo_accumulate_graph) and one full LM
solve, for well-conditioned icp blocks (cofactor inverse), MAC-VO-shaped blocks (nearly all take the Jacobi
eigen-decomposition) and, for scale, the "disp" graph. Device times from CUDA events, median of 7 runs of 20 launches;
prints one JSON line.

    python tools/bench_pgo_icp_weights.py
"""
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from macvo_b200 import build, ops  # noqa: E402
from tests.golden import cases  # noqa: E402

DEV = "cuda"


def timed_us(fn, reps=20, runs=7):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(runs):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(reps):
            fn()
        e.record()
        torch.cuda.synchronize()
        out.append(s.elapsed_time(e) * 1e3 / reps)
    return statistics.median(out)


def columns(g):
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(DEV)
    return dict(kp2_uv=t(g.kp2_uv), kp2_disp=t(g.kp2_disp), uv_cov=t(g.uv_cov), disp_cov=t(g.disp_cov), pc_obs=t(g.pc_obs),
                obs_cov=t(g.obs_cov), pts_cov=t(g.pts_cov))


def main():
    build.build(verbose=False)
    rows = []
    for K in (512, 2048, 4096):
        inputs = {"disp": cases.pgo_inputs_typed("disp", K, 6), "icp_well_conditioned": cases.pgo_inputs_typed("icp", K, 6),
                  "icp_macvo_fx1000": cases.pgo_inputs_macvo(K, 1, 1000.0)}
        for name, c in inputs.items():
            g = cases.pgo_graph(c)
            col, pos = columns(g), torch.from_numpy(g.pos_Tw).to(DEV)
            intr = (g.fx, g.fy, g.cx, g.cy, g.baseline)
            pose = torch.from_numpy(g.init_pose).to(DEV)
            acc_cols = dict(col)
            head = [acc_cols.pop(n) for n in ("kp2_uv", "kp2_disp", "uv_cov", "disp_cov")]
            acc = lambda: ops.pgo_accumulate(pos, *head, intr, pose, graph_type=g.graph_type, cluster=0, **acc_cols)
            solve = lambda: ops.pgo_solve_graph(g.graph_type, pos, intr, pose, **col)
            _, stats = solve()
            rows.append({"K": K, "inputs": name, "accumulate_us": round(timed_us(acc), 2),
                         "solve_us": round(timed_us(solve), 2), "steps": int(stats[0].item()),
                         "evaluations": int(stats[1].item())})
    print(json.dumps({"gpu": torch.cuda.get_device_name(), "rows": rows}))


if __name__ == "__main__":
    main()
