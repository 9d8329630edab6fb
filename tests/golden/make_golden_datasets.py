"""Generate tests/golden/net_{euroc,kitti,kitti00}.pt: the decoder_depth 12 parity fixtures at the shipped dataset frame
sizes (cases.LADDER_CASES), with the contents and method of net_cfgA.pt (make_golden_cfgA.py): the reference's own fp32
output, the float64 `FlowFormerCovNet` per-stage samples and the fp32 noise floor.

These are the sizes where the network's shape-dependent choices differ from 640x480: the correlation kernel (N % 8), the
fp16 GMA softmax kernel (N % 4), the padded vertical global attention (H1, W1 not multiples of 4), the remainder the
Twins sr = 8 key / value stride drops at 1/4 resolution, and odd H1 = 47.

Needs a MAC-VO checkout (one to three minutes per size; the float64 correlation volume alone is 0.9 GB at N = 7332):
    MACVO_REFERENCE_ROOT=<MAC-VO checkout> python tests/golden/make_golden_datasets.py [euroc|kitti|kitti00 ...]
"""
from __future__ import annotations

import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden_cfgA import generate  # noqa: E402

DATASET_CASES = ("euroc", "kitti", "kitti00")


if __name__ == "__main__":
    for case in sys.argv[1:] or DATASET_CASES:
        if case not in DATASET_CASES:
            raise SystemExit(f"unknown case {case!r}: one of {DATASET_CASES}")
        generate(case)
