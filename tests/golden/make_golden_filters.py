"""Generate tests/golden/filters_*.pt by running the MAC-VO tree's own observation filters (CPU):

    MACVO_REFERENCE_ROOT=<MAC-VO checkout> python tests/golden/make_golden_filters.py

For each bundle of tests/golden/filter_cases.py: CovarianceSanityFilter, SimpleDepthFilter (after `set_meta` on a StereoData
of the "auto" camera), LikelyFrontOfCamFilter and their FilterCompose (Module/OutlierFilter.py) on the MatchObs columns.
Stored: the four masks and the inputs' sha256."""
import os
import sys
from types import SimpleNamespace as NS

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
os.environ.setdefault("TORCHDYNAMO_DISABLE", "1")

import torch  # noqa: E402

from tests.golden import filter_cases as fc, refharness  # noqa: E402


class Bundle:
    def __init__(self, data):
        self.data = data

    def __len__(self):
        return next(iter(self.data.values())).shape[0]


def main() -> None:
    refharness.install()
    from DataLoader import StereoData
    from Module.OutlierFilter import (CovarianceSanityFilter, FilterCompose, LikelyFrontOfCamFilter,
                                      SimpleDepthFilter)
    meta = StereoData(T_BS=None, K=torch.tensor([[[fc.AUTO_FX, 0., 96.], [0., fc.AUTO_FX, 64.], [0., 0., 1.]]]),
                      baseline=torch.tensor([fc.AUTO_BASELINE]), time_ns=[0], height=128, width=192,
                      imageL=torch.zeros(1, 3, 128, 192), imageR=torch.zeros(1, 3, 128, 192))
    cpu = torch.device("cpu")
    for name in fc.BUNDLES:
        b = fc.filter_bundle(name)
        values = Bundle(b["data"])
        depth_args = lambda: NS(min_depth=b["min_depth"], max_depth=b["max_depth"])
        sd = SimpleDepthFilter(depth_args())
        sd.set_meta(meta)
        comp = FilterCompose(NS(filter_args=[NS(type="CovarianceSanityFilter", args=None),
                                             NS(type="SimpleDepthFilter", args=depth_args()),
                                             NS(type="LikelyFrontOfCamFilter", args=None)]))
        comp.set_meta(meta)
        out = {"bundle": name, "input_sha": fc.bundle_sha(b),
               "sanity": CovarianceSanityFilter(NS()).filter(values, cpu),
               "simple_depth": sd.filter(values, cpu),
               "front_of_cam": LikelyFrontOfCamFilter(NS()).filter(values, cpu),
               "compose": comp.filter(values, cpu), "max_depth": sd.config.max_depth}
        path = os.path.join(REPO, "tests", "golden", f"filters_{name}.pt")
        torch.save(out, path)
        print(f"wrote {path}: {len(values)} rows, kept {int(out['compose'].sum())} (max_depth {out['max_depth']})")


if __name__ == "__main__":
    main()
