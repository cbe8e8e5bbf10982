"""Writes tests/golden/hdri_records.npz: the frames of tests/test_hdri_records_gpu.py (accum, depth, raw, display of every fixture case)
rendered by the current build.  It was written with the last build whose HDRI frames went through wide sample records
(direction, L, depth, beta and tr per sample, the environment term added in k_resolve<0>), on an H100:

    VPT_LIB_NAME=<that build's library> python tests/golden/make_hdri_records.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from test_hdri_records_gpu import CASES, OUTPUTS, render_case  # noqa: E402

if __name__ == "__main__":
    volumes, out = {}, {}
    for name in sorted({c[5] for c in CASES.values()}):
        frame = render_case(name, volumes)
        out.update({f"{name}_{k}": v for k, v in frame.items()})
    np.savez_compressed(os.path.join(HERE, "hdri_records.npz"), **out)
    print({k: v.shape for k, v in out.items()})
