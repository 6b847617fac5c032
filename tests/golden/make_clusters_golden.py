"""Generates tests/golden/clusters_kat.npz from the REFERENCE'S OWN fillClusters code (oracle/_ref/libclusters_shim_b200.so, built by
oracle/build_ref.py; entry ref_clusters_fill).  Run in the build container only:  python tests/golden/make_clusters_golden.py

The inputs are the named cases of tests/test_clusters_cpu.py (CASES, case()), rebuilt there from the same seeds; per case the fixture
holds the bytes of lights[], clusters[], map[], the AtlasSorter list and the uncast-in-atlas list."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_clusters_cpu import CASES, OUTPUTS, as_bytes, case, run  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def clusters_kat():
    d = {}
    for name in CASES:
        out = as_bytes(run(case(name), which="shim"))
        for k in OUTPUTS:
            d[f"{name}_{k}"] = out[k]
    np.savez_compressed(os.path.join(OUT, "clusters_kat.npz"), **d)
    print("clusters_kat", len(CASES), "cases")


if __name__ == "__main__":
    clusters_kat()
