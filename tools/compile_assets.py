"""Compile the reference's MJCF models into committed fixtures (myosuite_b200/assets/*.npz).

The tests and the GPU runs need no MyoSuite checkout: the hot-path models are compiled by this repo's own
MJCF compiler from the reference's XML/STL inputs and committed as data fixtures.  Run:
    python tools/compile_assets.py <MyoSuite checkout root>/myosuite
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from myosuite_b200 import mjcf  # noqa: E402
from myosuite_b200.assets import MODEL_XML  # noqa: E402

root = sys.argv[1]
out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "myosuite_b200", "assets")
for name, (rel, kwargs) in MODEL_XML.items():
    m = mjcf.compile_mjcf(os.path.join(root, rel), **kwargs)
    m.source_path = rel
    mjcf.save_model(m, os.path.join(out, name + ".npz"))
    print(name, "nq", m.nq, "nv", m.nv, "nu", m.nu, "npair", m.npair, "unsupported pairs", len(m.pair_unsupported))
