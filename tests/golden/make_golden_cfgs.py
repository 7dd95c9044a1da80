"""Generates tests/golden/reference_cfgs.json: the estimator / tracker configs shipped with the reference (its cfg/ directory),
parsed as the host parser receives them, so that tests/test_host_logic.py checks them without a reference checkout.
usage: python tests/golden/make_golden_cfgs.py <reference checkout>"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_host_logic import SHIPPED  # noqa: E402
from xivo_b200 import sim  # noqa: E402

if __name__ == "__main__":
    cfgs = {name: sim.load_cfg(os.path.join(sys.argv[1], "cfg", name)) for name in sorted(SHIPPED)}
    with open(os.path.join(ROOT, "tests", "golden", "reference_cfgs.json"), "w") as f:  # one config per line
        f.write("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(v, sort_keys=True, separators=(',', ':'))}" for k, v in cfgs.items()) + "\n}\n")
