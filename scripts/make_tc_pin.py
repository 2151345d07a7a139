"""Writes the fixture of tests/test_gpu_tc_pin.py (needs an H100):

    python scripts/make_tc_pin.py [OUT.npz]        (default: tests/golden/tc_pin.npz)

Run it at the commit whose results the pin is to hold; it prints each case's keys."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from mvsmplfitting_b200 import synthetic as S  # noqa: E402
from tests import test_gpu_tc_pin as P  # noqa: E402

out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "tc_pin.npz")
model = S.make_model(0)
arrs = {}
for name in P.CASES:
    r = P.run_case(name, model)
    print(name, sorted(r))
    arrs.update({name + "/" + k: v for k, v in r.items()})
os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
np.savez_compressed(out, **arrs)
print("wrote", out)
