"""Writes the fixture of tests/test_gpu_resident_pin.py (needs an H100):

    python scripts/make_resident_pin.py [OUT.npz]        (default: tests/golden/resident_pin.npz)

Run it at the commit whose results the pin is to hold; it prints each case's counts."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from mvsmplfitting_b200 import synthetic as S  # noqa: E402
from tests import test_gpu_resident_pin as P  # noqa: E402

out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "resident_pin.npz")
model, gmm = S.make_model(0), S.make_gmm(7)
arrs = {}
for name in P.CASES:
    r = P.run_case(name, model, gmm)
    print(name, dict(zip(P.STATS, r["stats"].tolist())))
    arrs.update({name + "/" + k: v for k, v in r.items()})
os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
np.savez_compressed(out, **arrs)
print("wrote", out)
