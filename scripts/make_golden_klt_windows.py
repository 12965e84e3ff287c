"""Write tests/golden/reference_klt_windows.npz: the reference's own FeatureTracker::fbKltTracking (oracle/_ref/libov2ref_frontend.so)
on every case of tests/test_oracle_vs_reference_klt_windows.py, so that the test runs where the reference tree is absent.
Inputs are re-created from seeds by the test, so only the library's outputs are stored.

    python scripts/make_golden_klt_windows.py      (needs the reference library built by build() and cv2)
"""
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
os.environ["OV2_RECORD_REFERENCE"] = "1"

from oracle.ref_build import cv_callbacks as CB  # noqa: E402
from reference_golden import ReferenceOutputs  # noqa: E402
import test_oracle_vs_reference_klt_windows as T  # noqa: E402

lib = CB.load()
if lib is None:
    raise SystemExit("make_golden_klt_windows.py: the reference library is not built (oracle/_ref)")
rec = ReferenceOutputs("klt_windows", lib)
for case in T.CASES:
    r = T.reference_call(rec, *case)
    print(T.case_key(*case), "tracked", int(r["st"].sum()), "of", len(r["st"]))
rec.save()
print("wrote", rec.path)
