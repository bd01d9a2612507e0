"""Generates tests/golden/golden_jpeg.json: SHA-256 and length of the oracle's JPEG files for the cases of tests/golden_jpeg.py.  Like the
other golden files these pin the ORACLE and give the GPU tests fixed answers.
Run:  python tests/golden/make_golden_jpeg.py"""
import hashlib
import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))

import jpeg_oracle as jo  # noqa: E402
from golden_jpeg import CASES, case_input, case_options  # noqa: E402
from gpu_utils import sha  # noqa: E402

out = {"_about": "sha256 and length of oracle jpeg.encode outputs; see make_golden_jpeg.py", "cases": {}}
for name in CASES:
    img = case_input(name)
    data = jo.encode(img, **case_options(name))
    out["cases"][name] = {"input_sha256": sha(img), "sha256": hashlib.sha256(data).hexdigest(), "len": len(data)}
(HERE / "golden_jpeg.json").write_text(json.dumps(out, indent=1) + "\n")
print("wrote", HERE / "golden_jpeg.json", len(out["cases"]), "cases")
