"""Generates tests/golden/golden_binary.json: SHA-256 of the oracle's outputs for the 8-bit histogram family and binary morphology (cases in
tests/golden_binary.py).  Like golden_8f.json these pin the ORACLE and give the GPU tests fixed answers.
Run:  python tests/golden/make_golden_binary.py"""
import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
from golden_binary import CASES  # noqa: E402
from gpu_utils import sha  # noqa: E402

out = {"_about": "sha256 of oracle outputs for the histogram family and binary morphology; see make_golden_binary.py", "cases": {}}
for name, (build, oracle, _device) in CASES.items():
    img = build()
    res = oracle(img)
    out["cases"][name] = {"input_sha256": sha(img), "shape": list(res.shape), "dtype": str(res.dtype), "output_sha256": sha(res)}
(HERE / "golden_binary.json").write_text(json.dumps(out, indent=1) + "\n")
print("wrote", HERE / "golden_binary.json", len(out["cases"]), "cases")
