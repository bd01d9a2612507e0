"""Generates tests/golden/golden_hough.json: SHA-256 of the oracle's HoughTransform accumulators and line lists (cases in
tests/golden_hough.py).  Like golden_8f.json these pin the ORACLE and give the GPU tests fixed answers.
Run:  python tests/golden/make_golden_hough.py"""
import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
from golden_hough import CASES, edges, lines_array, oracle  # noqa: E402
from gpu_utils import sha  # noqa: E402

out = {"_about": "sha256 of oracle outputs of HoughTransform.compute / findLines; see make_golden_hough.py", "cases": {}}
for name, (_, box, size, _, an, rn) in CASES.items():
    img = edges(name)
    acc, lines = oracle(name, img)
    out["cases"][name] = {"box": list(box), "size": size, "input_sha256": sha(img), "edge_pixels": int((img > 0).sum()),
                          "votes": int(acc.sum(dtype="uint64")), "accumulator_sha256": sha(acc), "lines": len(lines),
                          "lines_sha256": sha(lines_array(lines))}
(HERE / "golden_hough.json").write_text(json.dumps(out, indent=1) + "\n")
print("wrote", HERE / "golden_hough.json", len(out["cases"]), "cases")
