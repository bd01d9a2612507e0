"""Generates tests/golden/golden_flood_fill.json: SHA-256 of the oracle's Image.floodFill outputs (cases in tests/golden_flood_fill.py).
Like golden_hough.json these pin the ORACLE and give the GPU tests fixed answers.
Run:  python tests/golden/make_golden_flood_fill.py"""
import json
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
from golden_flood_fill import CASES, image, oracle  # noqa: E402
from gpu_utils import sha  # noqa: E402

out = {"_about": "sha256 of oracle outputs of Image.floodFill; see make_golden_flood_fill.py", "cases": {}}
for name, (_, seed, fill, th, conn, mode) in CASES.items():
    img = image(name)
    got = oracle(name, img)
    out["cases"][name] = {"seed": list(seed), "threshold": th, "connectivity": conn, "mode": mode, "input_sha256": sha(img),
                          "changed_pixels": int((got.view(np.uint8) != img.view(np.uint8)).reshape(img.shape[0], img.shape[1], -1).any(axis=2).sum()),
                          "output_sha256": sha(got)}
(HERE / "golden_flood_fill.json").write_text(json.dumps(out, indent=1) + "\n")
print("wrote", HERE / "golden_flood_fill.json", len(out["cases"]), "cases")
