"""Generates tests/golden/golden_shen_castan.json: SHA-256 of the oracle's Shen-Castan outputs (cases in tests/golden_shen_castan.py).  Like
golden_8f.json these pin the ORACLE and give the GPU tests fixed answers.
Run:  python tests/golden/make_golden_shen_castan.py"""
import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
from golden_shen_castan import CASES, oracle  # noqa: E402
from gpu_utils import sha  # noqa: E402

out = {"_about": "sha256 of oracle outputs of Image.shenCastan; see make_golden_shen_castan.py", "cases": {}}
for name, (build, preset) in CASES.items():
    img = build()
    res = oracle(name, img)
    out["cases"][name] = {"preset": preset, "input_sha256": sha(img), "shape": list(res.shape), "edges": int((res > 0).sum()),
                          "output_sha256": sha(res)}
(HERE / "golden_shen_castan.json").write_text(json.dumps(out, indent=1) + "\n")
print("wrote", HERE / "golden_shen_castan.json", len(out["cases"]), "cases")
