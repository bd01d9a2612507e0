"""Generates tests/golden/golden_quantize.json: SHA-256 of the oracle's palettes, LUTs, index maps and dithered images (cases in
tests/golden_quantize.py).  Like golden_flood_fill.json these pin the ORACLE and give the GPU tests fixed answers.
Run:  python tests/golden/make_golden_quantize.py"""
import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
from golden_quantize import CASES, run_chain  # noqa: E402
from gpu_utils import sha  # noqa: E402

out = {"_about": "sha256 of oracle outputs of medianCut / buildPalette, ColorLookupTable, lookup and dither.apply; see make_golden_quantize.py",
       "cases": {}}
for name, (builder, kind, mode) in CASES.items():
    img = builder()
    pal, lut, idx, dithered = run_chain(name, img)
    out["cases"][name] = {"palette": kind, "mode": mode, "input_sha256": sha(img), "colors": int(pal.shape[0]), "palette_sha256": sha(pal),
                          "lut_sha256": sha(lut), "indices_sha256": sha(idx), "dithered_sha256": sha(dithered)}
(HERE / "golden_quantize.json").write_text(json.dumps(out, indent=1) + "\n")
print("wrote", HERE / "golden_quantize.json", len(out["cases"]), "cases")
