"""Generates tests/golden/golden_visual.json: SHA-256 of the oracle's diff / applyColormap / flip / invert outputs and the diff statistics
(cases in tests/golden_visual.py).  Like golden_quantize.json these pin the ORACLE and give the GPU tests fixed answers.

The viridis and inferno tables are data in the reference (image/colormaps.zig), not something the oracle computes.  With
`--tables <zignal>/src/image/colormaps.zig` the generator first extracts them into tests/golden/colormap_tables.json, the data fixture
the tests read them from.
Run:  python tests/golden/make_golden_visual.py [--tables path/to/colormaps.zig]"""
import json
import re
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))


def extract_tables(colormaps_zig: Path) -> dict:
    text = colormaps_zig.read_text()
    out = {}
    for name in ("viridis", "inferno"):
        body = re.search(r"const " + name + r"_lut = \[_\]\[3\]u8\{(.*?)\n\};", text, flags=re.S).group(1)
        rows = [[int(v) for v in m.groups()] for m in re.finditer(r"\.\{\s*(\d+),\s*(\d+),\s*(\d+)\s*\}", body)]
        assert len(rows) == 256, (name, len(rows))
        out[name] = rows
    return out


if "--tables" in sys.argv:
    src = Path(sys.argv[sys.argv.index("--tables") + 1])
    tables = {"_about": "viridis and inferno, 256 x [r, g, b], from zignal's image/colormaps.zig; see make_golden_visual.py"}
    tables.update(extract_tables(src))
    (HERE / "colormap_tables.json").write_text(json.dumps(tables, separators=(",", ":")) + "\n")
    print("wrote", HERE / "colormap_tables.json")

from golden_visual import CASES, case_inputs, run_case  # noqa: E402
from gpu_utils import sha  # noqa: E402

out = {"_about": "sha256 of oracle outputs of Image.diff / applyColormap / flipLeftRight / flipTopBottom / invert; see make_golden_visual.py",
       "cases": {}}
for name in CASES:
    res = run_case(name)
    entry = {"input_sha256": [sha(a) for a in case_inputs(name)], "output_sha256": sha(res["out"])}
    if "stats" in res:
        entry["stats"] = {k: (v.hex() if isinstance(v, float) else v) for k, v in res["stats"].items()}
    out["cases"][name] = entry
(HERE / "golden_visual.json").write_text(json.dumps(out, indent=1) + "\n")
print("wrote", HERE / "golden_visual.json", len(out["cases"]), "cases")
