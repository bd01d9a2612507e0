"""Writes tests/golden/golden_jpeg_decode.json: the sha256 of the decoder oracle's pixels (tests/jpeg_decode_oracle.py) for every
stored stream under tests/golden/jpeg_decode/ and every output pixel format.  Run from the repository root:
    python tests/golden/make_golden_jpeg_decode.py"""
import hashlib
import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
import jpeg_decode_oracle as jd  # noqa: E402

FORMATS = {"u8": 0, "f32": 1, "rgb8": 2, "rgba8": 3, "rgbaf32": 4}


def main():
    out = {}
    for f in sorted((HERE / "jpeg_decode").glob("*.jpg")):
        data = f.read_bytes()
        for name, fmt in FORMATS.items():
            out[f"{f.name}:{name}"] = hashlib.sha256(jd.decode(data, fmt).tobytes()).hexdigest()
    (HERE / "golden_jpeg_decode.json").write_text(json.dumps(out, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main()
