"""Where the time of the fused RGBA f32 blur goes (DESIGN.md section 4.1), in one run on one GPU:

  * the card: name, power limit, SM clock (sampled while the blur runs) and its maximum;
  * the copy ceiling: a 1 GiB -> 1 GiB f32 `copy_` (reads 1 GiB, writes 1 GiB), CUDA events;
  * the bench.py headline kernel (15 taps, sigma 2.25, mirror, 8192 x 8192 RGBA f32), 200 launches after warm-up, CUDA events;
  * sweeps at the same size: taps 3 / 5 / 7 / 9 / 11 / 15 x border zero / mirror, then conv.band_rows 256 / 1024 / 2048 at
    15 taps, mirror.  If 3 and 15 taps take the same time, the FFMA work is hidden.  conv.band_rows sets only the sharded
    kernel's bands, so here its sweep checks that the single-GPU plan ignores it.

Every timing is repeated (`--reps`) and printed as one JSON line; `--label` tags the lines so that two builds run in one session
can be told apart.  Rates count the algorithmic traffic, 32 B per pixel (read once, write once)."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import zignal_b200 as zb  # noqa: E402

N = 8192
ALGO_BYTES = 32 * N * N


def events_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def smi(query):
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={query}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    return out.stdout.strip()


def gauss_taps(k):
    if k == 15:
        return zb.gaussian_taps(2.25)
    x = np.arange(k, dtype=np.float64) - k // 2
    t = np.exp(-x * x / (2.0 * (k / 6.0) ** 2))
    return (t / t.sum()).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--label", default="")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    L = zb.lib()

    def emit(**kw):
        print(json.dumps({"label": args.label, **kw}), flush=True)

    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.rand(N, N, 4, device="cuda", generator=g)
    src, dst = zb.Image.from_tensor(x), zb.Image.from_tensor(torch.empty_like(x))
    taps15 = gauss_taps(15)

    def blur(taps=taps15, border=zb.BorderMode.MIRROR):
        return lambda: src.convolve_separable(taps, taps, border, out=dst)

    # the card, with the SM clock read while ~1.5 s of blurs are queued
    f = blur()
    events_ms(f, 1, 5)
    for _ in range(2000):
        f()
    clocks = smi("clocks.sm,clocks.max.sm")
    torch.cuda.synchronize()
    emit(what="card", card=smi("name,power.limit"), sm_clock_under_load_and_max=clocks, sms=torch.cuda.get_device_properties(0).multi_processor_count)

    # the ceiling: 1 GiB -> 1 GiB copy
    a = torch.empty(1 << 28, device="cuda", dtype=torch.float32).uniform_()
    b = torch.empty_like(a)
    for _ in range(args.reps):
        ms = events_ms(lambda: b.copy_(a), 50, 5)
        emit(what="copy_1GiB_f32", ms=ms, gbs=2 * a.numel() * 4 / (ms * 1e-3) / 1e9)
    del a, b

    def run(what, fn, **kw):
        for _ in range(args.reps):
            ms = events_ms(fn, args.steps, args.warmup)
            emit(what=what, ms=ms, gbs=ALGO_BYTES / (ms * 1e-3) / 1e9, kernel=L.zb_last_kernel().decode(), **kw)

    run("headline", blur())
    for k in (3, 5, 7, 9, 11, 15):
        for border in (zb.BorderMode.ZERO, zb.BorderMode.MIRROR):
            run("taps", blur(gauss_taps(k), border), taps=k, border=border.name.lower())
    for band in (256, 1024, 2048):
        assert L.zb_tune(b"conv.band_rows", band) == 0
        run("band_rows", blur(), band_rows=band)
    assert L.zb_tune(b"conv.band_rows", 256) == 0


if __name__ == "__main__":
    main()
