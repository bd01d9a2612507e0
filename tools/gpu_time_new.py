"""Device timings (CUDA events, warm, median of 5) of the 8(f) additions at 4096x4096: Canny, median / min / alpha-trimmed, ssim / psnr.
`--binary`: the histogram family and binary morphology instead (sizes as in DESIGN.md section 5), with the card's name and power limit.
`--edges [--profile]`: Shen-Castan and Canny (DESIGN.md section 5), with the card's name and power limit."""
import json
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import zignal_b200 as zb  # noqa: E402


def timed(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def binary_timings():
    import subprocess
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"card": card.splitlines()[0] if card else torch.cuda.get_device_name()}
    n = 8192
    g = torch.Generator(device="cuda").manual_seed(0)
    rgba = zb.Image.from_tensor(torch.randint(0, 256, (n, n, 4), dtype=torch.uint8, device="cuda", generator=g))
    const = zb.Image.from_tensor(torch.full((n, n, 4), 77, dtype=torch.uint8, device="cuda"))
    gray = zb.Image.from_tensor(torch.randint(0, 256, (n, n), dtype=torch.uint8, device="cuda", generator=g))
    outg = zb.Image.init(n, n, zb.PixFmt.U8, device="cuda")
    res["equalize_8192_rgba8_random_ms"] = timed(lambda: rgba.equalize(), reps=11)
    res["equalize_8192_rgba8_constant_ms"] = timed(lambda: const.equalize(), reps=11)
    res["otsu_8192_gray_ms"] = timed(lambda: gray.threshold_otsu(out=outg), reps=11)
    m = 4096
    yy, xx = torch.meshgrid(torch.arange(m, device="cuda"), torch.arange(m, device="cuda"), indexing="ij")
    smooth = zb.Image.from_tensor(((torch.sin(xx / 37.0) * torch.cos(yy / 53.0) * 100 + 128)).clamp(0, 255).to(torch.uint8).contiguous())
    out4 = zb.Image.init(m, m, zb.PixFmt.U8, device="cuda")
    res["adaptive_mean_4096_r8_ms"] = timed(lambda: smooth.threshold_adaptive_mean(8, 4.0, out=out4), reps=11)
    res["adaptive_mean_4096_r256_ms"] = timed(lambda: smooth.threshold_adaptive_mean(256, 4.0, out=out4), reps=11)
    binimg = zb.Image.from_tensor((torch.rand((n, n), device="cuda", generator=g) < 0.5).to(torch.uint8) * 255)
    k3 = np.ones((3, 3), np.uint8)
    res["open_3x3_x2_8192_gray_ms"] = timed(lambda: binimg.open_binary(k3, 2, out=outg), reps=11)
    print(json.dumps(res))


def edges_timings():
    """Image.shenCastan at 4096^2 and 8192^2 gray (smooth + noise, the Canny input of main()) for the default, thin and strong_only presets,
    at 4096^2 RGBA8, and Canny at 4096^2 in the same run.  --profile adds per-kernel device times from torch.profiler."""
    import subprocess
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"card": card.splitlines()[0] if card else torch.cuda.get_device_name()}
    presets = {"default": zb.ShenCastan.default, "thin": zb.ShenCastan.thin, "strong_only": zb.ShenCastan.strong_only}
    rng = np.random.default_rng(0)
    for n in (4096, 8192):
        yy, xx = np.mgrid[0:n, 0:n]
        gray = ((np.sin(xx / 37.0) * np.cos(yy / 53.0) * 100 + 128) + rng.normal(0, 3, (n, n))).clip(0, 255).astype(np.uint8)
        g = zb.Image.from_numpy(gray)
        out = zb.Image.init(n, n, zb.PixFmt.U8, device="cuda")
        for name, o in presets.items():
            res[f"shen_castan_{name}_{n}_gray_ms"] = timed(lambda: o.apply(g, out=out), reps=7)
        if n == 4096:
            res["canny_4096_gray_sigma1.4_ms"] = timed(lambda: g.canny(1.4, 20.0, 60.0, out=out), reps=7)
            rgba = zb.Image.from_numpy(np.repeat(gray[..., None], 4, axis=2))
            res["shen_castan_default_4096_rgba8_ms"] = timed(lambda: zb.ShenCastan.default.apply(rgba, out=out), reps=7)
            if "--profile" in sys.argv:
                from torch.profiler import ProfilerActivity, profile
                for name, o in presets.items():
                    o.apply(g, out=out)
                    torch.cuda.synchronize()
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        o.apply(g, out=out)
                        torch.cuda.synchronize()
                    per = {}
                    for ev in prof.key_averages():
                        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                        if t:
                            key = ev.key.replace("(anonymous namespace)::", "").replace("void ", "").replace("zb::", "")
                            key = key.split("(")[0].strip()
                            per[key] = round(per.get(key, 0.0) + t / 1000.0, 4)
                    res[f"profile_{name}_4096_gray_ms"] = per
    print(json.dumps(res))


def main():
    if "--binary" in sys.argv:
        return binary_timings()
    if "--edges" in sys.argv:
        return edges_timings()
    rng = np.random.default_rng(0)
    n = 4096
    yy, xx = np.mgrid[0:n, 0:n]
    gray = ((np.sin(xx / 37.0) * np.cos(yy / 53.0) * 100 + 128) + rng.normal(0, 3, (n, n))).clip(0, 255).astype(np.uint8)
    rgba = rng.integers(0, 256, (n, n, 4), dtype=np.uint8)
    g, c = zb.Image.from_numpy(gray), zb.Image.from_numpy(rgba)
    c2 = zb.Image.from_numpy(np.roll(rgba, 1, axis=1))
    out8 = zb.Image.init(n, n, zb.PixFmt.U8, device="cuda")
    outg = zb.Image.init(n, n, zb.PixFmt.U8, device="cuda")
    outc = zb.Image.init(n, n, zb.PixFmt.RGBA8, device="cuda")
    res = {"size": [n, n]}
    res["canny_gray_sigma1.4_ms"] = timed(lambda: g.canny(1.4, 20.0, 60.0, out=out8))
    res["canny_rgba_sigma1.0_ms"] = timed(lambda: c.canny(1.0, 20.0, 60.0, out=out8))
    res["median_r1_gray_ms"] = timed(lambda: g.median_blur(1, out=outg))
    res["median_r2_gray_ms"] = timed(lambda: g.median_blur(2, out=outg))
    res["median_r3_gray_ms"] = timed(lambda: g.median_blur(3, out=outg))
    res["median_r5_gray_ms"] = timed(lambda: g.median_blur(5, out=outg))
    res["median_r2_rgba_ms"] = timed(lambda: c.median_blur(2, out=outc))
    res["min_r3_rgba_ms"] = timed(lambda: c.min_blur(3, out=outc))
    res["alpha_trim_r2_gray_ms"] = timed(lambda: g.alpha_trimmed_mean_blur(2, 0.2, out=outg))
    from zignal_b200.compose import motion_blur_linear, motion_blur_radial
    res["motion_linear_diag_d15_rgba_ms"] = timed(lambda: motion_blur_linear(c, outc, 0.6, 15))
    res["motion_linear_horiz_d15_rgba_ms"] = timed(lambda: motion_blur_linear(c, outc, 0.0, 15))
    res["motion_zoom_rgba_ms"] = timed(lambda: motion_blur_radial(c, outc, 0.5, 0.5, 0.5))
    res["motion_spin_rgba_ms"] = timed(lambda: motion_blur_radial(c, outc, 0.5, 0.5, 0.5, spin=True))
    src = zb.Image.from_numpy(rng.integers(0, 256, (1024, 1024, 4), dtype=np.uint8))
    res["insert_blend_overlay_1024_into_4096_ms"] = timed(lambda: c.insert(src, (500.0, 400.0, 2500.0, 2400.0), 0.3, zb.Interpolation.BILINEAR,
                                                                            blend=zb.Blending.OVERLAY))
    outf = zb.Image.init(n, n, zb.PixFmt.RGBAF32, device="cuda")
    res["convert_rgba8_to_rgbaf32_ms"] = timed(lambda: c.convert(zb.PixFmt.RGBAF32, out=outf))
    res["convert_rgba8_to_u8_ms"] = timed(lambda: c.convert(zb.PixFmt.U8, out=outg))
    res["psnr_rgba_ms"] = timed(lambda: c.psnr(c2))
    res["ssim_rgba_ms"] = timed(lambda: c.ssim(c2))
    res["ssim_gray_ms"] = timed(lambda: g.ssim(outg))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
