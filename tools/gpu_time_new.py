"""Device timings (CUDA events, warm, median of 5) of the 8(f) additions at 4096x4096: Canny, median / min / alpha-trimmed, ssim / psnr.
`--binary`: the histogram family and binary morphology instead (sizes as in DESIGN.md section 5), with the card's name and power limit.
`--edges [--profile]`: Shen-Castan and Canny (DESIGN.md section 5), with the card's name and power limit.
`--hough`: HoughTransform compute / findLines (DESIGN.md section 5) next to the CPU oracle, with the card's name and power limit.
`--flood-fill`: Image.floodFill (DESIGN.md section 5) next to the CPU oracle, with the card's name and power limit.
`--quantize`: median cut, LUT, palette lookup and dithering (DESIGN.md section 5) next to the CPU oracle, with the card's name and power
limit.
`--visual`: Image.diff, applyColormap, the flips and invert at 8192^2 (DESIGN.md section 4.6) against a device copy of the same bytes,
with the card's name and power limit.
`--jpeg`: jpeg.encode on the device (DESIGN.md section 5) next to the single-threaded CPU oracle: the kernels' device time (summed from
torch.profiler's CUDA activity), the end-to-end time of one call including the copy of the bytes to the host, and the output size, with
the card's name and power limit.
`--jpeg-decode`: jpeg.loadFromBytes on the device (DESIGN.md section 5): per-kernel device time (torch.profiler, a run of its own),
end-to-end call time (host parse and host-to-device copy included), compressed MB/s and MP/s, next to the single-threaded CPU oracle,
Pillow (libjpeg-turbo, one thread) and torchvision's nvJPEG decode when it imports (timing only: not the same pixels), with the
card's name and power limit.
`--jpeg-decode-batch`: Image.decode_jpeg_batch (DESIGN.md section 5) on 1 / 16 / 256 / 1024 copies of liza.jpg, 256 mixed small
encoder streams from a seed and one 1080p file alone: images/s and MB/s end to end and in device time (torch.profiler), next to a
loop of Image.decode_jpeg, the CPU oracle and Pillow on one thread, and torchvision's list decode on cuda (timing only), with the
card's name and power limit."""
import json
import re
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


def hough_timings():
    """HoughTransform (DESIGN.md sections 4-5): (a) the reference example's call shape, per frame (accumulator fill + compute + findLines)
    on a host clock ending in the synchronise findLines performs; (b) size 4096 over a 4096^2 Canny map of main()'s gray image; (c) an all-255 box of
    size 2048, the densest case.  CUDA-event medians of compute, the single-thread CPU oracle on the same inputs (timed on a crop and scaled
    by the vote count where the whole run takes too long, flagged "scaled"), and a sweep of the vote kernel's CTA shape."""
    import subprocess
    import time
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
    import hough_oracle as zo
    from golden_hough import example_frame
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"card": card.splitlines()[0] if card else torch.cuda.get_device_name()}
    L = zb.lib()

    def oracle_ms(size, img, box, threshold=None):
        t0 = time.perf_counter()
        acc = zo.compute(size, img, box, np.zeros((size, size), np.uint32))
        t1 = time.perf_counter()
        if threshold is not None:
            zo.find_lines(size, acc, threshold, 5.0, 5.0)
        return (t1 - t0) * 1e3, (time.perf_counter() - t1) * 1e3, acc

    # (a) 400^2 frame, box (50, 50)-(350, 350), size 300
    frame = example_frame()
    h300 = zb.HoughTransform(300)
    dev = zb.Image.from_numpy(frame)
    acc = torch.zeros((300, 300), dtype=torch.int32, device="cuda")
    box = zb.Rectangle(50, 50, 350, 350)
    th = None

    def one_frame():
        nonlocal th
        acc.zero_()
        h300.compute(dev, box, acc)
        if th is None:
            th = max(1, int(acc.max()) // 2)
        return h300.find_lines(acc, th, 5.0, 5.0)

    for _ in range(10):
        one_frame()
    ts = []
    for _ in range(101):
        t0 = time.perf_counter()
        one_frame()
        ts.append((time.perf_counter() - t0) * 1e3)
    res["a_example_300_frame_ms"] = float(np.median(ts))
    res["a_example_300_compute_ms"] = timed(lambda: h300.compute(dev, box, acc), reps=51)
    oc, of, _ = oracle_ms(300, frame, (50, 50, 350, 350), th)
    res["a_example_300_oracle_compute_ms"], res["a_example_300_oracle_find_lines_ms"] = oc, of
    res["a_edge_pixels"] = int((frame[50:350, 50:350] > 0).sum())

    # (b) size 4096 over the 4096^2 gray image of main(); Canny at main()'s thresholds (20, 60) finds no edge in it, so (5, 15): 1.67 M
    #     edge pixels
    rng = np.random.default_rng(0)
    n = 4096
    yy, xx = np.mgrid[0:n, 0:n]
    gray = ((np.sin(xx / 37.0) * np.cos(yy / 53.0) * 100 + 128) + rng.normal(0, 3, (n, n))).clip(0, 255).astype(np.uint8)
    cmap = zb.Image.from_numpy(gray).canny(1.4, 5.0, 15.0)
    cmap_np = cmap.to_numpy()
    h4096 = zb.HoughTransform(n)
    acc4 = torch.zeros((n, n), dtype=torch.int32, device="cuda")
    box4 = zb.Rectangle(0, 0, n, n)
    h4096.compute(cmap, box4, acc4)
    votes = int(acc4.to(torch.int64).sum())
    edges_b = int((cmap_np > 0).sum())
    res["b_edge_pixels"], res["b_votes"] = edges_b, votes
    res["b_compute_4096_ms"] = timed(lambda: h4096.compute(cmap, box4, acc4), reps=11)
    res["b_votes_per_s"] = votes / (res["b_compute_4096_ms"] * 1e-3)
    res["b_angle_evals_per_s"] = edges_b * n / (res["b_compute_4096_ms"] * 1e-3)
    th4 = int(acc4.max()) // 2   # the example's threshold; a low one makes the greedy NMS (host, O(candidates x kept)) dominate
    res["b_find_lines_4096_ms"] = timed(lambda: h4096.find_lines(acc4, th4, 2.0, 8.0), reps=3)
    crop = cmap_np[:256]   # the first 256 rows, scaled by the edge count
    oc, _, _ = oracle_ms(n, crop, (0, 0, n, n))
    res["b_oracle_compute_4096_ms_scaled"] = oc * edges_b / max(1, int((crop > 0).sum()))

    # (c) all-255 box, size 2048: 2048^3 angle evaluations
    m = 2048
    full = zb.Image.from_tensor(torch.full((m, m), 255, dtype=torch.uint8, device="cuda"))
    h2048 = zb.HoughTransform(m)
    acc2 = torch.zeros((m, m), dtype=torch.int32, device="cuda")
    box2 = zb.Rectangle(0, 0, m, m)
    res["c_compute_2048_all255_ms"] = timed(lambda: h2048.compute(full, box2, acc2), reps=11)
    res["c_angle_evals_per_s"] = m ** 3 / (res["c_compute_2048_all255_ms"] * 1e-3)
    oc, _, _ = oracle_ms(m, np.full((16, m), 255, np.uint8), (0, 0, m, m))
    res["c_oracle_compute_2048_all255_ms_scaled"] = oc * m / 16

    # the vote kernel's CTA shape: threads per CTA x cap on the angle columns per CTA
    sweep = {}
    for threads in (512, 1024):
        for cols in (4, 8, 16, 32):
            L.zb_tune(b"hough.threads", threads)
            L.zb_tune(b"hough.max_cols", cols)
            sweep[f"t{threads}_c{cols}"] = {"b_4096_ms": timed(lambda: h4096.compute(cmap, box4, acc4), reps=5),
                                            "c_2048_ms": timed(lambda: h2048.compute(full, box2, acc2), reps=5),
                                            "a_300_ms": timed(lambda: h300.compute(dev, box, acc), reps=21)}
    L.zb_tune(b"hough.threads", 1024)
    L.zb_tune(b"hough.max_cols", 8)
    res["sweep"] = sweep
    print(json.dumps(res))


def flood_fill_timings():
    """Image.floodFill (DESIGN.md sections 4.6 and 5): CUDA-event medians over 21 warm calls of (a) an 8192^2 u8 uniform image (one
    component), (b) a 4096^2 Rgb image in .neighbor mode at a threshold near percolation, (c) a 4096^2 u8 spiral maze, (d) a 4096^2 Canny
    edge map (as in --hough) filled from a background pixel; the single-thread CPU oracle on the same input beside each, the bytes the
    kernels move at the least (image read once, labels written and read once, filled pixels written) and a per-kernel split from
    torch.profiler in a separate pass."""
    import subprocess
    import time
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
    import flood_fill_oracle as zo
    from golden_flood_fill import spiral
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"card": card.splitlines()[0] if card else torch.cuda.get_device_name()}

    rng = np.random.default_rng(0)
    n = 4096
    yy, xx = np.mgrid[0:n, 0:n]
    gray = ((np.sin(xx / 37.0) * np.cos(yy / 53.0) * 100 + 128) + rng.normal(0, 3, (n, n))).clip(0, 255).astype(np.uint8)
    canny = zb.Image.from_numpy(gray).canny(1.4, 5.0, 15.0).to_numpy()
    bg = np.argwhere(canny == 0)[0]
    # a random walk of Rgb colours along each row: horizontal neighbours differ by small steps, vertical ones by the rows' drift
    steps = rng.integers(-6, 7, (n, n, 3))
    rgb = np.clip(128 + np.cumsum(steps, axis=1) // 8, 0, 255).astype(np.uint8)
    workloads = {
        "a_uniform_8192_u8": (lambda: np.full((8192, 8192), 17, np.uint8), (4096, 4096), 200, 0.0, 4, zo.SEED),
        "b_rgb_4096_neighbor": (lambda: rgb, (n // 2, n // 2), (255, 0, 0), 2.0, 4, zo.NEIGHBOR),
        "c_spiral_4096_u8": (lambda: spiral(n), (0, 0), 100, 0.0, 4, zo.SEED),
        "d_canny_4096_background": (lambda: canny, (int(bg[0]), int(bg[1])), 128, 0.0, 4, zo.SEED),
    }
    for name, (make, (r, c), fill, th, conn, mode) in workloads.items():
        img = make()
        src = zb.Image.from_numpy(img)
        dev = zb.Image.init_like(src)
        px = img.dtype.itemsize * (img.shape[2] if img.ndim == 3 else 1)

        def call():
            src.copy(dev)
            dev.flood_fill(r, c, fill, th, zb.Connectivity(conn), zb.FloodFillMode(mode))
        copy_ms = timed(lambda: src.copy(dev), reps=21)
        ms = timed(call, reps=21) - copy_ms
        want = zo.flood_fill(img.copy(), r, c, fill, th, conn, mode)
        t0 = time.perf_counter()
        zo.flood_fill(img.copy(), r, c, fill, th, conn, mode)
        oracle_ms = (time.perf_counter() - t0) * 1e3
        call()
        got = dev.to_numpy()
        filled = int((got.view(np.uint8) != img.view(np.uint8)).reshape(img.shape[0], img.shape[1], -1).any(axis=2).sum())
        pixels = img.shape[0] * img.shape[1]
        least_bytes = pixels * (px + 4 + 4) + filled * px
        res[name] = {"device_ms": round(ms, 4), "oracle_ms": round(oracle_ms, 1), "bit_exact": bool(np.array_equal(got.view(np.uint8),
                     want.view(np.uint8))), "filled_pixels": filled, "least_bytes": least_bytes,
                     "least_bytes_GBps": round(least_bytes / (ms * 1e-3) / 1e9, 1)}
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                call()
            torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            if t and "flood" in ev.key:
                key = ev.key.split("flood_")[1].split("<")[0]
                per[key] = round(per.get(key, 0.0) + t / 5000.0, 4)
        res[name]["kernel_ms"] = per
    print(json.dumps(res))


def quantize_timings():
    """Colour quantization and dithering (DESIGN.md sections 4.6 and 5), CUDA-event medians of warm calls: the median cut at 8192^2 Rgb
    split into the device histogram (torch.profiler) and the host cut, the LUT, ordered dither and the index lookup at 8192^2 as a
    fraction of the bandwidth of a device copy of the same bytes, Floyd-Steinberg and Atkinson at 1080p and 8192^2 with ns per wavefront
    step (time / (cols + 2 rows)) and a sweep of the publishing granularity; the single-thread CPU oracle beside each number."""
    import subprocess
    import time
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
    import quantize_oracle as zo
    from golden_quantize import smooth_rgb
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"card": card.splitlines()[0] if card else torch.cuda.get_device_name()}
    L = zb.lib()

    def host_ms(fn):
        t0 = time.perf_counter()
        fn()
        return round((time.perf_counter() - t0) * 1e3, 1)

    n = 8192
    img = smooth_rgb(n, n, 1)
    src = zb.Image.from_numpy(img)
    dev = zb.Image.init_like(src)
    zb.median_cut(src, 256)
    t0 = time.perf_counter()
    for _ in range(5):
        pal = zb.median_cut(src, 256)
    total = (time.perf_counter() - t0) * 1e3 / 5
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            zb.median_cut(src, 256)
        torch.cuda.synchronize()
    hist = sum((getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)) for ev in prof.key_averages()
               if "mc_histogram" in ev.key) / 5000.0
    res["median_cut_8192_rgb"] = {"total_ms": round(total, 3), "device_histogram_ms": round(hist, 3), "host_cut_ms": round(total - hist, 3),
                                  "oracle_ms": host_ms(lambda: zo.median_cut(img, 256)), "colors": int(len(pal))}
    lut = zb.ColorLookupTable(pal)
    pal_c = np.ascontiguousarray(pal)
    s = torch.cuda.current_stream().cuda_stream
    res["lut_256"] = {"device_ms": round(timed(lambda: L.zb_color_lut(pal_c.ctypes.data, len(pal_c), lut.table.data_ptr(), s), reps=21), 4),
                      "oracle_ms": host_ms(lambda: zo.color_lut(pal))}
    copy_ms = timed(lambda: src.copy(dev), reps=21)                 # reads and writes 3 B / pixel, as ordered dither does
    res["copy_8192_rgb_ms"] = round(copy_ms, 4)
    copy_gbps = 2 * 3 * n * n / (copy_ms * 1e-3) / 1e9
    ms = timed(lambda: (src.copy(dev), dev.dither(lut, zb.DitherMode.ORDERED)), reps=21) - copy_ms
    res["ordered_8192"] = {"device_ms": round(ms, 4), "fraction_of_copy": round(copy_ms / ms, 3),
                           "oracle_ms": host_ms(lambda: zo.dither(img.copy(), pal, zo.color_lut(pal), zo.ORDERED))}
    out = zb.Image.init(n, n, zb.PixFmt.U8)
    ms = timed(lambda: src.palette_indices(lut, out), reps=21)
    res["lookup_8192"] = {"device_ms": round(ms, 4), "fraction_of_copy": round(4 * n * n / (ms * 1e-3) / 1e9 / copy_gbps, 3),
                          "oracle_ms": host_ms(lambda: zo.palette_lookup(img, zo.color_lut(pal)))}
    for rows, cols in ((1080, 1920), (8192, 8192)):
        im = smooth_rgb(rows, cols, 2)
        a = zb.Image.from_numpy(im)
        b = zb.Image.init_like(a)
        base = timed(lambda: a.copy(b), reps=11)
        for mode in (zb.DitherMode.FLOYD_STEINBERG, zb.DitherMode.ATKINSON):
            entry = {"oracle_ms": host_ms(lambda: zo.dither(im.copy(), pal, zo.color_lut(pal), int(mode)))}
            for publish in (8, 16, 32, 64, 128):
                L.zb_tune(b"dither.publish", publish)
                ms = timed(lambda: (a.copy(b), b.dither(lut, mode)), reps=11) - base
                entry[f"publish_{publish}"] = {"device_ms": round(ms, 3), "ns_per_step": round(ms * 1e6 / (cols + 2 * rows), 1)}
            L.zb_tune(b"dither.publish", 32)
            res[f"{mode.name.lower()}_{rows}x{cols}"] = entry
    print(json.dumps(res))


def visual_timings():
    """diff (Rgba(u8) and Rgba(f32), with and without stats), applyColormap (U8 and F32, automatic range), both flips and invert at
    8192^2: CUDA-event medians of warm calls, the algorithmic bytes (every input read once, every output written once; the range pass's
    second read of the source is not counted) over that time, and that rate as a fraction of the faster of two contiguous device copies
    of the same 8192^2 Rgba(u8) bytes timed in the same run: cudaMemcpyAsync (torch copy_) and a streaming elementwise kernel (torch
    bitwise_not).  Every call goes straight to its C entry point, so each event window holds the same kind of host call."""
    import ctypes as C
    import subprocess
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"card": card.splitlines()[0] if card else torch.cuda.get_device_name(), "size": [8192, 8192]}
    L = zb.lib()
    n = 8192
    rng = np.random.default_rng(0)
    s = torch.cuda.current_stream().cuda_stream
    a8 = zb.Image.from_numpy(rng.integers(0, 256, (n, n, 4), dtype=np.uint8))
    b8 = zb.Image.from_numpy(rng.integers(0, 256, (n, n, 4), dtype=np.uint8))
    o8 = zb.Image.init_like(a8)
    src_t, dst_t = a8.tensor().reshape(-1), o8.tensor().reshape(-1)
    copies = {"memcpy": timed(lambda: dst_t.copy_(src_t), reps=21),
              "stream_kernel": timed(lambda: torch.bitwise_not(src_t, out=dst_t), reps=21)}
    for name, ms in copies.items():
        res[f"copy_rgba8_{name}"] = {"device_ms": round(ms, 4), "gb_per_s": round(2 * 4 * n * n / (ms * 1e-3) / 1e9, 1)}
    copy_gbps = 2 * 4 * n * n / (min(copies.values()) * 1e-3) / 1e9

    def entry(ms, nbytes):
        gbps = nbytes / (ms * 1e-3) / 1e9
        return {"device_ms": round(ms, 4), "gb_per_s": round(gbps, 1), "fraction_of_copy": round(gbps / copy_gbps, 3)}

    af = zb.Image.from_numpy(rng.random((n, n, 4), dtype=np.float32))
    bf = zb.Image.from_numpy(rng.random((n, n, 4), dtype=np.float32))
    of = zb.Image.init_like(af)
    st = zb._ffi.ZbDiffStats()
    for name, (x, y, o, pb) in {"rgba8": (a8, b8, o8, 4), "rgbaf32": (af, bf, of, 16)}.items():
        xa, ya, oa = x._zb(), y._zb(), o._zb()
        for with_stats in (False, True):
            ptr = C.byref(st) if with_stats else None
            ms = timed(lambda: L.zb_diff(xa, ya, oa, int(x.pixfmt), C.c_float(1.0), C.c_float(2.0), 0, 1, ptr, s), reps=21)
            res[f"diff_{name}_{'stats' if with_stats else 'no_stats'}"] = entry(ms, 3 * pb * n * n)
    lut = zb.colormap_lut(zb.Colormap.TURBO)
    rgb = zb.Image.init(n, n, zb.PixFmt.RGB8)
    for name, img, pb in (("u8", zb.Image.from_numpy(rng.integers(0, 256, (n, n), dtype=np.uint8)), 1),
                          ("f32", zb.Image.from_numpy(rng.random((n, n), dtype=np.float32)), 4)):
        xa, da = img._zb(), rgb._zb()
        ms = timed(lambda: L.zb_apply_colormap(xa, int(img.pixfmt), lut.ctypes.data_as(C.c_void_p), 0, C.c_double(0), 0, C.c_double(0), da, s),
                   reps=21)
        res[f"colormap_{name}_auto"] = entry(ms, (pb + 3) * n * n)
    oa = o8._zb()
    for name, fn in (("flip_left_right", L.zb_flip_left_right), ("flip_top_bottom", L.zb_flip_top_bottom), ("invert", L.zb_invert)):
        res[f"{name}_rgba8"] = entry(timed(lambda: fn(oa, int(o8.pixfmt), s), reps=21), 2 * 4 * n * n)
    print(json.dumps(res))


def jpeg_timings():
    import subprocess
    import time

    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
    import jpeg_oracle as jo
    from golden_jpeg import noise, smooth
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"card": card.splitlines()[0] if card else torch.cuda.get_device_name()}
    work = [("rgb8_8192_q90_420_smooth", smooth("rgb8", 8192, 8192, 1), 90, 2),
            ("u8_4096_q90_smooth", smooth("u8", 4096, 4096, 2), 90, 2),
            ("rgba8_1080p_q85_444_smooth", smooth("rgba8", 1080, 1920, 3), 85, 0),
            ("rgb8_8192_q100_444_noise", noise("rgb8", 8192, 8192, 4), 100, 0)]
    for name, img, q, sub in work:
        dev = zb.Image.from_numpy(img)
        data = dev.encode_jpeg(q, sub)
        torch.cuda.synchronize()
        walls = []
        for _ in range(5):
            t0 = time.perf_counter()
            dev.encode_jpeg(q, sub)
            walls.append((time.perf_counter() - t0) * 1e3)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            dev.encode_jpeg(q, sub)
        kern = sum(e.self_device_time_total for e in prof.key_averages() if "jpeg" in e.key or "scan_" in e.key) / 1e3
        t0 = time.perf_counter()
        want = jo.encode(img, q, sub)
        oracle_ms = (time.perf_counter() - t0) * 1e3
        assert want == data, name
        res[name] = {"kernels_ms": round(kern, 3), "end_to_end_ms": round(float(np.median(walls)), 3), "bytes": len(data),
                     "oracle_1thread_ms": round(oracle_ms, 1)}
    print(json.dumps(res))


def jpeg_decode_timings():
    import io
    import subprocess
    import time

    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
    import jpeg_decode_oracle as jd
    from golden_jpeg import smooth
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"card": card.splitlines()[0] if card else torch.cuda.get_device_name()}
    try:
        from PIL import Image as PILImage
    except ImportError:
        PILImage = None
    try:
        import torchvision.io as tvio
        probe = zb.Image.from_numpy(smooth("rgb8", 64, 64, 1)).encode_jpeg()
        tvio.decode_jpeg(torch.frombuffer(bytearray(probe), dtype=torch.uint8), device="cuda")
    except Exception:
        tvio = None
    def textured(rows, cols, seed):   # a smooth gradient with +-25 levels of noise: every block carries AC detail, as photographs do
        rng = np.random.default_rng(seed)
        y, x = np.mgrid[0:rows, 0:cols]
        base = np.stack([(x * 7 + y * 3) % 256, (y * 5) % 256, ((x ^ y) * 3) % 256], -1)
        return np.clip(base + rng.integers(-25, 26, base.shape), 0, 255).astype(np.uint8)
    work = []
    for name, r, c in (("1080p", 1080, 1920), ("4096", 4096, 4096), ("8192", 8192, 8192)):
        work.append((f"enc_{name}_q90_420_textured", zb.Image.from_numpy(textured(r, c, r)).encode_jpeg(90, 2), r * c))
    # large flat areas give a nearly periodic bit stream in which a wrongly started decoder never re-synchronises (DESIGN.md §4.9)
    work.append(("enc_1080p_q90_420_smooth", zb.Image.from_numpy(smooth("rgb8", 1080, 1920, 1)).encode_jpeg(90, 2), 1080 * 1920))
    liza = (Path(__file__).resolve().parents[1] / "tests" / "golden" / "jpeg_decode" / "liza.jpg").read_bytes()
    work.append(("liza_1024_420", liza, 1024 * 1024))
    if PILImage is not None:   # a restart-interval stream written by Pillow (libjpeg)
        b = io.BytesIO()
        PILImage.fromarray(smooth("rgb8", 4096, 4096, 5)).save(b, "JPEG", quality=85, subsampling=2, restart_marker_blocks=4)
        work.append(("pillow_4096_restart4_420", b.getvalue(), 4096 * 4096))
    lim = zb.JpegLimits(max_width=0, max_height=0, max_pixels=0, max_blocks=0)
    olim = jd.Limits(max_width=0, max_height=0, max_pixels=0, max_blocks=0)
    for name, data, px in work:
        out = zb.Image.decode_jpeg(data, limits=lim)
        torch.cuda.synchronize()
        walls = []
        for _ in range(5):
            t0 = time.perf_counter()
            zb.Image.decode_jpeg(data, limits=lim, out=out)
            walls.append((time.perf_counter() - t0) * 1e3)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            zb.Image.decode_jpeg(data, limits=lim, out=out)
        per = {}
        for e in prof.key_averages():
            m = re.search(r"(dec_\w+|scan_\w+|Memcpy \w+|Memset)", e.key)
            if m and e.self_device_time_total > 0:
                per[m.group(1)] = round(per.get(m.group(1), 0) + e.self_device_time_total / 1e3, 3)
        e2e = float(np.median(walls))
        row = {"bytes": len(data), "kernels_ms": per, "end_to_end_ms": round(e2e, 3), "MB_s": round(len(data) / e2e / 1e3, 1),
               "MP_s": round(px / e2e / 1e3, 1)}
        t0 = time.perf_counter()
        want = jd.native(data, olim)
        row["oracle_1thread_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        assert np.array_equal(out.to_numpy(), want), name
        if PILImage is not None:
            ts = []
            for _ in range(3):
                t0 = time.perf_counter()
                PILImage.open(io.BytesIO(data)).load()
                ts.append((time.perf_counter() - t0) * 1e3)
            row["pillow_1thread_ms"] = round(float(np.median(ts)), 2)
        if tvio is not None:
            raw = torch.frombuffer(bytearray(data), dtype=torch.uint8)
            tvio.decode_jpeg(raw, device="cuda")
            torch.cuda.synchronize()
            ts = []
            for _ in range(5):
                t0 = time.perf_counter()
                tvio.decode_jpeg(raw, device="cuda")
                torch.cuda.synchronize()
                ts.append((time.perf_counter() - t0) * 1e3)
            row["nvjpeg_ms"] = round(float(np.median(ts)), 2)
        res[name] = row
    print(json.dumps(res))


def jpeg_decode_batch_timings():
    import io
    import subprocess
    import time

    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
    import jpeg_decode_oracle as jd
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"card": card.splitlines()[0] if card else torch.cuda.get_device_name()}
    try:
        from PIL import Image as PILImage
    except ImportError:
        PILImage = None
    try:
        import torchvision.io as tvio
    except ImportError:
        tvio = None

    def textured(rows, cols, seed, gray=False):   # gradient plus +-25 levels of noise, as in --jpeg-decode
        rng = np.random.default_rng(seed)
        y, x = np.mgrid[0:rows, 0:cols]
        base = np.stack([(x * 7 + y * 3) % 256, (y * 5) % 256, ((x ^ y) * 3) % 256], -1)
        img = np.clip(base + rng.integers(-25, 26, base.shape), 0, 255).astype(np.uint8)
        return img[..., 0].copy() if gray else img

    liza = (Path(__file__).resolve().parents[1] / "tests" / "golden" / "jpeg_decode" / "liza.jpg").read_bytes()
    rng = np.random.default_rng(256)
    mixed = []
    for k in range(256):   # small encoder streams: 160^2 to 640 x 480, q75-95, gray / 4:4:4 / 4:2:0
        rows, cols = int(rng.integers(160, 481)), int(rng.integers(160, 641))
        kind = int(rng.integers(0, 3))
        img = textured(rows, cols, k, gray=kind == 0)
        mixed.append(zb.Image.from_numpy(img).encode_jpeg(int(rng.integers(75, 96)), 0 if kind == 1 else 2))
    hd = zb.Image.from_numpy(textured(1080, 1920, 1080)).encode_jpeg(90, 2)
    work = [(f"liza_x{n}", [liza] * n) for n in (1, 16, 256, 1024)] + [("mixed_256", mixed), ("enc_1080p_q90_420_x1", [hd])]

    def median_ms(fn, reps):
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(ts))

    for name, datas in work:
        n, nbytes = len(datas), sum(len(d) for d in datas)
        reps = 5 if n >= 256 else 11
        out = zb.Image.decode_jpeg_batch(datas)
        singles = [zb.Image.decode_jpeg(d) for d in datas]
        for o, s in zip(out, singles):
            assert np.array_equal(o.to_numpy(), s.to_numpy()), name
        batch_ms = median_ms(lambda: zb.Image.decode_jpeg_batch(datas), reps)
        loop_ms = median_ms(lambda: [zb.Image.decode_jpeg(d, out=o) for d, o in zip(datas, singles)], reps)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            zb.Image.decode_jpeg_batch(datas)
        per = {}
        for e in prof.key_averages():
            m = re.search(r"(dec_\w+|scan_\w+|Memcpy \w+|Memset)", e.key)
            if m and e.self_device_time_total > 0:
                per[m.group(1)] = round(per.get(m.group(1), 0) + e.self_device_time_total / 1e3, 3)
        dev_ms = sum(per.values())
        row = {"files": n, "bytes": nbytes, "batch_ms": round(batch_ms, 3), "batch_img_s": round(n / batch_ms * 1e3, 1),
               "batch_MB_s": round(nbytes / batch_ms / 1e3, 1), "device_ms": round(dev_ms, 3),
               "device_img_s": round(n / dev_ms * 1e3, 1), "device_MB_s": round(nbytes / dev_ms / 1e3, 1), "kernels_ms": per,
               "loop_decode_jpeg_ms": round(loop_ms, 3), "loop_img_s": round(n / loop_ms * 1e3, 1)}
        if n == 1:
            row["single_decode_jpeg_ms"] = round(median_ms(lambda: zb.Image.decode_jpeg(datas[0], out=singles[0]), 21), 3)
            row["batch_of_one_ms_21"] = round(median_ms(lambda: zb.Image.decode_jpeg_batch(datas), 21), 3)
        sample = datas[:64]   # the host baselines on up to 64 files, as a rate
        t0 = time.perf_counter()
        for d in sample:
            jd.native(d)
        row["oracle_1thread_img_s"] = round(len(sample) / (time.perf_counter() - t0), 1)
        if PILImage is not None:
            t0 = time.perf_counter()
            for d in sample:
                PILImage.open(io.BytesIO(d)).load()
            row["pillow_1thread_img_s"] = round(len(sample) / (time.perf_counter() - t0), 1)
        if tvio is not None:
            try:
                raws = [torch.frombuffer(bytearray(d), dtype=torch.uint8) for d in datas]
                tvio.decode_jpeg(raws, device="cuda")
                tv_ms = median_ms(lambda: tvio.decode_jpeg(raws, device="cuda"), reps)
                row["torchvision_list_cuda_img_s"] = round(n / tv_ms * 1e3, 1)
            except Exception as e:   # recorded, not fatal: torchvision is a reference only
                row["torchvision_list_cuda"] = f"failed: {type(e).__name__}"
        res[name] = row
        print(name, json.dumps(row), flush=True)
    print(json.dumps(res))


def main():
    if "--jpeg-decode-batch" in sys.argv:
        return jpeg_decode_batch_timings()
    if "--jpeg-decode" in sys.argv:
        return jpeg_decode_timings()
    if "--jpeg" in sys.argv:
        return jpeg_timings()
    if "--visual" in sys.argv:
        return visual_timings()
    if "--quantize" in sys.argv:
        return quantize_timings()
    if "--flood-fill" in sys.argv:
        return flood_fill_timings()
    if "--binary" in sys.argv:
        return binary_timings()
    if "--edges" in sys.argv:
        return edges_timings()
    if "--hough" in sys.argv:
        return hough_timings()
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
