"""The work plan of the fused RGBA f32 convolution (row segments x 256-px strips, edge strips cut apart from the inner ones;
zb_conv_fused.cu plan_units) against the oracle: exact mode bit-identical, FFMA mode within TOL_F32, every border mode, on shapes
where the plan is uneven -- one segment, segments of different heights, heights that are not a multiple of 8 per segment, images
narrower than one strip, ragged right edges -- and through the host pipeline's 256-row windows."""
import numpy as np
import pytest

import oracle_lib as zo
from gpu_utils import BORDERS, border_enum, rand_image, rel_err

pytestmark = pytest.mark.gpu
TOL_F32 = 1e-5  # BASELINE.json north_star: "within 1e-5 relative for f32 paths"

SHAPES = [
    (64, 8192),    # one segment (8 chunks)
    (129, 8192),   # two segments of 9 and 8 chunks, the last one ragged
    (300, 8190),   # 3 segments on the inner strips, 4 on the edge strips (the last one ragged), cols % 8 != 0
    (2100, 1024),  # .zero: 30 segments of 9 and 8 chunks over 4 strips; else 24 on the 2 inner strips and 32 on the 2 edge strips
    (1000, 264),   # 14 segments over two edge strips, the second 8 px wide
    (40, 100),     # smaller than one strip
    (203, 17),     # smaller than one strip, cols % 8 != 0
]


@pytest.fixture(scope="module")
def zb():
    import torch
    assert torch.cuda.is_available()
    import zignal_b200 as zb
    yield zb
    zb.lib().zb_set_exact_f32(0)


def _taps(rng, n):
    k = (rng.random(n) + 0.05).astype(np.float32)
    return (k / k.sum()).astype(np.float32)


@pytest.mark.parametrize("rows,cols", SHAPES)
@pytest.mark.parametrize("border", BORDERS)
def test_fused_rgbaf32_plan_shapes(zb, rows, cols, border):
    L = zb.lib()
    rng = np.random.default_rng(rows * 7919 + cols)
    img = rand_image(rng, (rows, cols, 4), np.float32)
    dev = zb.Image.from_numpy(img)
    for half in (2, 7):
        k = _taps(rng, 2 * half + 1)
        want = zo.conv_separable(img, k, k, border)
        try:
            L.zb_set_exact_f32(1)
            got = dev.convolve_separable(k, k, border_enum(zb, border)).to_numpy()
            assert L.zb_last_kernel().decode() == "fused_sep_rgbaf32_exact"
            assert np.array_equal(got, want), ("exact", half)
        finally:
            L.zb_set_exact_f32(0)
        got = dev.convolve_separable(k, k, border_enum(zb, border)).to_numpy()
        assert L.zb_last_kernel().decode() == "fused_sep_rgbaf32"
        assert rel_err(got, want) <= TOL_F32, ("fma", half)


@pytest.mark.parametrize("border", ["zero", "replicate", "mirror"])
def test_host_pipeline_row_windows(zb, border):
    """zb_host_gaussian_blur / zb_host_conv_separable run the kernel on 256-row windows [row0, row1) of a device copy while the
    next window uploads; 1100 rows leave a ragged last window of 76 rows."""
    L = zb.lib()
    rng = np.random.default_rng(11)
    img = rand_image(rng, (1100, 2048, 4), np.float32)   # 36 MB: above the pipeline's 32 MiB floor
    taps = zb.gaussian_taps(2.25)
    want = zo.conv_separable(img, taps, taps, border)
    bm = border_enum(zb, border)
    try:
        L.zb_set_exact_f32(1)
        got = zb.host_conv_separable(img, taps, taps, bm)
        assert L.zb_last_kernel().decode() == "fused_sep_rgbaf32_exact"
        assert np.array_equal(got, want)
    finally:
        L.zb_set_exact_f32(0)
    got = zb.host_conv_separable(img, taps, taps, bm)
    assert L.zb_last_kernel().decode() == "fused_sep_rgbaf32"
    assert rel_err(got, want) <= TOL_F32
    if border == "mirror":
        got = zb.host_gaussian_blur(img, 2.25)
        assert L.zb_last_kernel().decode() == "fused_sep_rgbaf32"
        assert rel_err(got, zo.gaussian_blur(img, 2.25)) <= TOL_F32
