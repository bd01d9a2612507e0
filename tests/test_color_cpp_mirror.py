"""The colour types of the C++ host mirror (zignal_b200/host/zignal.hpp): their layout is the one zb_color_image describes, their
(space, component) tags are the C ABI's, and DeviceImage<T>::convertInto picks zb_convert between the five pixel formats and
zb_convert_color for every other pair; run without a device, a convert_color call is refused with the C ABI's statuses."""
import shutil
import subprocess
import textwrap
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
LIB_DIR = ROOT / "zignal_b200" / "lib"

PROGRAM = textwrap.dedent(r"""
    #include <cstddef>
    #include <cstdio>
    #include "zignal_b200/host/zignal.hpp"
    using namespace zignal;
    static_assert(sizeof(Rgba<double>) == 32 && offsetof(Rgba<double>, a) == 24, "Rgba(f64) is packed r, g, b, a");
    static_assert(sizeof(Ycbcr<uint8_t>) == 3 && offsetof(Ycbcr<uint8_t>, cr) == 2, "Ycbcr(u8)");
    static_assert(sizeof(Lab<float>) == 12 && offsetof(Lab<float>, b) == 8, "Lab(f32)");
    static_assert(sizeof(Gray<float>) == 4, "Gray(f32)");
    static_assert(color_format_of<Ycbcr<uint8_t>>().space == ZB_SPACE_YCBCR && color_format_of<Rgb8>().space == ZB_SPACE_RGB, "space");
    static_assert(color_format_of<double>().space == ZB_SPACE_SCALAR && color_format_of<double>().component == ZB_COMPONENT_F64, "scalar");
    static_assert(color_format_of<Oklch<double>>().component == ZB_COMPONENT_F64, "component");
    static_assert(has_pixfmt<RgbaF32>() && !has_pixfmt<Gray<float>>() && !has_pixfmt<Rgba<double>>(), "pixfmt");
    template <typename T, typename U> void instantiate() { DeviceImage<T>{}.template convertInto<U>(DeviceImage<U>{}); }
    template void instantiate<Rgb8, Lab<float>>();
    template void instantiate<Lab<double>, Hsv<float>>();
    template void instantiate<Ycbcr<uint8_t>, uint8_t>();
    template void instantiate<double, Oklch<double>>();
    int main() {
        DeviceImage<Lab<float>> src{4, 4, nullptr, 4, nullptr};
        DeviceImage<Rgb<uint8_t>> bad{4, 5, nullptr, 5, nullptr};
        try { src.convertInto(bad); } catch (const Error& err) { std::printf("%d\n", err.status); }
        auto a = src.color_raw();
        std::printf("%d %d\n", a.space, a.component);
        return 0;
    }
""")


@pytest.mark.skipif(shutil.which("g++") is None, reason="no host compiler")
def test_cpp_colour_types_and_convert_into(tmp_path):
    if not (LIB_DIR / "libzignal_b200.so").exists():
        pytest.fail("libzignal_b200.so missing: run __graft_entry__.build()")
    src = tmp_path / "colour.cpp"
    src.write_text(PROGRAM)
    exe = tmp_path / "colour"
    gxx = "/usr/bin/g++" if Path("/usr/bin/g++").exists() else "g++"
    cmd = [gxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", str(ROOT), str(src), "-o", str(exe), "-L", str(LIB_DIR), "-lzignal_b200",
           f"-Wl,-rpath,{LIB_DIR}"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    assert out.stdout.split() == ["1", "3", "1"]   # DimensionMismatch; Lab = 3, f32 = 1
