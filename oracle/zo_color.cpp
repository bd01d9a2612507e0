// zo_color.cpp -- CPU oracle of convertColor between the 33 colour formats (reference color.zig:108-151, image.zig:396-421) (TEST
// INFRASTRUCTURE ONLY).  Built on its own by the Makefile with -ffp-contract=off, so every product and sum is rounded on its own as in
// the reference; hslToRgb's std.math.lerp is @mulAdd (a fused multiply-add), so it is std::fma here.
//
// Conversion in three stages, as the reference composes it: the source's `.as(C)` (C the compute type convertColor picks, :113-150),
// the hops of the `to` switches from the source's space to the destination's, and the destination's `.as(D)`.
//
// Transcendentals.  std.math.pow (lib/std/math/pow.zig of the pinned Zig) is restated with its special cases and its split of y into
// an integer part (frexp and repeated squaring, then scalbn) and a fraction (exp(yf * log(x))); exp, log, cbrt, atan2, sin and cos
// come from the host libm.  Zig builds those from its own compiler-rt, so outputs whose path uses them can differ from the reference
// by a few ulp; tests/test_color_host.py lists the known test values with their distance.
//
// @mod on floats follows Zig's LLVM lowering: fmod(a, b), and fmod(fmod(a, b) + b, b) when a < 0, so a tiny negative hue gives 0.
// hslToRgb's trunc(h / 60) -> usize traps in the reference for a NaN or infinite hue; here such a hue takes sector 0.
#include <cmath>
#include <cstddef>
#include <cstdint>

namespace {

using std::atan2;
using std::cbrt;
using std::cos;
using std::exp;
using std::fabs;
using std::fma;
using std::fmod;
using std::frexp;
using std::log;
using std::modf;
using std::round;
using std::scalbn;
using std::sin;
using std::sqrt;
using std::trunc;

enum { GRAY = 0, HSL, HSV, LAB, LCH, LMS, OKLAB, OKLCH, RGB, RGBA, XYB, XYZ, YCBCR, SCALAR, NSPACES };
enum { U8 = 0, F32 = 1, F64 = 2 };

struct ColorPlan {
    int ns, nd;
    int in_space, out_space;
    int nhops;
    uint32_t hops;
};

template <typename T> struct IsU8 { static constexpr bool value = false; };
template <> struct IsU8<uint8_t> { static constexpr bool value = true; };

// Zig's @min / @max on floats return the non-NaN operand; for equal operands (+0, -0) the second.
template <typename C> static inline C zmin(C a, C b) { return a != a ? b : (b != b ? a : (a < b ? a : b)); }
template <typename C> static inline C zmax(C a, C b) { return a != a ? b : (b != b ? a : (a > b ? a : b)); }
// std.math.clamp(v, lo, hi) = @max(lo, @min(v, hi)): NaN gives hi.
template <typename C> static inline C zclamp(C v, C lo, C hi) { return v < hi ? (v > lo ? v : lo) : hi; }

// @mod(a, b) on floats as Zig's LLVM backend lowers it: fmod, and for a < 0 fmod(fmod(a, b) + b, b), so the result lies in [0, b).
template <typename C> static inline C zmod(C a, C b) {
    const C r = fmod(a, b);
    return a < C(0) ? fmod(r + b, b) : r;
}

// std.math.pow(T, x, y) for f32 / f64 (lib/std/math/pow.zig): special cases, then exp(yf * log(x)) for the fraction of y times the
// integer part by frexp and repeated squaring, put together with scalbn.
template <typename C> static inline C zpow(C x, C y) {
    if (y == C(0) || x == C(1)) return C(1);
    if (x != x || y != y) return x + y;
    if (y == C(1)) return x;
    // y here is 2.4, 1 / 2.4 or 1 / 3, positive and not an odd integer, and every caller passes x > 0 or +inf; the two special
    // cases below are the reference's results for such a y
    if (x == C(0)) return C(0);
    if (std::isinf(x)) return C(INFINITY);   // pow(-inf, y) = pow(-0, -y) = +inf too
    C yi;
    C yf = modf(fabs(y), &yi);
    if (yf != C(0) && x < C(0)) return C(NAN);
    C a1 = C(1);
    int ae = 0;
    if (yf != C(0)) {
        if (yf > C(0.5)) { yf -= C(1); yi += C(1); }
        a1 = exp(yf * log(x));
    }
    int xe;
    C x1 = frexp(x, &xe);
    constexpr int overflow = 1 << ((sizeof(C) == 4 ? 8 : 11) + 1);
    for (long long i = (long long)yi; i != 0; i >>= 1) {
        if (xe < -overflow || overflow < xe) { ae += xe; break; }
        if (i & 1) { a1 *= x1; ae += xe; }
        x1 *= x1;
        xe <<= 1;
        if (x1 < C(0.5)) { x1 += x1; xe -= 1; }
    }
    if (y < C(0)) { a1 = C(1) / a1; ae = -ae; }
    return scalbn(a1, ae);
}

// ---- the conversion functions of color.zig, in compute type C (float or double) ----

template <typename C> static inline C gamma_to_linear(C c) {   // :1252-1258
    return c > C(0.04045) ? zpow((c + C(0.055)) / C(1.055), C(2.4)) : c / C(12.92);
}
template <typename C> static inline C linear_to_gamma(C c) {   // :1243-1249
    return c > C(0.0031308) ? C(1.055) * zpow(c, C(1.0 / 2.4)) - C(0.055) : c * C(12.92);
}
template <typename C> static inline C lab_forward(C t) {       // :1289-1291
    return t > C(0.008856) ? zpow(t, C(1.0 / 3.0)) : C(7.787) * t + C(16.0 / 116.0);
}

template <typename C> static inline void rgb_to_hsv(C* v) {    // :1087-1108
    const C r = v[0], g = v[1], b = v[2];
    const C mn = zmin(r, zmin(g, b)), mx = zmax(r, zmax(g, b)), delta = mx - mn;
    C h;
    if (delta == C(0)) h = C(0);
    else if (mx == r) h = (g - b) / delta * C(60);
    else if (mx == g) h = C(120) + (b - r) / delta * C(60);
    else h = C(240) + (r - g) / delta * C(60);
    v[0] = zmod(h, C(360));
    v[1] = mx == C(0) ? C(0) : (delta / mx) * C(100);
    v[2] = mx * C(100);
}
template <typename C> static inline void rgb_to_hsl(C* v) {    // :1150-1174
    const C r = v[0], g = v[1], b = v[2];
    const C mn = zmin(r, zmin(g, b)), mx = zmax(r, zmax(g, b)), delta = mx - mn;
    C hue;
    if (delta == C(0)) hue = C(0);
    else if (mx == r) hue = (g - b) / delta;
    else if (mx == g) hue = C(2) + (b - r) / delta;
    else hue = C(4) + (r - g) / delta;
    const C l = (mx + mn) / C(2);
    const C s = delta == C(0) ? C(0) : (l < C(0.5) ? delta / (C(2) * l) : delta / (C(2) - C(2) * l));
    v[0] = zmod(hue * C(60), C(360));
    v[1] = zclamp(s, C(0), C(1)) * C(100);
    v[2] = zclamp(l, C(0), C(1)) * C(100);
}
// hslToRgb (:1111-1147).  The reference converts trunc(h / 60) to usize, which traps for a NaN or infinite hue; here such a hue
// takes sector 0, so its fraction (NaN) reaches every channel the sector's factors use.  std.math.lerp(a, b, t) is
// @mulAdd(T, b - a, t, a).
template <typename C> static inline void hsl_to_rgb(C* v) {
    const C h = zmod(v[0], C(360));
    const C s = zclamp(v[1] / C(100), C(0), C(1));
    const C l = zclamp(v[2] / C(100), C(0), C(1));
    const C hue_sector = h / C(60);
    const C tr = trunc(hue_sector);
    const int sector = tr == tr && !std::isinf(tr) ? (int)tr : 0;
    const C f = hue_sector - C(sector);
    C k0, k1, k2;
    switch (sector % 6) {
        case 0: k0 = C(1); k1 = f; k2 = C(0); break;
        case 1: k0 = C(1) - f; k1 = C(1); k2 = C(0); break;
        case 2: k0 = C(0); k1 = C(1); k2 = f; break;
        case 3: k0 = C(0); k1 = C(1) - f; k2 = C(1); break;
        case 4: k0 = f; k1 = C(0); k2 = C(1); break;
        default: k0 = C(1); k1 = C(0); k2 = C(1) - f; break;
    }
    const C r = fma(C(2) * k0 - C(1), s, C(1));
    const C g = fma(C(2) * k1 - C(1), s, C(1));
    const C b = fma(C(2) * k2 - C(1), s, C(1));
    if (l < C(0.5)) {
        v[0] = r * l; v[1] = g * l; v[2] = b * l;
    } else {
        v[0] = fma(C(2) - r, l, r) - C(1);
        v[1] = fma(C(2) - g, l, g) - C(1);
        v[2] = fma(C(2) - b, l, b) - C(1);
    }
}
template <typename C> static inline void hsv_to_rgb(C* v) {    // :1177-1208
    const C hue = zclamp(v[0] / C(360), C(0), C(1));
    const C sat = zclamp(v[1] / C(100), C(0), C(1));
    const C val = zclamp(v[2] / C(100), C(0), C(1));
    if (sat == C(0)) { v[0] = v[1] = v[2] = val; return; }
    const C sector = hue * C(6);
    const int index = (int)trunc(sector);
    const C f = sector - C(index);
    const C p = val * (C(1) - sat);
    const C q = val * (C(1) - (sat * f));
    const C t = val * (C(1) - sat * (C(1) - f));
    switch (index % 6) {
        case 0: v[0] = val; v[1] = t; v[2] = p; break;
        case 1: v[0] = q; v[1] = val; v[2] = p; break;
        case 2: v[0] = p; v[1] = val; v[2] = t; break;
        case 3: v[0] = p; v[1] = q; v[2] = val; break;
        case 4: v[0] = t; v[1] = p; v[2] = val; break;
        default: v[0] = val; v[1] = p; v[2] = q; break;
    }
}
template <typename C> static inline void hsv_to_hsl(C* v) {    // :1211-1224
    const C s_v = v[1] / C(100), val = v[2] / C(100);
    const C l = val * (C(1) - s_v / C(2));
    const C s_l = (l == C(0) || l == C(1)) ? C(0) : (val - l) / zmin(l, C(1) - l);
    v[1] = s_l * C(100);
    v[2] = l * C(100);
}
template <typename C> static inline void hsl_to_hsv(C* v) {    // :1227-1240
    const C s_l = v[1] / C(100), l = v[2] / C(100);
    const C val = l + s_l * zmin(l, C(1) - l);
    const C s_v = val == C(0) ? C(0) : C(2) * (C(1) - l / val);
    v[1] = s_v * C(100);
    v[2] = val * C(100);
}
// The linear-RGB -> XYZ product of rgbToXyz / xybToXyz (:1267-1271, :1475-1479).
template <typename C> static inline void linear_to_xyz(C r, C g, C b, C* v) {
    v[0] = (r * C(0.4124) + g * C(0.3576) + b * C(0.1805)) * C(100);
    v[1] = (r * C(0.2126) + g * C(0.7152) + b * C(0.0722)) * C(100);
    v[2] = (r * C(0.0193) + g * C(0.1192) + b * C(0.9505)) * C(100);
}
// The XYZ -> linear-RGB product of xyzToRgb / xyzToXyb (:1277-1279, :1437-1439).
template <typename C> static inline void xyz_to_linear(const C* v, C* r, C* g, C* b) {
    *r = (v[0] * C(3.2406) + v[1] * C(-1.5372) + v[2] * C(-0.4986)) / C(100);
    *g = (v[0] * C(-0.9689) + v[1] * C(1.8758) + v[2] * C(0.0415)) / C(100);
    *b = (v[0] * C(0.0557) + v[1] * C(-0.2040) + v[2] * C(1.0570)) / C(100);
}
// Linear RGB -> XYB (:1441-1453, :1489-1501).
template <typename C> static inline void linear_to_xyb(C r, C g, C b, C* v) {
    const C bias = C(0.00379307325527544933), enc = C(0.15595420054924863);
    const C l = zmax(C(0), C(0.30) * r + C(0.622) * g + C(0.078) * b + bias);
    const C m = zmax(C(0), C(0.23) * r + C(0.692) * g + C(0.078) * b + bias);
    const C s = zmax(C(0), C(0.24342268924547819) * r + C(0.20476744424496821) * g + C(0.5518098665095536) * b + bias);
    const C ld = cbrt(l) - enc, md = cbrt(m) - enc, sd = cbrt(s) - enc;
    v[0] = C(0.5) * (ld - md);
    v[1] = C(0.5) * (ld + md);
    v[2] = sd;
}
// XYB -> linear RGB (:1459-1473, :1507-1521).
template <typename C> static inline void xyb_to_linear(const C* v, C* r, C* g, C* b) {
    const C bias = C(0.00379307325527544933), dec = C(0.15594113236791331);
    const C lc = (v[1] + v[0]) + dec, mc = (v[1] - v[0]) + dec, sc = v[2] + dec;
    const C l = (lc * lc * lc) - bias, m = (mc * mc * mc) - bias, s = (sc * sc * sc) - bias;
    *r = C(11.031566901960783) * l - C(9.866943921568629) * m - C(0.16462299647058826) * s;
    *g = C(-3.254147380392157) * l + C(4.418770392156863) * m - C(0.16462299647058826) * s;
    *b = C(-3.6588512862745097) * l + C(2.7129230470588235) * m + C(1.9459282392156863) * s;
}
template <typename C> static inline void xyz_to_lab(C* v) {    // :1294-1308
    const C fx = lab_forward(v[0] / C(95.047)), fy = lab_forward(v[1] / C(100.0)), fz = lab_forward(v[2] / C(108.883));
    v[0] = zmax(C(0), C(116.0) * fy - C(16.0));
    v[1] = C(500.0) * (fx - fy);
    v[2] = C(200.0) * (fy - fz);
}
// labToXyz (:1311-1330): the first quotients in T, everything after in f64.
template <typename C> static inline void lab_to_xyz(C* v) {
    const double fy = (double)((v[0] + C(16.0)) / C(116.0));
    const double fx = (double)(v[1] / C(500.0)) + fy;
    const double fz = fy - (double)(v[2] / C(200.0));
    const double y3 = fy * fy * fy, x3 = fx * fx * fx, z3 = fz * fz * fz;
    const double delta = 16.0 / 116.0;
    const double y = y3 > 0.008856 ? y3 : (fy - delta) / 7.787;
    const double x = x3 > 0.008856 ? x3 : (fx - delta) / 7.787;
    const double z = z3 > 0.008856 ? z3 : (fz - delta) / 7.787;
    v[0] = C(x * 95.047);
    v[1] = C(y * 100.000);
    v[2] = C(z * 108.883);
}
// cartesianToCylindrical / cylindricalToCartesian (:1333-1344): std.math.radiansToDegrees / degreesToRadians multiply by
// deg_per_rad / rad_per_deg.
template <typename C> static inline void to_cylindrical(C* v) {
    const C a = v[1], b = v[2];
    v[1] = sqrt(a * a + b * b);
    v[2] = zmod(atan2(b, a) * C(57.295779513082320876798154814105170332405472466564321549160243861), C(360.0));
}
template <typename C> static inline void to_cartesian(C* v) {
    const C c = v[1];
    const C h = v[2] * C(0.017453292519943295769236907684886127134428718885417254560971914);
    v[1] = c * cos(h);
    v[2] = c * sin(h);
}
template <typename C> static inline void xyz_to_lms(C* v) {    // :1361-1368
    const C x = v[0], y = v[1], z = v[2];
    v[0] = (C(0.8951) * x + C(0.2664) * y - C(0.1614) * z) / C(100);
    v[1] = (C(-0.7502) * x + C(1.7135) * y + C(0.0367) * z) / C(100);
    v[2] = (C(0.0389) * x - C(0.0685) * y + C(1.0296) * z) / C(100);
}
template <typename C> static inline void lms_to_xyz(C* v) {    // :1371-1378
    const C l = v[0], m = v[1], s = v[2];
    v[0] = C(100) * (C(0.9869929) * l - C(0.1470543) * m + C(0.1599627) * s);
    v[1] = C(100) * (C(0.4323053) * l + C(0.5183603) * m + C(0.0492912) * s);
    v[2] = C(100) * (C(-0.0085287) * l + C(0.0400428) * m + C(0.9684867) * s);
}
template <typename C> static inline void xyz_to_oklab(C* v) {  // :1381-1400
    const C x = v[0] / C(100.0), y = v[1] / C(100.0), z = v[2] / C(100.0);
    const C ll = C(0.8189330101) * x + C(0.3618667424) * y - C(0.1288597137) * z;
    const C ml = C(0.0329845436) * x + C(0.9293118715) * y + C(0.0361456387) * z;
    const C sl = C(0.0482003018) * x + C(0.2643662691) * y + C(0.6338517070) * z;
    const C ld = cbrt(ll), md = cbrt(ml), sd = cbrt(sl);
    v[0] = C(0.2104542553) * ld + C(0.7936177850) * md - C(0.0040720468) * sd;
    v[1] = C(1.9779984951) * ld - C(2.4285922050) * md + C(0.4505937099) * sd;
    v[2] = C(0.0259040371) * ld + C(0.7827717662) * md - C(0.8086757660) * sd;
}
template <typename C> static inline void oklab_to_xyz(C* v) {  // :1403-1418
    const C l = v[0], a = v[1], b = v[2];
    const C ld = l + C(0.3963377774) * a + C(0.2158037573) * b;
    const C md = l - C(0.1055613458) * a - C(0.0638541728) * b;
    const C sd = l - C(0.0894841775) * a - C(1.2914855480) * b;
    const C ll = ld * ld * ld, ml = md * md * md, sl = sd * sd * sd;
    v[0] = C(100.0) * (C(1.2270138511) * ll - C(0.5577999807) * ml + C(0.2812561490) * sl);
    v[1] = C(100.0) * (C(-0.0405801784) * ll + C(1.1122568696) * ml - C(0.0716766787) * sl);
    v[2] = C(100.0) * (C(-0.0763812845) * ll - C(0.4214819784) * ml + C(1.5861632204) * sl);
}
template <typename C> static inline void rgb_to_ycbcr(C* v) {  // :1009-1016
    const C y = zclamp(C(0.299) * v[0] + C(0.587) * v[1] + C(0.114) * v[2], C(0), C(1));
    const C cb = zclamp((v[2] - y) / C(1.772), C(-0.5), C(0.5));
    const C cr = zclamp((v[0] - y) / C(1.402), C(-0.5), C(0.5));
    v[0] = y; v[1] = cb; v[2] = cr;
}
template <typename C> static inline void ycbcr_to_rgb(C* v) {  // :1068-1083
    const C y = v[0], cb = v[1], cr = v[2];
    const C r = y + C(1.402) * cr;
    const C g = y - C(0.344136) * cb - C(0.714136) * cr;
    const C b = y + C(1.772) * cb;
    v[0] = zclamp(r, C(0), C(1)); v[1] = zclamp(g, C(0), C(1)); v[2] = zclamp(b, C(0), C(1));
}

// One hop of a `to` switch, from space `s` to space `t`, in place on v.  Only the edges next_hop produces occur.
template <typename C> static inline void hop(int s, int t, C* v) {
    if constexpr (IsU8<C>::value) {
        // u8 colours: Gray, Rgb, Rgba and Ycbcr only, in the reference's integer arithmetic
        if (s == GRAY) { v[1] = v[2] = v[0]; }                                        // grayToRgb :1050-1052
        else if (s == RGBA) { }                                                       // drop alpha :478
        else if (s == YCBCR) {                                                        // ycbcrToRgb :1058-1067
            const long long y = v[0], cb = (long long)v[1] - 128, cr = (long long)v[2] - 128;
            const long long r = (65536 * y + 91881 * cr + 32768) >> 16;
            const long long g = (65536 * y - 22554 * cb - 46802 * cr + 32768) >> 16;
            const long long b = (65536 * y + 116130 * cb + 32768) >> 16;
            v[0] = (uint8_t)(r < 0 ? 0 : r > 255 ? 255 : r);
            v[1] = (uint8_t)(g < 0 ? 0 : g > 255 ? 255 : g);
            v[2] = (uint8_t)(b < 0 ? 0 : b > 255 ? 255 : b);
        } else if (t == GRAY) {                                                       // rgbToGray :1032-1041
            const int y = (13933 * (int)v[0] + 46871 * (int)v[1] + 4732 * (int)v[2] + 32768) >> 16;
            v[0] = (uint8_t)(y < 0 ? 0 : y > 255 ? 255 : y);
        } else if (t == RGBA) {
            v[3] = 255;
        } else {                                                                      // rgbToYcbcr :988-1008
            const long long r = v[0], g = v[1], b = v[2];
            const long long y = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
            const long long cb = ((-11059 * r - 21710 * g + 32768 * b + 32768) >> 16) + 128;
            const long long cr = ((32768 * r - 27439 * g - 5329 * b + 32768) >> 16) + 128;
            v[0] = (uint8_t)(y < 0 ? 0 : y > 255 ? 255 : y);
            v[1] = (uint8_t)(cb < 0 ? 0 : cb > 255 ? 255 : cb);
            v[2] = (uint8_t)(cr < 0 ? 0 : cr > 255 ? 255 : cr);
        }
    } else {
        switch (s) {
            case GRAY: v[1] = v[2] = v[0]; break;
            case RGBA: break;
            case HSL: if (t == HSV) hsl_to_hsv(v); else hsl_to_rgb(v); break;
            case HSV: if (t == HSL) hsv_to_hsl(v); else hsv_to_rgb(v); break;
            case YCBCR: ycbcr_to_rgb(v); break;
            case LAB: if (t == LCH) to_cylindrical(v); else lab_to_xyz(v); break;
            case LCH: to_cartesian(v); break;
            case OKLAB: if (t == OKLCH) to_cylindrical(v); else oklab_to_xyz(v); break;
            case OKLCH: to_cartesian(v); break;
            case LMS: lms_to_xyz(v); break;
            case XYB: {
                C r, g, b;
                xyb_to_linear(v, &r, &g, &b);
                if (t == XYZ) { linear_to_xyz(r, g, b, v); break; }
                v[0] = zclamp(linear_to_gamma(r), C(0), C(1));
                v[1] = zclamp(linear_to_gamma(g), C(0), C(1));
                v[2] = zclamp(linear_to_gamma(b), C(0), C(1));
                break;
            }
            case XYZ:
                if (t == LAB) xyz_to_lab(v);
                else if (t == LMS) xyz_to_lms(v);
                else if (t == OKLAB) xyz_to_oklab(v);
                else {
                    C r, g, b;
                    xyz_to_linear(v, &r, &g, &b);
                    if (t == XYB) { linear_to_xyb(r, g, b, v); break; }
                    v[0] = zclamp(linear_to_gamma(r), C(0), C(1));
                    v[1] = zclamp(linear_to_gamma(g), C(0), C(1));
                    v[2] = zclamp(linear_to_gamma(b), C(0), C(1));
                }
                break;
            default:   // RGB
                if (t == GRAY) {
                    v[0] = zclamp(C(0.2126) * v[0] + C(0.7152) * v[1] + C(0.0722) * v[2], C(0), C(1));
                } else if (t == HSL) rgb_to_hsl(v);
                else if (t == HSV) rgb_to_hsv(v);
                else if (t == RGBA) v[3] = C(1);
                else if (t == YCBCR) rgb_to_ycbcr(v);
                else {
                    const C r = gamma_to_linear(v[0]), g = gamma_to_linear(v[1]), b = gamma_to_linear(v[2]);
                    if (t == XYB) linear_to_xyb(r, g, b, v);
                    else linear_to_xyz(r, g, b, v);
                }
                break;
        }
    }
}

// `.as(U)` of a colour of space `sp` from T to U (color.zig:365-388, 484-510, 541-558, 952-980; the other spaces only cast floats).
template <typename T, typename U> static inline void as_type(int sp, int n, const T* in, U* out) {
    if constexpr (IsU8<T>::value && IsU8<U>::value) {
        for (int k = 0; k < 4; ++k) if (k < n) out[k] = in[k];
    } else if constexpr (IsU8<T>::value) {
        for (int k = 0; k < 4; ++k)
            if (k < n) out[k] = (sp == YCBCR && k > 0) ? (U(in[k]) - U(128)) / U(255) : U(in[k]) / U(255);
    } else if constexpr (IsU8<U>::value) {
        for (int k = 0; k < 4; ++k) {
            if (k < n) {
                const T x = (sp == YCBCR && k > 0) ? in[k] + T(0.5) : in[k];
                out[k] = (uint8_t)round(T(255) * zclamp(x, T(0), T(1)));
            }
        }
    } else {
        for (int k = 0; k < 4; ++k) if (k < n) out[k] = U(in[k]);
    }
}

// convertColor for one pixel: s has p.ns components of S, d receives p.nd components of D; C is the compute type.
template <typename S, typename D, typename C> static inline void convert_pixel(const ColorPlan& p, const S* s, D* d) {
    C v[4] = {};
    as_type<S, C>(p.in_space, p.ns, s, v);
    int sp = p.in_space;
    for (int i = 0; i < p.nhops; ++i) {
        const int t = (p.hops >> (4 * i)) & 15;
        hop<C>(sp, t, v);
        sp = t;
    }
    as_type<C, D>(p.out_space, p.nd, v, d);
}


int channels_of_space(int space) { return space == RGBA ? 4 : (space == GRAY || space == SCALAR) ? 1 : 3; }

bool valid_format(int space, int component) {
    if (space < 0 || space >= NSPACES || component < U8 || component > F64) return false;
    return component != U8 || space == SCALAR || space == GRAY || space == RGB || space == RGBA || space == YCBCR;
}

// color.zig's `to` switches: the next space from s towards t.
int next_hop(int s, int t) {
    switch (s) {
        case GRAY: return RGB;                                                                   // :533-538
        case RGBA: return RGB;                                                                   // :475-481
        case YCBCR: return RGB;                                                                  // :943-948
        case RGB:                                                                                // :350-361
            return (t == GRAY || t == HSL || t == HSV || t == RGBA || t == XYB || t == XYZ || t == YCBCR) ? t : XYZ;
        case HSV: return t == HSL ? HSL : RGB;                                                   // :586-592
        case HSL: return t == HSV ? HSV : RGB;                                                   // :624-630
        case XYZ:                                                                                // :667-678
            if (t == LAB || t == LMS || t == OKLAB || t == RGB || t == XYB) return t;
            return t == LCH ? LAB : t == OKLCH ? OKLAB : RGB;
        case LAB: return t == LCH ? LCH : XYZ;                                                   // :711-717
        case LCH: return LAB;                                                                    // :750-755
        case LMS: return XYZ;                                                                    // :786-791
        case OKLAB: return t == OKLCH ? OKLCH : XYZ;                                             // :824-830
        case OKLCH: return OKLAB;                                                                // :863-868
        default: return t == RGB ? RGB : XYZ;                                                    // Xyb :902-908
    }
}

int make_plan(int s_space, int s_comp, int d_space, int d_comp, ColorPlan* p) {
    p->ns = channels_of_space(s_space);
    p->nd = channels_of_space(d_space);
    p->in_space = s_space == SCALAR ? GRAY : s_space;
    p->out_space = d_space == SCALAR ? GRAY : d_space;
    int c;
    if (s_space == SCALAR && d_space == SCALAR) c = s_comp == U8 ? d_comp : d_comp == U8 ? F64 : d_comp;   // :113-119
    else if (s_space == SCALAR) c = d_comp;                                                               // :121-131
    else if (d_space == SCALAR) c = s_comp;                                                               // :133-136
    else c = d_comp != U8 ? d_comp : s_comp;                                                              // :144-150
    p->nhops = 0;
    p->hops = 0;
    for (int sp = p->in_space; sp != p->out_space; ++p->nhops) {
        sp = next_hop(sp, p->out_space);
        p->hops |= (uint32_t)sp << (4 * p->nhops);
    }
    return c;
}

template <typename S, typename D, typename C>
void run(const ColorPlan& p, const void* src, void* dst, size_t n) {
    const S* s = (const S*)src;
    D* d = (D*)dst;
    for (size_t i = 0; i < n; ++i) {
        S in[4] = {};
        for (int k = 0; k < p.ns; ++k) in[k] = s[i * p.ns + k];
        D out[4];
        convert_pixel<S, D, C>(p, in, out);
        for (int k = 0; k < p.nd; ++k) d[i * p.nd + k] = out[k];
    }
}

template <typename S, typename D>
void run_c(int c, const ColorPlan& p, const void* src, void* dst, size_t n) {
    if (c == U8) run<S, D, uint8_t>(p, src, dst, n);
    else if (c == F32) run<S, D, float>(p, src, dst, n);
    else run<S, D, double>(p, src, dst, n);
}
template <typename S>
void run_dc(int dc, int c, const ColorPlan& p, const void* src, void* dst, size_t n) {
    if (dc == U8) run_c<S, uint8_t>(c, p, src, dst, n);
    else if (dc == F32) run_c<S, float>(c, p, src, dst, n);
    else run_c<S, double>(c, p, src, dst, n);
}

}  // namespace

extern "C" {

// 1 when (space, component) is one of the 33 formats.
int zo_color_valid(int space, int component) { return valid_format(space, component) ? 1 : 0; }

// The spaces a conversion visits after the source's, lowest 4 bits first; returns their number (-1 for an invalid pair).
int zo_color_path(int s_space, int s_comp, int d_space, int d_comp, uint32_t* hops) {
    if (!valid_format(s_space, s_comp) || !valid_format(d_space, d_comp)) return -1;
    ColorPlan p;
    make_plan(s_space, s_comp, d_space, d_comp, &p);
    *hops = p.hops;
    return p.nhops;
}

// dst[i] = convertColor(dst format, src[i]) for n contiguous pixels.  Returns 0, or 3 (Unsupported) for an invalid format.
int zo_convert_color(const void* src, int s_space, int s_comp, void* dst, int d_space, int d_comp, size_t n) {
    if (!valid_format(s_space, s_comp) || !valid_format(d_space, d_comp)) return 3;
    ColorPlan p;
    const int c = make_plan(s_space, s_comp, d_space, d_comp, &p);
    if (s_space == d_space && s_comp == d_comp) {   // image.zig:398
        const size_t bytes = n * (size_t)p.ns * (s_comp == U8 ? 1 : s_comp == F32 ? 4 : 8);
        for (size_t i = 0; i < bytes; ++i) ((uint8_t*)dst)[i] = ((const uint8_t*)src)[i];
        return 0;
    }
    if (s_comp == U8) run_dc<uint8_t>(d_comp, c, p, src, dst, n);
    else if (s_comp == F32) run_dc<float>(d_comp, c, p, src, dst, n);
    else run_dc<double>(d_comp, c, p, src, dst, n);
    return 0;
}

}  // extern "C"
