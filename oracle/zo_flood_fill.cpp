// zo_flood_fill.cpp -- CPU oracle of Image.floodFill (image.zig:831-840, image/flood_fill.zig:1-131).  TEST INFRASTRUCTURE ONLY (see
// zignal_oracle.h).  Restates the reference line by line on one thread: the explicit stack, the dense `visited` array indexed by `cols`,
// pixelDistance in f64 (built with -ffp-contract=off, so d * d and the sum are rounded separately, as in Zig).
//
// Built on its own into oracle/libzo_flood_fill.so (Makefile; ctypes binding in tests/flood_fill_oracle.py), so its entry point is
// declared here rather than in zignal_oracle.h.  Statuses use the values of zignal_b200.h.
#include <cmath>
#include <vector>

#include "zo_common.h"

extern "C" {
enum { ZO_FLOOD_OK = 0, ZO_FLOOD_UNSUPPORTED = 3, ZO_FLOOD_INVALID_ARGUMENT = 5, ZO_FLOOD_OUT_OF_BOUNDS = 27 };
enum { ZO_FLOOD_SEED = 0, ZO_FLOOD_NEIGHBOR = 1 };   // FloodFillOptions.ThresholdMode, flood_fill.zig:11-16
int zo_flood_fill(zo_image* img, int pixfmt, uint32_t start_row, uint32_t start_col, const void* fill_value, double threshold,
                  int connectivity, int mode);
}

namespace zo {
namespace {

struct Rgb8 { uint8_t r, g, b; };
struct Rgba8 { uint8_t r, g, b, a; };
struct RgbaF32 { float r, g, b, a; };

// :28-51 pixelDistance.  .int, .float: @abs(as(f64, p1) - as(f64, p2)).
double pixel_distance(uint8_t p1, uint8_t p2) { return std::fabs((double)p1 - (double)p2); }
double pixel_distance(float p1, float p2) { return std::fabs((double)p1 - (double)p2); }
// .@"struct": sum_sq += diff * diff over the fields in declaration order, then @sqrt.
double pixel_distance(Rgb8 p1, Rgb8 p2) {
    double sum_sq = 0.0;
    double diff = (double)p1.r - (double)p2.r;
    sum_sq += diff * diff;
    diff = (double)p1.g - (double)p2.g;
    sum_sq += diff * diff;
    diff = (double)p1.b - (double)p2.b;
    sum_sq += diff * diff;
    return std::sqrt(sum_sq);
}
template <typename S> double pixel_distance4(S p1, S p2) {
    double sum_sq = 0.0;
    double diff = (double)p1.r - (double)p2.r;
    sum_sq += diff * diff;
    diff = (double)p1.g - (double)p2.g;
    sum_sq += diff * diff;
    diff = (double)p1.b - (double)p2.b;
    sum_sq += diff * diff;
    diff = (double)p1.a - (double)p2.a;
    sum_sq += diff * diff;
    return std::sqrt(sum_sq);
}
double pixel_distance(Rgba8 p1, Rgba8 p2) { return pixel_distance4(p1, p2); }
double pixel_distance(RgbaF32 p1, RgbaF32 p2) { return pixel_distance4(p1, p2); }

// :54-57 neighbor_offsets in row / col order; the first four are 4-connectivity.
const int kOffsets[8][2] = {{-1, 0}, {1, 0}, {0, -1}, {0, 1}, {-1, -1}, {-1, 1}, {1, -1}, {1, 1}};

template <typename T>
int flood_fill(Img<T> image, uint32_t start_row, uint32_t start_col, T fill_value, double threshold, int connectivity, int mode) {
    // :68-70
    if (start_row >= image.rows || start_col >= image.cols) return ZO_FLOOD_OUT_OF_BOUNDS;
    // :72
    const T seed_val = image.at(start_row, start_col);
    struct Coord { uint32_t r, c; };
    std::vector<Coord> stack;   // :75-76
    // :78-81 `visited` is densely packed (indexed by `cols`)
    std::vector<bool> visited((size_t)image.rows * image.cols, false);
    // :83-84
    stack.push_back({start_row, start_col});
    visited[(size_t)start_row * image.cols + start_col] = true;
    // :93-103 Ctx.check
    auto check = [&](uint32_t nr, uint32_t nc, T comp) {
        const size_t idx = (size_t)nr * image.cols + nc;
        if (!visited[idx]) {
            const T val = image.at(nr, nc);
            if (pixel_distance(val, comp) <= threshold) {
                visited[idx] = true;
                stack.push_back({nr, nc});
            }
        }
    };
    // :114 neighbor_count = connectivity's tag value
    const int neighbor_count = connectivity;
    // :116-130
    while (!stack.empty()) {
        const Coord curr = stack.back();
        stack.pop_back();
        const T orig_val = image.at(curr.r, curr.c);
        image.at(curr.r, curr.c) = fill_value;
        const T compare_val = mode == ZO_FLOOD_SEED ? seed_val : orig_val;
        for (int k = 0; k < neighbor_count; ++k) {
            const int64_t nr = (int64_t)curr.r + kOffsets[k][0];
            const int64_t nc = (int64_t)curr.c + kOffsets[k][1];
            if (nr < 0 || nr >= image.rows || nc < 0 || nc >= image.cols) continue;
            check((uint32_t)nr, (uint32_t)nc, compare_val);
        }
    }
    return ZO_FLOOD_OK;
}

template <typename T>
int run(zo_image* img, uint32_t r, uint32_t c, const void* fill, double threshold, int connectivity, int mode) {
    T v;
    std::memcpy(&v, fill, sizeof(T));
    return flood_fill(Img<T>(img), r, c, v, threshold, connectivity, mode);
}

}  // namespace
}  // namespace zo

extern "C" int zo_flood_fill(zo_image* img, int pixfmt, uint32_t start_row, uint32_t start_col, const void* fill_value, double threshold,
                             int connectivity, int mode) {
    using namespace zo;
    if (!img || !fill_value) return ZO_FLOOD_INVALID_ARGUMENT;
    if ((connectivity != 4 && connectivity != 8) || (mode != ZO_FLOOD_SEED && mode != ZO_FLOOD_NEIGHBOR)) return ZO_FLOOD_INVALID_ARGUMENT;
    switch (pixfmt) {
        case ZO_PIX_U8: return run<uint8_t>(img, start_row, start_col, fill_value, threshold, connectivity, mode);
        case ZO_PIX_F32: return run<float>(img, start_row, start_col, fill_value, threshold, connectivity, mode);
        case ZO_PIX_RGB8: return run<Rgb8>(img, start_row, start_col, fill_value, threshold, connectivity, mode);
        case ZO_PIX_RGBA8: return run<Rgba8>(img, start_row, start_col, fill_value, threshold, connectivity, mode);
        case ZO_PIX_RGBAF32: return run<RgbaF32>(img, start_row, start_col, fill_value, threshold, connectivity, mode);
    }
    return ZO_FLOOD_UNSUPPORTED;
}
