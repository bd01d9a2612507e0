// zo_hough.cpp -- CPU oracle of HoughTransform (image/hough.zig:10-257).  TEST INFRASTRUCTURE ONLY (see zignal_oracle.h).
// Restates init (:38-66), compute (:75-139), findLines (:142-204), getLineProperties (:207-212), createLine (:214-229) and clipLine
// (:232-257) line by line on one thread: i32 votes with arithmetic shifts, f32 geometry (built with -ffp-contract=off; cosf / sinf are
// the host libm's), a stable sort by score.
//
// Built on its own into oracle/libzo_hough.so (Makefile; ctypes binding in tests/hough_oracle.py), so its entry points are declared
// here rather than in zignal_oracle.h.  Statuses use the values of zignal_b200.h.
#include <algorithm>
#include <cmath>
#include <vector>

#include "zo_common.h"

extern "C" {
enum { ZO_HOUGH_OK = 0, ZO_HOUGH_DIMENSION_MISMATCH = 1, ZO_HOUGH_UNSUPPORTED = 3, ZO_HOUGH_INVALID_ARGUMENT = 5 };
typedef struct zo_hough_line { float angle, radius; uint32_t score; float p1x, p1y, p2x, p2y; } zo_hough_line;   // Line, :13-25
int zo_hough_tables(uint32_t size, int32_t* cos_table, int32_t* sin_table);
int zo_hough_compute(uint32_t size, const zo_image* edges, uint32_t l, uint32_t t, uint32_t r, uint32_t b, zo_image* accumulator);
int zo_hough_find_lines(uint32_t size, const zo_image* accumulator, uint32_t threshold, float angle_nms_thresh, float radius_nms_thresh,
                        zo_hough_line* out, uint32_t cap, uint32_t* n);
}

namespace zo {
namespace {

struct Hough {
    uint32_t size, even_size;
    std::vector<int32_t> cos_table, sin_table;
};

// :38-66 init.  size > 32768 is refused: the i32 rho of compute can overflow there (zignal_b200.h, zb_hough_create).
int hough_init(uint32_t size, Hough* h) {
    if (size <= 1) return ZO_HOUGH_INVALID_ARGUMENT;
    if (size > 32768) return ZO_HOUGH_UNSUPPORTED;
    h->size = size;
    h->even_size = (size % 2 == 0) ? size : size - 1;
    h->cos_table.resize(size);
    h->sin_table.resize(size);
    const double scale = (double)(1 << 16);
    const double sqrt_2 = std::sqrt(2.0);
    for (uint32_t t = 0; t < size; ++t) {
        const double theta = (double)t * M_PI / (double)h->even_size;
        h->cos_table[t] = (int32_t)std::trunc(scale * std::cos(theta) / sqrt_2);
        h->sin_table[t] = (int32_t)std::trunc(scale * std::sin(theta) / sqrt_2);
    }
    return ZO_HOUGH_OK;
}

struct Line { float angle, radius; uint32_t score; float p1x, p1y, p2x, p2y; };

// :232-257
void clip_line(float rect_l, float rect_t, float rect_r, float rect_b, float& p1x, float& p1y, float& p2x, float& p2y) {
    float t0 = 0.0f;
    float t1 = 1.0f;
    const float dx = p2x - p1x;
    const float dy = p2y - p1y;
    const float p[4] = {-dx, dx, -dy, dy};
    const float q[4] = {p1x - rect_l, rect_r - p1x, p1y - rect_t, rect_b - p1y};
    for (int i = 0; i < 4; ++i) {
        if (p[i] == 0) {
            if (q[i] < 0) return;
        } else {
            const float r = q[i] / p[i];
            if (p[i] < 0) {
                if (r > t1) return;
                if (r > t0) t0 = r;
            } else {
                if (r < t0) return;
                if (r < t1) t1 = r;
            }
        }
    }
    if (t0 > t1) return;
    const float old_x = p1x, old_y = p1y;
    p1x = old_x + t0 * dx;
    p1y = old_y + t0 * dy;
    p2x = old_x + t1 * dx;
    p2y = old_y + t1 * dy;
}

// :207-212
void get_line_properties(const Hough& h, float theta_idx, float rho_idx, float* angle, float* radius) {
    const float center_val = (float)(h.size - 1) / 2.0f;
    *angle = 180.0f * (theta_idx - center_val) / (float)h.even_size;
    *radius = (rho_idx - center_val) * std::sqrt(2.0f);
}

// :214-229
Line create_line(const Hough& h, float angle, float radius, uint32_t score) {
    const float center = (float)(h.size - 1) / 2.0f;
    const float theta_rad = (angle + 90.0f) * (float)M_PI / 180.0f;
    const float cos_t = cosf(theta_rad);
    const float sin_t = sinf(theta_rad);
    const float pcx = radius * cos_t, pcy = radius * sin_t;
    const float dirx = -sin_t, diry = cos_t;
    const float huge = (float)h.size * 2.0f;
    Line line;
    line.p1x = center + pcx + dirx * huge;
    line.p1y = center + pcy + diry * huge;
    line.p2x = center + pcx - dirx * huge;
    line.p2y = center + pcy - diry * huge;
    clip_line(0.0f, 0.0f, (float)h.size, (float)h.size, line.p1x, line.p1y, line.p2x, line.p2y);
    line.angle = angle;
    line.radius = radius;
    line.score = score;
    return line;
}

}  // namespace
}  // namespace zo

using namespace zo;

extern "C" {

int zo_hough_tables(uint32_t size, int32_t* cos_table, int32_t* sin_table) {
    Hough h;
    const int rc = hough_init(size, &h);
    if (rc) return rc;
    std::copy(h.cos_table.begin(), h.cos_table.end(), cos_table);
    std::copy(h.sin_table.begin(), h.sin_table.end(), sin_table);
    return ZO_HOUGH_OK;
}

// :75-139
int zo_hough_compute(uint32_t size, const zo_image* edges_, uint32_t l, uint32_t t, uint32_t r, uint32_t b, zo_image* accumulator_) {
    Hough h;
    int rc = hough_init(size, &h);
    if (rc) return rc;
    const uint32_t box_w = l >= r ? 0 : r - l, box_h = t >= b ? 0 : b - t;
    if (box_w != h.size || box_h != h.size) return ZO_HOUGH_DIMENSION_MISMATCH;
    if (accumulator_->rows != h.size || accumulator_->cols != h.size) return ZO_HOUGH_DIMENSION_MISMATCH;
    const Img<const uint8_t> edges(edges_);
    const Img<uint32_t> accumulator(accumulator_);
    // :79 box.intersect(edges.getRectangle()) orelse return
    const uint32_t area_l = std::max(l, 0u), area_t = std::max(t, 0u);
    const uint32_t area_r = std::min(r, edges.cols), area_b = std::min(b, edges.rows);
    if (area_l >= area_r || area_t >= area_b) return ZO_HOUGH_OK;

    const int32_t size_minus_one = (int32_t)(h.size - 1);
    const int32_t box_t = (int32_t)t;
    const int32_t box_l = (int32_t)l;
    const int32_t offset = (int32_t)std::round((double)(1 << 16) * (double)h.even_size / 4.0);
    std::vector<int32_t> y_cache(h.size);
    for (uint32_t row = area_t; row < area_b; ++row) {
        const int32_t y_val = 2 * ((int32_t)row - box_t) - size_minus_one;
        for (uint32_t k = 0; k < h.size; ++k) y_cache[k] = y_val * h.sin_table[k];
        for (uint32_t c = area_l; c < area_r; ++c) {
            if (edges.at(row, c) == 0) continue;
            const int32_t x_val = 2 * ((int32_t)c - box_l) - size_minus_one;
            for (uint32_t k = 0; k < h.size; ++k) {
                const int32_t rho = x_val * h.cos_table[k] + y_cache[k];
                const int32_t rr = ((rho >> 1) + (offset << 1)) >> 16;
                if (rr >= 0 && (uint32_t)rr < h.size) accumulator.at((size_t)rr, k) += 1;
            }
        }
    }
    return ZO_HOUGH_OK;
}

// :142-204
int zo_hough_find_lines(uint32_t size, const zo_image* accumulator_, uint32_t threshold, float angle_nms_thresh, float radius_nms_thresh,
                        zo_hough_line* out, uint32_t cap, uint32_t* n) {
    Hough h;
    int rc = hough_init(size, &h);
    if (rc) return rc;
    *n = 0;
    const Img<const uint32_t> accumulator(accumulator_);
    if (accumulator.rows < 3 || accumulator.cols < 3) return ZO_HOUGH_OK;
    std::vector<Line> lines;
    for (size_t r = 1; r < accumulator.rows - 1; ++r) {
        for (size_t c = 1; c < accumulator.cols - 1; ++c) {
            const uint32_t votes = accumulator.at(r, c);
            if (votes < threshold) continue;
            bool is_local_max = true;
            for (size_t nr = r - 1; nr < r + 2 && is_local_max; ++nr) {
                for (size_t nc = c - 1; nc < c + 2; ++nc) {
                    if (nr == r && nc == c) continue;
                    if (accumulator.at(nr, nc) > votes) {
                        is_local_max = false;
                        break;
                    }
                }
            }
            if (is_local_max) {
                float angle, radius;
                get_line_properties(h, (float)c, (float)r, &angle, &radius);
                lines.push_back(create_line(h, angle, radius, votes));
            }
        }
    }
    std::stable_sort(lines.begin(), lines.end(), [](const Line& a, const Line& b) { return a.score > b.score; });
    std::vector<Line> final_lines;
    for (const Line& candidate : lines) {
        bool too_close = false;
        for (const Line& existing : final_lines) {
            const float da = std::fabs(existing.angle - candidate.angle);
            const float dr = std::fabs(existing.radius - candidate.radius);
            if ((da < angle_nms_thresh && dr < radius_nms_thresh) ||
                ((180.0f - da) < angle_nms_thresh && std::fabs(existing.radius + candidate.radius) < radius_nms_thresh)) {
                too_close = true;
                break;
            }
        }
        if (!too_close) final_lines.push_back(candidate);
    }
    *n = (uint32_t)final_lines.size();
    for (uint32_t i = 0; i < std::min(*n, cap); ++i) {
        const Line& L = final_lines[i];
        out[i] = zo_hough_line{L.angle, L.radius, L.score, L.p1x, L.p1y, L.p2x, L.p2y};
    }
    return ZO_HOUGH_OK;
}

}  // extern "C"
