// zo_shen_castan.cpp -- CPU oracle of Image.shenCastan (TEST INFRASTRUCTURE ONLY, see zignal_oracle.h).
// A literal restatement of image.zig:1015-1027 -> image/edges.zig:83-198 with the options of image/ShenCastan.zig, stage by stage in the
// reference's order, every f32 operation rounded on its own (-ffp-contract=off).  The summed-area tables come from the main oracle's
// zo_integral_plane (integral.zig:41-78).  Built as a library of its own by the Makefile and bound in tests/shen_castan_oracle.py.
#include <cstdint>
#include <cstring>
#include <vector>

#include "zo_common.h"

namespace {

enum { ZO_ERR_INVALID_B_PARAMETER = 24 /* ShenCastan.zig:40 */, ZO_ERR_WINDOW_SIZE_MUST_BE_ODD = 25 /* :41 */,
       ZO_ERR_WINDOW_SIZE_TOO_SMALL = 26 /* :42 */ };

// edges.zig:283-306 isefFilter1D over `n` elements `stride` apart
void isef_1d(float* data, size_t n, size_t stride, float b, std::vector<float>& temp) {
    if (n == 0) return;
    const float a = 1.0f - b;
    temp[0] = b * data[0];
    for (size_t i = 1; i < n; ++i) temp[i] = b * data[i * stride] + a * temp[i - 1];
    data[(n - 1) * stride] = temp[n - 1];
    if (n > 1) {
        size_t i = n - 2;
        while (true) {
            data[i * stride] = b * temp[i] + a * data[(i + 1) * stride];
            if (i == 0) break;
            i -= 1;
        }
    }
}

// edges.zig:356-414 findZeroCrossings
void zero_crossings(const std::vector<uint8_t>& bli, std::vector<uint8_t>& edges, size_t rows, size_t cols, bool use_forward) {
    std::fill(edges.begin(), edges.end(), 0);
    auto at = [&](size_t r, size_t c) { return bli[r * cols + c]; };
    if (use_forward) {
        for (size_t r = 0; r < rows; ++r)
            for (size_t c = 0; c < cols; ++c) {
                const uint8_t center = at(r, c);
                bool mark = false;
                if (!mark && c + 1 < cols) mark = center != at(r, c + 1);                        // East
                if (!mark && r + 1 < rows) mark = center != at(r + 1, c);                        // South
                if (!mark && r + 1 < rows && c + 1 < cols) mark = center != at(r + 1, c + 1);   // South-East
                if (!mark && r + 1 < rows && c > 0) mark = center != at(r + 1, c - 1);           // South-West
                if (mark) edges[r * cols + c] = 255;
            }
    } else if (rows >= 3 && cols >= 3) {
        for (size_t r = 1; r < rows - 1; ++r)
            for (size_t c = 1; c < cols - 1; ++c) {
                const uint8_t center = at(r, c);
                if (center != at(r, c - 1) || center != at(r, c + 1) || center != at(r - 1, c) || center != at(r + 1, c))
                    edges[r * cols + c] = 255;
            }
    } else {                                                                                      // :400-411
        for (size_t r = 0; r < rows; ++r)
            for (size_t c = 0; c < cols; ++c) {
                const uint8_t center = at(r, c);
                bool mark = false;
                if (!mark && c > 0) mark = center != at(r, c - 1);
                if (!mark && c + 1 < cols) mark = center != at(r, c + 1);
                if (!mark && r > 0) mark = center != at(r - 1, c);
                if (!mark && r + 1 < rows) mark = center != at(r + 1, c);
                if (mark) edges[r * cols + c] = 255;
            }
    }
}

// integral.zig:85-90 Integral.sum, reached through computeAdaptiveGradients' boxSum(img, r1, r2, c1, c2) (edges.zig:462-466)
float box_sum(const std::vector<float>& sat, size_t cols, size_t r1, size_t r2, size_t c1, size_t c2) {
    return sat[r2 * cols + c2] - (c1 > 0 ? sat[r2 * cols + (c1 - 1)] : 0.0f) - (r1 > 0 ? sat[(r1 - 1) * cols + c2] : 0.0f) +
           ((r1 > 0 && c1 > 0) ? sat[(r1 - 1) * cols + (c1 - 1)] : 0.0f);
}

int integral(const float* plane, size_t rows, size_t cols, std::vector<float>& sat) {
    zo_image im{(void*)plane, (uint32_t)rows, (uint32_t)cols, (uint64_t)cols};
    return zo_integral_plane(&im, ZO_PIX_F32, sat.data());
}

// edges.zig:417-495 computeAdaptiveGradients
int adaptive_gradients(const std::vector<float>& gray, const std::vector<uint8_t>& bli, const std::vector<uint8_t>& edges, size_t rows,
                       size_t cols, uint64_t window_size, std::vector<float>& gradients) {
    const uint64_t half_window = window_size / 2;
    std::fill(gradients.begin(), gradients.end(), 0.0f);
    const size_t n = rows * cols;
    std::vector<float> integral_gray(n), integral_mask(n), integral_gray_masked(n), mask(n), gray_masked(n);
    int rc;
    if ((rc = integral(gray.data(), rows, cols, integral_gray))) return rc;
    for (size_t i = 0; i < n; ++i) mask[i] = (float)bli[i];                                     // Integral(u8): as(f32, v)
    if ((rc = integral(mask.data(), rows, cols, integral_mask))) return rc;
    for (size_t i = 0; i < n; ++i) gray_masked[i] = gray[i] * (float)bli[i];                    // :446-448
    if ((rc = integral(gray_masked.data(), rows, cols, integral_gray_masked))) return rc;
    for (size_t r = 0; r < rows; ++r)
        for (size_t c = 0; c < cols; ++c) {
            if (edges[r * cols + c] == 0) continue;
            const size_t r_start = r > half_window ? r - half_window : 0;
            const size_t r_end = (size_t)std::min<uint64_t>(r + half_window, rows - 1);
            const size_t c_start = c > half_window ? c - half_window : 0;
            const size_t c_end = (size_t)std::min<uint64_t>(c + half_window, cols - 1);
            const float area = (float)((r_end - r_start + 1) * (c_end - c_start + 1));
            const float count1 = box_sum(integral_mask, cols, r_start, r_end, c_start, c_end);
            const float count0 = area - count1;
            if (count0 > 0 && count1 > 0) {
                const float sum1 = box_sum(integral_gray_masked, cols, r_start, r_end, c_start, c_end);
                const float sum_total = box_sum(integral_gray, cols, r_start, r_end, c_start, c_end);
                const float sum0 = sum_total - sum1;
                const float mean0 = sum0 / count0;
                const float mean1 = sum1 / count1;
                gradients[r * cols + c] = std::fabs(mean1 - mean0);
            }
        }
    return ZO_OK;
}

// edges.zig:582-656 nonMaxSuppressEdges
void non_max_suppress(const std::vector<float>& smoothed, const std::vector<float>& gradients, const std::vector<uint8_t>& edges_in,
                      std::vector<uint8_t>& edges_out, size_t rows, size_t cols) {
    std::fill(edges_out.begin(), edges_out.end(), 0);
    const float K = 0.414213562f;
    if (rows < 3 || cols < 3) return;
    for (size_t r = 1; r < rows - 1; ++r)
        for (size_t c = 1; c < cols - 1; ++c) {
            if (edges_in[r * cols + c] == 0) continue;
            const float gx = 0.5f * (smoothed[r * cols + c + 1] - smoothed[r * cols + c - 1]);
            const float gy = 0.5f * (smoothed[(r + 1) * cols + c] - smoothed[(r - 1) * cols + c]);
            const float ax = std::fabs(gx), ay = std::fabs(gy);
            long dr1, dc1, dr2, dc2;
            if (ay <= K * ax) { dr1 = 0; dc1 = -1; dr2 = 0; dc2 = 1; }
            else if (ax <= K * ay) { dr1 = -1; dc1 = 0; dr2 = 1; dc2 = 0; }
            else if (gx * gy > 0) { dr1 = -1; dc1 = 1; dr2 = 1; dc2 = -1; }
            else { dr1 = -1; dc1 = -1; dr2 = 1; dc2 = 1; }
            const float m = gradients[r * cols + c];
            const float n1 = gradients[(size_t)((long)r + dr1) * cols + (size_t)((long)c + dc1)];
            const float n2 = gradients[(size_t)((long)r + dr2) * cols + (size_t)((long)c + dc2)];
            if (m >= n1 && m >= n2) edges_out[r * cols + c] = 255;
        }
}

// edges.zig:499-575 applyHysteresis (breadth-first, 8-connected; a pixel is marked before it is enqueued)
void hysteresis(const std::vector<uint8_t>& edges, const std::vector<float>& gradients, float threshold_low, float threshold_high,
                const zo_image* out, size_t rows, size_t cols) {
    uint8_t* o = (uint8_t*)out->data;
    const size_t stride = (size_t)out->stride;
    for (size_t r = 0; r < rows; ++r) std::memset(o + r * stride, 0, cols);
    std::vector<std::pair<size_t, size_t>> queue;
    queue.reserve(rows * cols);
    for (size_t r = 0; r < rows; ++r)
        for (size_t c = 0; c < cols; ++c)
            if (edges[r * cols + c] > 0 && gradients[r * cols + c] >= threshold_high) {
                o[r * stride + c] = 255;
                queue.emplace_back(r, c);
            }
    for (size_t pop = 0; pop < queue.size(); ++pop) {
        const size_t r = queue[pop].first, c = queue[pop].second;
        const size_t r_start = r > 0 ? r - 1 : 0, r_end = std::min(r + 2, rows);
        const size_t c_start = c > 0 ? c - 1 : 0, c_end = std::min(c + 2, cols);
        for (size_t nr = r_start; nr < r_end; ++nr)
            for (size_t nc = c_start; nc < c_end; ++nc) {
                if (nr == r && nc == c) continue;
                if (o[nr * stride + nc] > 0) continue;
                if (edges[nr * cols + nc] > 0 && gradients[nr * cols + nc] >= threshold_low) {
                    o[nr * stride + nc] = 255;
                    queue.emplace_back(nr, nc);
                }
            }
    }
}

}  // namespace

extern "C" {

// image.zig:1015-1027 / edges.zig:83-198.  t_high / t_low / candidates (may be NULL) receive the thresholds and the number of candidate
// pixels the histogram counted (0: no candidate, the thresholds are left at 0).
int zo_shen_castan(const zo_image* src, zo_image* dst, int pixfmt, float smooth, uint64_t window_size, float high_ratio, float low_rel,
                   int use_hysteresis, int use_nms, float* t_high_out, float* t_low_out, uint64_t* candidates_out) {
    if (pixfmt != ZO_PIX_U8 && pixfmt != ZO_PIX_F32 && pixfmt != ZO_PIX_RGB8 && pixfmt != ZO_PIX_RGBA8) return ZO_ERR_UNSUPPORTED;
    if (src->rows != dst->rows || src->cols != dst->cols) return ZO_ERR_DIMENSION_MISMATCH;   // image.zig:1023
    if (!(smooth > 0 && smooth < 1)) return ZO_ERR_INVALID_B_PARAMETER;                        // ShenCastan.zig:40
    if (window_size % 2 == 0) return ZO_ERR_WINDOW_SIZE_MUST_BE_ODD;                            // :41
    if (window_size < 3) return ZO_ERR_WINDOW_SIZE_TOO_SMALL;                                   // :42
    if (!(high_ratio > 0 && high_ratio < 1)) return ZO_ERR_INVALID_THRESHOLD;                  // :43
    if (!(low_rel > 0 && low_rel < 1)) return ZO_ERR_INVALID_THRESHOLD;                        // :44
    if (t_high_out) *t_high_out = 0;
    if (t_low_out) *t_low_out = 0;
    if (candidates_out) *candidates_out = 0;
    const size_t rows = src->rows, cols = src->cols, n = rows * cols;
    if (n == 0) return ZO_OK;

    std::vector<float> gray(n);                                                                 // :91-100 as(f32, convertColor(u8, px))
    for (size_t r = 0; r < rows; ++r)
        for (size_t c = 0; c < cols; ++c) {
            float v;
            if (pixfmt == ZO_PIX_F32) {                                                          // color.zig:114-118 through f64
                double d = (double)((const float*)src->data)[r * src->stride + c];
                d = zo::zig_max(0.0, zo::zig_min(d, 1.0));   // std.math.clamp: NaN -> 1
                v = (float)(uint8_t)std::round(d * 255.0);
            } else if (pixfmt == ZO_PIX_U8) {
                v = (float)((const uint8_t*)src->data)[r * src->stride + c];
            } else {
                const int ch = pixfmt == ZO_PIX_RGB8 ? 3 : 4;
                const uint8_t* px = (const uint8_t*)src->data + (r * src->stride + c) * ch;
                int y = (13933 * (int)px[0] + 46871 * (int)px[1] + 4732 * (int)px[2] + 32768) >> 16;   // color.zig:1031-1041
                y = y < 0 ? 0 : (y > 255 ? 255 : y);
                v = (float)y;
            }
            gray[r * cols + c] = v;
        }

    std::vector<float> smoothed(gray);                                                          // :104-106 isefFilter2D
    {
        std::vector<float> temp(std::max(rows, cols));
        for (size_t r = 0; r < rows; ++r) isef_1d(smoothed.data() + r * cols, cols, 1, smooth, temp);   // :318-330
        for (size_t c = 0; c < cols; ++c) isef_1d(smoothed.data() + c, rows, cols, smooth, temp);       // :338-349
    }
    std::vector<uint8_t> bli(n);                                                                // :108-122
    for (size_t i = 0; i < n; ++i) {
        const float laplacian = smoothed[i] - gray[i];
        bli[i] = laplacian >= 0 ? 1 : 0;
    }
    std::vector<uint8_t> edges(n);                                                              // :124-128
    zero_crossings(bli, edges, rows, cols, !use_nms);
    std::vector<float> gradients(n);                                                            // :130-133
    int rc = adaptive_gradients(gray, bli, edges, rows, cols, window_size, gradients);
    if (rc) return rc;

    uint64_t hist[256] = {0}, total = 0;                                                        // :139-152
    for (size_t i = 0; i < n; ++i) {
        if (edges[i] == 0) continue;
        float g = gradients[i];
        if (g < 0) g = 0;
        if (g > 255) g = 255;
        hist[(size_t)std::round(g)] += 1;                                                       // @round: half away from zero
        total += 1;
    }
    uint8_t* o = (uint8_t*)dst->data;
    if (total == 0) {                                                                           // :153-161
        for (size_t r = 0; r < rows; ++r) std::memset(o + r * dst->stride, 0, cols);
        return ZO_OK;
    }
    const uint64_t target = (uint64_t)std::floor((float)total * high_ratio);                  // :162
    uint64_t cum = 0;
    size_t idx = 0;
    while (idx < 256 && cum < target) {                                                         // :165-167
        cum += hist[idx];
        idx += 1;
    }
    const float t_high = (float)std::min<size_t>(idx, 255);                                    // :169 (idx is one past the bin that reached the target)
    const float t_low = low_rel * t_high;                                                       // :170
    if (t_high_out) *t_high_out = t_high;
    if (t_low_out) *t_low_out = t_low;
    if (candidates_out) *candidates_out = total;

    std::vector<uint8_t> edges_nms;                                                             // :172-183
    const std::vector<uint8_t>* edges_for_thresh = &edges;
    if (use_nms) {
        edges_nms.resize(n);
        non_max_suppress(smoothed, gradients, edges, edges_nms, rows, cols);
        edges_for_thresh = &edges_nms;
    }
    if (!use_hysteresis) {                                                                      // :185-194
        for (size_t r = 0; r < rows; ++r)
            for (size_t c = 0; c < cols; ++c) {
                const bool is_edge = (*edges_for_thresh)[r * cols + c] > 0 && gradients[r * cols + c] >= t_high;
                o[r * dst->stride + c] = is_edge ? 255 : 0;
            }
        return ZO_OK;
    }
    hysteresis(*edges_for_thresh, gradients, t_low, t_high, dst, rows, cols);                  // :197
    return ZO_OK;
}

}  // extern "C"
