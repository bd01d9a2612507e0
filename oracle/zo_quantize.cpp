// zo_quantize.cpp -- CPU oracle of colour quantization and dithering (image/quantize.zig, image/dither.zig).  TEST INFRASTRUCTURE ONLY
// (see zignal_oracle.h).  Restates the reference line by line on one thread: medianCut with its first-touch colour list and its box
// loop, std.sort.heap, ColorLookupTable.init (the 16-wide SIMD blocks and the scalar tail), buildPalette and the fixed palettes, and
// dither.apply (the SIMD and scalar ordered paths, and both branches of each error-diffusion loop).
//
// std.sort.heap: this image has no Zig toolchain or standard library, so heap_sort below follows the published lib/std/sort.zig of the
// Zig version the reference pins (build.zig.zon: minimum_zig_version 0.17.0-dev): `heap` calls `heapContext(0, items.len, ctx)`, which
// builds the heap with `i = a + (b - a) / 2; while (i > a) { i -= 1; siftDown(a, i, b, ctx); }` and pops with `i = b; while (i > a)
// { i -= 1; ctx.swap(a, i); siftDown(a, a, i, ctx); }`; `siftDown(a, target, b, ctx)` computes `child = (cur - a) * 2 + a + 1`, breaks
// when `!(child < b)`, moves to `child + 1` when `next_child < b and lessThan(child, next_child)`, breaks when `lessThan(child, cur)`,
// and otherwise swaps and descends.  It is unstable.
//
// Two deviations, as in the library (DESIGN.md §7): a LUT index >= palette.len reads a zero-padded 256-entry palette, and Atkinson on a
// 1-row image takes the bounds-checked branch (the reference's `rows - 2` underflows in usize at dither.zig:271).
//
// Only Rgb(u8) images come in here; the binding (tests/quantize_oracle.py) converts other formats with the main oracle's convertColor
// first, as medianCut and the index lookup do per pixel.  Built on its own into oracle/libzo_quantize.so (Makefile).
#include <cstring>
#include <vector>

#include "zo_common.h"

extern "C" {
enum { ZO_Q_OK = 0, ZO_Q_INVALID_ARGUMENT = 5, ZO_Q_NO_PALETTE_COLORS = 28 };
int zo_median_cut(const zo_image* img, uint16_t max_colors, uint8_t* palette, uint32_t cap, uint32_t* n);
int zo_build_palette(const zo_image* img, int mode, uint16_t max_colors, uint8_t* palette, uint32_t* n);
int zo_color_lut(const uint8_t* palette, uint32_t n, uint8_t* lut);
int zo_dither(zo_image* img, const uint8_t* palette, uint32_t n, const uint8_t* lut, int mode);
int zo_palette_lookup(const zo_image* img, const uint8_t* lut, zo_image* dst);
void zo_heap_sort_u8(uint8_t* items, uint32_t n);
}

namespace zo {
namespace {

struct Rgb { uint8_t r, g, b; };
static_assert(sizeof(Rgb) == 3, "Rgb(u8) is 3 packed bytes");
constexpr int kBits = 5;   // color_quantize_bits

// ---- quantize.zig -------------------------------------------------------------------------------------------------------------------

struct ColorCount { uint8_t r, g, b; uint32_t count; };   // :22-27

struct ColorBox {   // :30-59
    ColorCount* colors;
    size_t len;
    uint8_t r_min, r_max, g_min, g_max, b_min, b_max;
    uint32_t population;
    uint32_t volume() const {
        if (r_max < r_min || g_max < g_min || b_max < b_min) return 0;
        const uint32_t r_size = (uint32_t)r_max - (uint32_t)r_min + 1;
        const uint32_t g_size = (uint32_t)g_max - (uint32_t)g_min + 1;
        const uint32_t b_size = (uint32_t)b_max - (uint32_t)b_min + 1;
        return r_size * g_size * b_size;
    }
    uint8_t largestDimension() const {
        const uint8_t r_range = r_max >= r_min ? r_max - r_min : 0;
        const uint8_t g_range = g_max >= g_min ? g_max - g_min : 0;
        const uint8_t b_range = b_max >= b_min ? b_max - b_min : 0;
        if (g_range >= r_range && g_range >= b_range) return 1;   // green
        if (r_range >= b_range) return 0;                        // red
        return 2;                                                // blue
    }
};

// std.sort.heap (see the header comment), generic over the item type and lessThan.
template <typename T, typename Less> void sift_down(size_t a, size_t target, size_t b, T* items, Less lessThan) {
    size_t cur = target;
    for (;;) {
        size_t child = (cur - a) * 2 + a + 1;
        if (!(child < b)) break;
        const size_t next_child = child + 1;
        if (next_child < b && lessThan(items[child], items[next_child])) child = next_child;
        if (lessThan(items[child], items[cur])) break;
        std::swap(items[child], items[cur]);
        cur = child;
    }
}
template <typename T, typename Less> void heap_sort(T* items, size_t len, Less lessThan) {
    const size_t a = 0, b = len;
    size_t i = a + (b - a) / 2;
    while (i > a) {
        i -= 1;
        sift_down(a, i, b, items, lessThan);
    }
    i = b;
    while (i > a) {
        i -= 1;
        std::swap(items[a], items[i]);
        sift_down(a, a, i, items, lessThan);
    }
}

inline void add_pixel(Rgb rgb, std::vector<uint32_t>& counts, std::vector<uint16_t>& touched) {
    const uint8_t r5 = rgb.r >> (8 - kBits), g5 = rgb.g >> (8 - kBits), b5 = rgb.b >> (8 - kBits);
    const uint16_t key = (uint16_t)(((uint16_t)r5 << (2 * kBits)) | ((uint16_t)g5 << kBits) | (uint16_t)b5);
    if (counts[key] == 0) touched.push_back(key);
    counts[key] += 1;
}

ColorBox fresh_box(ColorCount* colors, size_t len) { return ColorBox{colors, len, 255, 0, 255, 0, 255, 0, 0}; }
void grow(ColorBox& box) {
    for (size_t i = 0; i < box.len; ++i) {
        const ColorCount& c = box.colors[i];
        box.r_min = std::min(box.r_min, c.r);
        box.r_max = std::max(box.r_max, c.r);
        box.g_min = std::min(box.g_min, c.g);
        box.g_max = std::max(box.g_max, c.g);
        box.b_min = std::min(box.b_min, c.b);
        box.b_max = std::max(box.b_max, c.b);
        box.population += c.count;
    }
}

// :175-412
int median_cut(Img<Rgb> image, Rgb* palette, size_t palette_len, uint16_t max_colors, size_t* out) {
    std::vector<ColorCount> color_list;
    std::vector<uint16_t> touched_indices;
    touched_indices.reserve(1024);
    std::vector<uint32_t> counts((size_t)1 << (3 * kBits), 0);
    if (image.stride == image.cols) {   // :193-203
        const size_t total = (size_t)image.rows * image.cols;
        for (size_t i = 0; i < total; ++i) add_pixel(image.data[i], counts, touched_indices);
    } else {                            // :204-218
        for (size_t r = 0; r < image.rows; ++r)
            for (size_t c = 0; c < image.cols; ++c) add_pixel(image.at(r, c), counts, touched_indices);
    }
    color_list.reserve(touched_indices.size());   // :220-237
    for (const uint16_t key_u16 : touched_indices) {
        const size_t key = key_u16;
        const uint8_t r5 = (key >> (2 * kBits)) & 0x1F, g5 = (key >> kBits) & 0x1F, b5 = key & 0x1F;
        const uint8_t r8 = (uint8_t)((r5 << (8 - kBits)) | (r5 >> (2 * kBits - 8)));
        const uint8_t g8 = (uint8_t)((g5 << (8 - kBits)) | (g5 >> (2 * kBits - 8)));
        const uint8_t b8 = (uint8_t)((b5 << (8 - kBits)) | (b5 >> (2 * kBits - 8)));
        color_list.push_back({r8, g8, b8, counts[key]});
    }
    const size_t palette_size = std::min(std::min(color_list.size(), (size_t)max_colors), palette_len);   // :239
    if (palette_size == 0) return ZO_Q_NO_PALETTE_COLORS;
    if (color_list.size() == 1) {   // :245-252
        palette[0] = {color_list[0].r, color_list[0].g, color_list[0].b};
        *out = 1;
        return ZO_Q_OK;
    }
    std::vector<ColorBox> boxes;
    ColorBox initial_box = fresh_box(color_list.data(), color_list.size());
    grow(initial_box);
    boxes.push_back(initial_box);
    while (boxes.size() < palette_size) {   // :280-380
        bool have = false;
        size_t largest_idx = 0;
        uint64_t largest_score = 0;
        for (size_t i = 0; i < boxes.size(); ++i) {
            const ColorBox& box = boxes[i];
            if (box.len <= 1) continue;
            if (box.r_max <= box.r_min && box.g_max <= box.g_min && box.b_max <= box.b_min) continue;
            const uint64_t score = (uint64_t)box.volume() * (uint64_t)box.population;
            if (score > largest_score) {
                largest_score = score;
                largest_idx = i;
                have = true;
            }
        }
        if (!have) break;
        ColorBox box_to_split = boxes[largest_idx];
        boxes.erase(boxes.begin() + (long)largest_idx);   // orderedRemove
        const uint8_t dim = box_to_split.largestDimension();
        heap_sort(box_to_split.colors, box_to_split.len, [dim](const ColorCount& a, const ColorCount& b) {
            return dim == 0 ? a.r < b.r : (dim == 1 ? a.g < b.g : a.b < b.b);
        });
        uint64_t total_weight = 0;
        for (size_t i = 0; i < box_to_split.len; ++i) total_weight += box_to_split.colors[i].count;
        const uint64_t half_weight = total_weight / 2;
        uint64_t accumulated_weight = 0;
        size_t cut_point = 0;
        for (size_t i = 0; i < box_to_split.len; ++i) {
            accumulated_weight += box_to_split.colors[i].count;
            if (accumulated_weight >= half_weight) {
                cut_point = std::max<size_t>(1, std::min(i + 1, box_to_split.len - 1));
                break;
            }
        }
        ColorBox box1 = fresh_box(box_to_split.colors, cut_point);
        ColorBox box2 = fresh_box(box_to_split.colors + cut_point, box_to_split.len - cut_point);
        grow(box1);
        grow(box2);
        if (box1.len > 0 && box1.r_max >= box1.r_min) boxes.push_back(box1);
        if (box2.len > 0 && box2.r_max >= box2.r_min) boxes.push_back(box2);
    }
    const size_t actual_size = std::min(boxes.size(), palette_len);   // :382-411
    for (size_t i = 0; i < actual_size; ++i) {
        const ColorBox& box = boxes[i];
        uint64_t r_sum = 0, g_sum = 0, b_sum = 0, weight_sum = 0;
        for (size_t k = 0; k < box.len; ++k) {
            const ColorCount& c = box.colors[k];
            r_sum += (uint64_t)c.r * (uint64_t)c.count;
            g_sum += (uint64_t)c.g * (uint64_t)c.count;
            b_sum += (uint64_t)c.b * (uint64_t)c.count;
            weight_sum += c.count;
        }
        if (weight_sum > 0) {
            palette[i] = {(uint8_t)(r_sum / weight_sum), (uint8_t)(g_sum / weight_sum), (uint8_t)(b_sum / weight_sum)};
        } else {
            palette[i] = {(uint8_t)((box.r_min + box.r_max) / 2), (uint8_t)((box.g_min + box.g_max) / 2), (uint8_t)((box.b_min + box.b_max) / 2)};
        }
    }
    *out = actual_size;
    return ZO_Q_OK;
}

// :414-473
void fixed6x7x6Palette(Rgb* palette) {
    size_t idx = 0;
    for (int r = 0; r < 6; ++r)
        for (int g = 0; g < 7; ++g)
            for (int b = 0; b < 6; ++b) palette[idx++] = {(uint8_t)((r * 255 + 2) / 5), (uint8_t)((g * 255 + 3) / 6), (uint8_t)((b * 255 + 2) / 5)};
}
void web216Palette(Rgb* palette) {
    size_t idx = 0;
    for (int r = 0; r < 6; ++r)
        for (int g = 0; g < 6; ++g)
            for (int b = 0; b < 6; ++b) palette[idx++] = {(uint8_t)(r * 51), (uint8_t)(g * 51), (uint8_t)(b * 51)};
}
const Rgb vga16_palette[16] = {{0, 0, 0},     {128, 0, 0},   {0, 128, 0},   {128, 128, 0}, {0, 0, 128},   {128, 0, 128},
                               {0, 128, 128}, {192, 192, 192}, {128, 128, 128}, {255, 0, 0}, {0, 255, 0},   {255, 255, 0},
                               {0, 0, 255},   {255, 0, 255}, {0, 255, 255}, {255, 255, 255}};

// :97-159 findNearestColorSIMD: 16-wide blocks reduced with @reduce(.Min), then the scalar tail.
uint8_t find_nearest(size_t len, const int32_t* pal_r, const int32_t* pal_g, const int32_t* pal_b, Rgb target) {
    constexpr size_t VecWidth = 16;
    const int32_t tr = target.r, tg = target.g, tb = target.b;
    uint32_t best_score = 0xffffffffu;
    size_t i = 0;
    while (i + VecWidth <= len) {
        uint32_t min_vec_score = 0xffffffffu;
        for (size_t k = 0; k < VecWidth; ++k) {
            const int32_t dr = pal_r[i + k] - tr, dg = pal_g[i + k] - tg, db = pal_b[i + k] - tb;
            const int32_t dist = dr * dr + dg * dg + db * db;
            const uint32_t score = ((uint32_t)dist << 8) | (uint32_t)(int32_t)(k + i);
            min_vec_score = std::min(min_vec_score, score);
        }
        if (min_vec_score < best_score) best_score = min_vec_score;
        i += VecWidth;
    }
    while (i < len) {
        const int32_t dr = pal_r[i] - tr, dg = pal_g[i] - tg, db = pal_b[i] - tb;
        const int32_t dist = dr * dr + dg * dg + db * db;
        const uint32_t score = ((uint32_t)dist << 8) | (uint32_t)i;
        if (score < best_score) best_score = score;
        i += 1;
    }
    return (uint8_t)(best_score & 0xFF);
}

// :66-94 ColorLookupTable.init
void lut_init(const Rgb* palette, size_t len, uint8_t* table) {
    int32_t pal_r[256] = {}, pal_g[256] = {}, pal_b[256] = {};
    for (size_t i = 0; i < len; ++i) {
        pal_r[i] = palette[i].r;
        pal_g[i] = palette[i].g;
        pal_b[i] = palette[i].b;
    }
    const size_t lut_size = (size_t)1 << kBits;
    for (size_t r = 0; r < lut_size; ++r)
        for (size_t g = 0; g < lut_size; ++g)
            for (size_t b = 0; b < lut_size; ++b) {
                const Rgb rgb = {(uint8_t)(r << (8 - kBits) | (r >> (2 * kBits - 8))), (uint8_t)(g << (8 - kBits) | (g >> (2 * kBits - 8))),
                                 (uint8_t)(b << (8 - kBits) | (b >> (2 * kBits - 8)))};
                table[(r << 10) | (g << 5) | b] = find_nearest(len, pal_r, pal_g, pal_b, rgb);
            }
}

// :163-168
inline uint8_t lut_lookup(const uint8_t* table, Rgb rgb) {
    const uint8_t r5 = rgb.r >> (8 - kBits), g5 = rgb.g >> (8 - kBits), b5 = rgb.b >> (8 - kBits);
    return table[((size_t)r5 << 10) | ((size_t)g5 << 5) | b5];
}

// ---- dither.zig ---------------------------------------------------------------------------------------------------------------------

enum Mode { NONE = 0, FLOYD_STEINBERG = 1, ATKINSON = 2, ORDERED = 3, AUTO = 4 };

struct DitherEntry { int dx, dy, weight, divisor_shift; };
const DitherEntry floyd_steinberg_config[4] = {{1, 0, 7, 4}, {-1, 1, 3, 4}, {0, 1, 5, 4}, {1, 1, 1, 4}};
const DitherEntry atkinson_config[6] = {{1, 0, 1, 3}, {2, 0, 1, 3}, {-1, 1, 1, 3}, {0, 1, 1, 3}, {1, 1, 1, 3}, {0, 2, 1, 3}};

const int32_t bayer8x8[8][8] = {
    {0, 32, 8, 40, 2, 34, 10, 42},   {48, 16, 56, 24, 50, 18, 58, 26}, {12, 44, 4, 36, 14, 46, 6, 38}, {60, 28, 52, 20, 62, 30, 54, 22},
    {3, 35, 11, 43, 1, 33, 9, 41},   {51, 19, 59, 27, 49, 17, 57, 25}, {15, 47, 7, 39, 13, 45, 5, 37}, {63, 31, 55, 23, 61, 29, 53, 21},
};

inline int32_t divTruncPow2(int32_t value, int shift) {   // :97-104
    if (shift == 0) return value;
    if (value >= 0) return value >> shift;
    const int32_t d = (int32_t)1 << shift;
    return (value + d - 1) >> shift;
}
inline uint8_t clampToU8(int32_t value) {   // :106-110
    if (value < 0) return 0;
    if (value > 255) return 255;
    return (uint8_t)value;
}
inline uint8_t meta_clamp_u8(int32_t v) { return clampToU8(v); }

// :113-196
void applyOrdered(Img<Rgb> img, const Rgb* pal, const uint8_t* table) {
    const size_t rows = img.rows, cols = img.cols, stride = img.stride;
    for (size_t r = 0; r < rows; ++r) {
        Rgb* row_slice = img.data + r * stride;
        const int32_t* bayer_row = bayer8x8[r & 7];
        int32_t offsets[8];
        for (int i = 0; i < 8; ++i) offsets[i] = (bayer_row[i] - 32) >> 1;
        size_t c = 0;
        // can_simd (@sizeOf(Rgb) == 3): 24 lanes of i16 per 8 pixels
        int16_t offset_arr[24];
        for (int i = 0; i < 8; ++i) offset_arr[i * 3] = offset_arr[i * 3 + 1] = offset_arr[i * 3 + 2] = (int16_t)offsets[i];
        while (cols >= 8 && c <= cols - 8) {
            const uint8_t* ptr = (const uint8_t*)row_slice + c * 3;
            uint8_t q_arr[24];
            for (int k = 0; k < 24; ++k) {
                const int16_t v = (int16_t)((int16_t)ptr[k] + offset_arr[k]);
                const int16_t clamped = std::min<int16_t>(std::max<int16_t>(v, 0), 255);
                q_arr[k] = (uint8_t)clamped >> (8 - kBits);
            }
            for (int k = 0; k < 8; ++k) {
                const uint8_t idx = table[((size_t)q_arr[k * 3] << 10) | ((size_t)q_arr[k * 3 + 1] << 5) | q_arr[k * 3 + 2]];
                row_slice[c + k] = pal[idx];
            }
            c += 8;
        }
        while (c < cols) {   // the scalar tail (:184-194); the non-SIMD 8-wide path computes the same per pixel
            const Rgb pixel = row_slice[c];
            const int32_t offset = offsets[c & 7];
            const uint8_t r5 = meta_clamp_u8((int32_t)pixel.r + offset) >> (8 - kBits);
            const uint8_t g5 = meta_clamp_u8((int32_t)pixel.g + offset) >> (8 - kBits);
            const uint8_t b5 = meta_clamp_u8((int32_t)pixel.b + offset) >> (8 - kBits);
            const uint8_t idx = table[((size_t)r5 << 10) | ((size_t)g5 << 5) | b5];
            row_slice[c] = pal[idx];
            c += 1;
        }
    }
}

inline void updatePixel(Rgb* ptr, int16_t r_err, int16_t g_err, int16_t b_err, int32_t weight, int shift) {   // :223-229
    ptr->r = clampToU8((int32_t)ptr->r + divTruncPow2((int32_t)r_err * weight, shift));
    ptr->g = clampToU8((int32_t)ptr->g + divTruncPow2((int32_t)g_err * weight, shift));
    ptr->b = clampToU8((int32_t)ptr->b + divTruncPow2((int32_t)b_err * weight, shift));
}

// the bounds-checked branch (:255-262 / :293-300)
inline void distribute(Img<Rgb> img, size_t r, size_t c, const DitherEntry* dists, int n_dists, int16_t re, int16_t ge, int16_t be) {
    const int64_t rows = img.rows, cols = img.cols;
    for (int k = 0; k < n_dists; ++k) {
        const DitherEntry& dist = dists[k];
        const int64_t nc = (int64_t)c + dist.dx, nr = (int64_t)r + dist.dy;
        if (nr >= 0 && nr < rows && nc >= 0 && nc < cols)
            updatePixel(&img.data[(size_t)nr * img.stride + (size_t)nc], re, ge, be, dist.weight, dist.divisor_shift);
    }
}

// :208-331
void applyErrorDiffusion(Img<Rgb> img, const Rgb* pal, const uint8_t* table, int mode) {
    const size_t rows = img.rows, cols = img.cols, stride = img.stride;
    if (mode == FLOYD_STEINBERG) {
        for (size_t r = 0; r < rows; ++r) {
            const size_t row_offset = r * stride;
            Rgb* row_slice = img.data + row_offset;
            const bool is_safe_row = r < rows - 1;
            for (size_t c = 0; c < cols; ++c) {
                const Rgb current = row_slice[c];
                const Rgb quantized = pal[lut_lookup(table, current)];
                row_slice[c] = quantized;
                const int16_t r_err = (int16_t)current.r - (int16_t)quantized.r;
                const int16_t g_err = (int16_t)current.g - (int16_t)quantized.g;
                const int16_t b_err = (int16_t)current.b - (int16_t)quantized.b;
                if (is_safe_row && c > 0 && c < cols - 1) {
                    const size_t next_row_offset = (r + 1) * stride;
                    updatePixel(&img.data[row_offset + c + 1], r_err, g_err, b_err, 7, 4);
                    updatePixel(&img.data[next_row_offset + c - 1], r_err, g_err, b_err, 3, 4);
                    updatePixel(&img.data[next_row_offset + c], r_err, g_err, b_err, 5, 4);
                    updatePixel(&img.data[next_row_offset + c + 1], r_err, g_err, b_err, 1, 4);
                } else {
                    distribute(img, r, c, floyd_steinberg_config, 4, r_err, g_err, b_err);
                }
            }
        }
    } else {   // ATKINSON
        for (size_t r = 0; r < rows; ++r) {
            const size_t row_offset = r * stride;
            Rgb* row_slice = img.data + row_offset;
            const bool is_safe_row = rows >= 2 && r < rows - 2;   // deviation 2: rows == 1 takes the bounds-checked branch
            for (size_t c = 0; c < cols; ++c) {
                const Rgb current = row_slice[c];
                const Rgb quantized = pal[lut_lookup(table, current)];
                row_slice[c] = quantized;
                const int16_t r_err = (int16_t)current.r - (int16_t)quantized.r;
                const int16_t g_err = (int16_t)current.g - (int16_t)quantized.g;
                const int16_t b_err = (int16_t)current.b - (int16_t)quantized.b;
                if (is_safe_row && c > 0 && c < cols - 2) {
                    const size_t r1_offset = (r + 1) * stride, r2_offset = (r + 2) * stride;
                    updatePixel(&img.data[row_offset + c + 1], r_err, g_err, b_err, 1, 3);
                    updatePixel(&img.data[row_offset + c + 2], r_err, g_err, b_err, 1, 3);
                    updatePixel(&img.data[r1_offset + c - 1], r_err, g_err, b_err, 1, 3);
                    updatePixel(&img.data[r1_offset + c], r_err, g_err, b_err, 1, 3);
                    updatePixel(&img.data[r1_offset + c + 1], r_err, g_err, b_err, 1, 3);
                    updatePixel(&img.data[r2_offset + c], r_err, g_err, b_err, 1, 3);
                } else {
                    distribute(img, r, c, atkinson_config, 6, r_err, g_err, b_err);
                }
            }
        }
    }
}

Img<Rgb> rgb_image(const zo_image* img) { return Img<Rgb>(const_cast<zo_image*>(img)); }

// palette as the zero-padded 256-entry table of deviation 1
void padded(const uint8_t* palette, uint32_t n, Rgb* out) {
    std::memset(out, 0, 256 * sizeof(Rgb));
    std::memcpy(out, palette, (size_t)n * 3);
}

}  // namespace
}  // namespace zo

extern "C" int zo_median_cut(const zo_image* img, uint16_t max_colors, uint8_t* palette, uint32_t cap, uint32_t* n) {
    using namespace zo;
    if (!img || !palette || !n) return ZO_Q_INVALID_ARGUMENT;
    size_t out = 0;
    const int rc = median_cut(rgb_image(img), (Rgb*)palette, cap, max_colors, &out);
    if (rc == ZO_Q_OK) *n = (uint32_t)out;
    return rc;
}

// quantize.zig:502-527
extern "C" int zo_build_palette(const zo_image* img, int mode, uint16_t max_colors, uint8_t* palette, uint32_t* n) {
    using namespace zo;
    if (!palette || !n) return ZO_Q_INVALID_ARGUMENT;
    Rgb* pal = (Rgb*)palette;
    switch (mode) {
        case 0: fixed6x7x6Palette(pal); *n = 252; return ZO_Q_OK;
        case 1: std::memcpy(pal, vga16_palette, sizeof(vga16_palette)); *n = 16; return ZO_Q_OK;
        case 2: web216Palette(pal); *n = 216; return ZO_Q_OK;
        case 3: {
            if (!img) return ZO_Q_INVALID_ARGUMENT;
            size_t out = 0;
            if (median_cut(rgb_image(img), pal, 256, max_colors, &out) != ZO_Q_OK) {
                fixed6x7x6Palette(pal);
                out = 252;
            }
            *n = (uint32_t)out;
            return ZO_Q_OK;
        }
    }
    return ZO_Q_INVALID_ARGUMENT;
}

extern "C" int zo_color_lut(const uint8_t* palette, uint32_t n, uint8_t* lut) {
    using namespace zo;
    if (!palette || !lut || n == 0 || n > 256) return ZO_Q_INVALID_ARGUMENT;
    lut_init((const Rgb*)palette, n, lut);
    return ZO_Q_OK;
}

// dither.zig:34-41
extern "C" int zo_dither(zo_image* img, const uint8_t* palette, uint32_t n, const uint8_t* lut, int mode) {
    using namespace zo;
    if (!img || !palette || !lut || n == 0 || n > 256 || mode < NONE || mode > AUTO) return ZO_Q_INVALID_ARGUMENT;
    Rgb pal[256];
    padded(palette, n, pal);
    switch (mode) {
        case FLOYD_STEINBERG: case ATKINSON: applyErrorDiffusion(rgb_image(img), pal, lut, mode); break;
        case ORDERED: applyOrdered(rgb_image(img), pal, lut); break;
        default: break;   // .none, .auto
    }
    return ZO_Q_OK;
}

// ColorLookupTable.lookup per pixel of an Rgb(u8) image into a u8 image of the same shape
extern "C" int zo_palette_lookup(const zo_image* img, const uint8_t* lut, zo_image* dst) {
    using namespace zo;
    if (!img || !lut || !dst || img->rows != dst->rows || img->cols != dst->cols) return ZO_Q_INVALID_ARGUMENT;
    const Img<Rgb> src = rgb_image(img);
    const Img<uint8_t> out(dst);
    for (size_t r = 0; r < src.rows; ++r)
        for (size_t c = 0; c < src.cols; ++c) out.at(r, c) = lut_lookup(lut, src.at(r, c));
    return ZO_Q_OK;
}

// std.sort.heap on bytes with `<`, for the host tests' check of the sort against an independent restatement.
extern "C" void zo_heap_sort_u8(uint8_t* items, uint32_t n) {
    zo::heap_sort(items, n, [](uint8_t a, uint8_t b) { return a < b; });
}
