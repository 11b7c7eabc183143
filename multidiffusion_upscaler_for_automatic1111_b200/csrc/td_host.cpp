// Host-side tile bookkeeping of the C-ABI (no GPU needed).
//
// The reference does this arithmetic in Python: `/` is float64 division,
// math.ceil works on that float64, int() truncates toward zero.  C `double`
// reproduces every intermediate bit-for-bit, so the integer results are exact.
//
//   td_split_bboxes     <- tile_utils/utils.py:160-177
//   td_splitable        <- tile_utils/utils.py:151-158
//   td_gaussian_weights <- tile_utils/utils.py:180-194
//   td_grid_init        <- tile_methods/abstractdiffusion.py:172-186
//   td_grid_weights     <- tile_utils/utils.py:167,175 (+ abstractdiffusion.py:182)
//   td_rescale_factor   <- tile_methods/mixtureofdiffusers.py:32
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "td_b200.h"
#include "td_internal.h"

static thread_local char g_err[512] = "";

void td_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" const char* td_last_error(void) { return g_err; }
extern "C" int td_abi_version(void) { return TD_ABI_VERSION; }

namespace {

// cols = math.ceil((w - overlap) / (tile_w - overlap))          utils.py:161
inline int ceil_div_py(int num, int den) { return (int)std::ceil((double)num / (double)den); }

struct Split {
    int cols, rows;
    double dx, dy;
};

// One axis of split_bboxes: tile count (utils.py:161-162) and origin stride (utils.py:163-164).  Requires t != ov.
// NB: overlap > tile is legal when the tile was clamped to the canvas
// (abstractdiffusion.py:176-178): (L-ov)/(t-ov) is then negative/negative.
inline void axis_split(int L, int t, int ov, int* n, double* d) {
    *n = std::max(0, ceil_div_py(L - ov, t - ov));  // Python: range(negative) is empty -> no tiles
    *d = *n > 1 ? (double)(L - t) / (double)(*n - 1) : 0.0;
}

inline int split_counts(int w, int h, int tile_w, int tile_h, int overlap, Split* s) {
    if (w <= 0 || h <= 0 || tile_w <= 0 || tile_h <= 0 || overlap < 0) {
        td_set_error("split_bboxes: non-positive size (w=%d h=%d tile=%dx%d overlap=%d)", w, h, tile_w, tile_h, overlap);
        return TD_ERR_INVALID_ARG;
    }
    if (tile_w == overlap || tile_h == overlap) {  // Python: ZeroDivisionError at utils.py:161-162
        td_set_error("split_bboxes: overlap %d equals the tile size (%dx%d): division by zero", overlap, tile_w, tile_h);
        return TD_ERR_INVALID_ARG;
    }
    if (tile_w > w || tile_h > h) {  // not reachable through init_grid_bbox (tile is clamped first)
        td_set_error("split_bboxes: tile %dx%d larger than canvas %dx%d", tile_w, tile_h, w, h);
        return TD_ERR_INVALID_ARG;
    }
    axis_split(w, tile_w, overlap, &s->cols, &s->dx);
    axis_split(h, tile_h, overlap, &s->rows, &s->dy);
    return TD_OK;
}

// x = min(int(col * dx), w - tile_w)                              utils.py:171
inline int origin(int idx, double d, int limit) { return std::min((int)((double)idx * d), limit); }

}  // namespace

extern "C" int td_split_bboxes(int w, int h, int tile_w, int tile_h, int overlap, int32_t* out_xywh, int cap,
                               int* out_cols, int* out_rows) {
    Split s;
    int st = split_counts(w, h, tile_w, tile_h, overlap, &s);
    if (st != TD_OK) return st;
    if (out_cols) *out_cols = s.cols;
    if (out_rows) *out_rows = s.rows;
    const long long T = (long long)s.cols * s.rows;
    if (out_xywh == nullptr) return (int)T;  // count query
    if (T > cap) {
        td_set_error("split_bboxes: %lld tiles exceed capacity %d", T, cap);
        return TD_ERR_CAPACITY;
    }
    int32_t* o = out_xywh;
    for (int row = 0; row < s.rows; ++row) {
        const int y = origin(row, s.dy, h - tile_h);
        for (int col = 0; col < s.cols; ++col) {
            const int x = origin(col, s.dx, w - tile_w);
            *o++ = x; *o++ = y; *o++ = tile_w; *o++ = tile_h;
        }
    }
    return (int)T;
}

extern "C" int td_splitable(int w, int h, int tile_w, int tile_h, int overlap) {
    w /= 8; h /= 8;  // opt_f, utils.py:152
    const int min_tile = std::min(tile_w, tile_h);
    if (overlap >= min_tile) overlap = min_tile - 4;
    if (tile_w - overlap <= 0 || tile_h - overlap <= 0) {
        td_set_error("splitable: tile %dx%d too small for overlap %d", tile_w, tile_h, overlap);
        return TD_ERR_INVALID_ARG;
    }
    const int cols = ceil_div_py(w - overlap, tile_w - overlap);
    const int rows = ceil_div_py(h - overlap, tile_h - overlap);
    return (cols > 1 || rows > 1) ? 1 : 0;
}

extern "C" int td_gaussian_weights(int tile_w, int tile_h, float* out) {
    if (tile_w <= 0 || tile_h <= 0 || out == nullptr) {
        td_set_error("gaussian_weights: bad args");
        return TD_ERR_INVALID_ARG;
    }
    // f(x, mid) = exp(-(x-mid)*(x-mid) / (tile_w*tile_w) / (2*var)) / sqrt(2*pi*var), var = 0.01
    // evaluated left to right in float64 exactly as utils.py:189 writes it.
    const double var = 0.01;
    const double norm = std::sqrt(2.0 * M_PI * var);
    const double tw2 = (double)(tile_w * tile_w);
    auto f = [&](double x, double mid) { return std::exp(-(x - mid) * (x - mid) / tw2 / (2.0 * var)) / norm; };
    const double xmid = (double)(tile_w - 1) / 2.0;  // utils.py:190
    const double ymid = (double)tile_h / 2.0;        // utils.py:191 (asymmetric on purpose)
    for (int y = 0; y < tile_h; ++y) {
        const double yp = f((double)y, ymid);
        for (int x = 0; x < tile_w; ++x) out[(size_t)y * tile_w + x] = (float)(yp * f((double)x, xmid));  // np.outer -> fp32
    }
    return TD_OK;
}

extern "C" int td_feather_mask(int w, int h, double ratio, float* out) {
    if (w <= 0 || h <= 0 || out == nullptr) {
        td_set_error("feather_mask: bad args");
        return TD_ERR_INVALID_ARG;
    }
    for (size_t i = 0; i < (size_t)w * h; ++i) out[i] = 1.0f;
    // feather_radius = int(min(w//2, h//2) * ratio): float64 product, truncation (utils.py:200)
    const int radius = (int)((double)std::min(w / 2, h / 2) * ratio);
    for (int i = 0; i < h / 2; ++i)
        for (int j = 0; j < w / 2; ++j) {
            const int dist = std::min(i, j);
            if (dist >= radius) continue;
            // (dist / radius) ** 2 in float64, stored into a float32 array (utils.py:208)
            const float wt = (float)std::pow((double)dist / (double)radius, 2.0);
            out[(size_t)i * w + j] = wt;
            out[(size_t)i * w + (w - j - 1)] = wt;
            out[(size_t)(h - i - 1) * w + j] = wt;
            out[(size_t)(h - i - 1) * w + (w - j - 1)] = wt;
        }
    return TD_OK;
}

extern "C" int td_custom_bbox_rect(double x, double y, double w, double h, int canvas_w, int canvas_h, int32_t* out_xywh) {
    if (out_xywh == nullptr || canvas_w <= 0 || canvas_h <= 0) {
        td_set_error("custom_bbox_rect: bad args");
        return TD_ERR_INVALID_ARG;
    }
    if (x > 1.0 || y > 1.0 || w <= 0.0 || h <= 0.0) return 0;   // skipped by the reference (abstractdiffusion.py:207)
    // int(x * W), math.ceil(w * W) on float64 products; then clamps (abstractdiffusion.py:208-215)
    int xi = (int)(x * (double)canvas_w);
    int yi = (int)(y * (double)canvas_h);
    int wi = (int)std::ceil(w * (double)canvas_w);
    int hi = (int)std::ceil(h * (double)canvas_h);
    xi = std::max(0, xi);
    yi = std::max(0, yi);
    wi = std::min(canvas_w - xi, wi);
    hi = std::min(canvas_h - yi, hi);
    out_xywh[0] = xi; out_xywh[1] = yi; out_xywh[2] = wi; out_xywh[3] = hi;
    return 1;
}

// ---------------------------------------------------------------------------------------------------------
// One axis of a tile plan: tile count n and origin stride d.  A bounded axis follows split_bboxes (origins
// min(int(k * d), L - t)).  A periodic axis of length L is tiled as a circle: tile k starts at floor(k * d),
// d = L / n with n = ceil(L / (t - overlap)), so the gap between neighbours -- the last and the first
// included -- is at most ceil(L / n) <= t - overlap, and a tile may run past L, continuing at 0.
// ---------------------------------------------------------------------------------------------------------
namespace {

int linear_axis(int L, int t, int ov, int* n, double* d) {
    if (t == ov) {  // Python: ZeroDivisionError at utils.py:161-162
        td_set_error("grid_init: overlap %d equals the tile size %d: division by zero", ov, t);
        return TD_ERR_INVALID_ARG;
    }
    axis_split(L, t, ov, n, d);
    return TD_OK;
}

int periodic_axis(int L, int t, int ov, int* n, double* d) {
    if (t == L) {
        *n = 1;
        *d = 0.0;
        return TD_OK;
    }
    if (t <= ov) {
        td_set_error("grid_init: overlap %d leaves no stride on a periodic axis with tile %d", ov, t);
        return TD_ERR_INVALID_ARG;
    }
    *n = ceil_div_py(L, t - ov);
    *d = (double)L / (double)*n;
    return TD_OK;
}

int axis(int L, int t, int ov, bool periodic, int* n, double* d) {
    return periodic ? periodic_axis(L, t, ov, n, d) : linear_axis(L, t, ov, n, d);
}

void fill_origins(int n, double d, int L, int t, bool periodic, int32_t* org) {
    for (int k = 0; k < n; ++k) org[k] = periodic ? (int32_t)std::floor((double)k * d) : origin(k, d, L - t);
}

}  // namespace

extern "C" int td_grid_init(td_grid* g, int w, int h, int tile_w, int tile_h, int overlap, int tile_bs, int wrap) {
    if (g == nullptr || tile_bs <= 0 || (wrap & ~(int)(TD_WRAP_X | TD_WRAP_Y)) != 0) {
        td_set_error("grid_init: bad args");
        return TD_ERR_INVALID_ARG;
    }
    if (tile_w <= 0 || tile_h <= 0 || w <= 0 || h <= 0) {
        td_set_error("grid_init: non-positive size");
        return TD_ERR_INVALID_ARG;
    }
    std::memset(g, 0, sizeof(*g));
    g->W = w; g->H = h;
    g->wrap = wrap;
    g->tile_w = std::min(tile_w, w);                                     // abstractdiffusion.py:176
    g->tile_h = std::min(tile_h, h);                                     // :177
    g->overlap = std::max(0, std::min(overlap, std::min(tile_w, tile_h) - 4));  // :178 (unclamped tile args)
    const bool px = (wrap & TD_WRAP_X) != 0, py = (wrap & TD_WRAP_Y) != 0;
    int cols = 0, rows = 0;
    double dx = 0.0, dy = 0.0;
    int st = axis(w, g->tile_w, g->overlap, px, &cols, &dx);           // utils.py:161,163
    if (st != TD_OK) return st;
    st = axis(h, g->tile_h, g->overlap, py, &rows, &dy);               // utils.py:162,164
    if (st != TD_OK) return st;
    if (rows > TD_MAX_GRID_DIM || cols > TD_MAX_GRID_DIM) {
        td_set_error("grid_init: %dx%d tile grid exceeds TD_MAX_GRID_DIM=%d", rows, cols, TD_MAX_GRID_DIM);
        return TD_ERR_UNSUPPORTED;
    }
    g->rows = rows; g->cols = cols;
    fill_origins(rows, dy, h, g->tile_h, py, g->ys);                     // utils.py:169
    fill_origins(cols, dx, w, g->tile_w, px, g->xs);                     // utils.py:171
    g->num_tiles = rows * cols;                                          // :183
    if (g->num_tiles == 0) {  // Python: ZeroDivisionError at :185
        td_set_error("grid_init: the split produced no tiles (w=%d h=%d tile=%dx%d overlap=%d)", w, h, g->tile_w, g->tile_h, g->overlap);
        return TD_ERR_INVALID_ARG;
    }
    g->num_batches = ceil_div_py(g->num_tiles, tile_bs);                 // :184
    g->tile_bs = ceil_div_py(g->num_tiles, g->num_batches);              // :185
    return g->num_tiles;
}

extern "C" int td_grid_weights(const td_grid* g, const float* tile_weights, float* out) {
    if (g == nullptr || out == nullptr) {
        td_set_error("grid_weights: null");
        return TD_ERR_INVALID_ARG;
    }
    const int W = g->W, H = g->H, tw = g->tile_w, th = g->tile_h;
    const bool px = (g->wrap & TD_WRAP_X) != 0, py = (g->wrap & TD_WRAP_Y) != 0;
    for (int c = 0; c < g->cols; ++c)
        if (g->xs[c] < 0 || g->xs[c] >= W || tw > W || (!px && g->xs[c] + tw > W)) {
            td_set_error("grid_weights: tile column %d (x=%d, w=%d) leaves the %d-wide canvas", c, g->xs[c], tw, W);
            return TD_ERR_INVALID_ARG;
        }
    for (int r = 0; r < g->rows; ++r)
        if (g->ys[r] < 0 || g->ys[r] >= H || th > H || (!py && g->ys[r] + th > H)) {
            td_set_error("grid_weights: tile row %d (y=%d, h=%d) leaves the %d-high canvas", r, g->ys[r], th, H);
            return TD_ERR_INVALID_ARG;
        }
    std::fill(out, out + (size_t)W * H, 0.0f);
    for (int r = 0; r < g->rows; ++r)
        for (int c = 0; c < g->cols; ++c) {  // list order: row outer, col inner
            const int x0 = g->xs[c], y0 = g->ys[r];
            for (int v = 0; v < th; ++v) {
                float* o = out + (size_t)((y0 + v) % H) * W;
                for (int u = 0; u < tw; ++u) {
                    const int x = (x0 + u) % W;
                    o[x] = o[x] + (tile_weights ? tile_weights[(size_t)v * tw + u] : 1.0f);
                }
            }
        }
    return TD_OK;
}

// ---------------------------------------------------------------------------------------------------------
// SpotDiffusion step plans: the base plan with every window moved back by a per-call shift (td_b200.h).
// ---------------------------------------------------------------------------------------------------------
namespace {

struct ShiftAxis {
    int lo, hi;  // accepted shifts [lo, hi)
    bool grows;  // bounded axis that gains the window at L - t
};

// One axis of a base plan: origins in [0, L), inside the canvas when bounded, non-decreasing.
bool valid_axis(const int32_t* b, int n, int L, int t, bool periodic) {
    if (n < 1 || n > TD_MAX_GRID_DIM || L <= 0 || t <= 0 || t > L) return false;
    for (int k = 0; k < n; ++k)
        if (b[k] < 0 || b[k] >= L || (!periodic && b[k] + t > L) || (k > 0 && b[k] < b[k - 1])) return false;
    return true;
}

ShiftAxis shift_axis_bounds(const int32_t* b, int n, int L, bool periodic) {
    int gap = periodic ? L + b[0] - b[n - 1] : L;  // n == 1: L
    for (int k = 1; k < n; ++k) gap = std::min(gap, b[k] - b[k - 1]);
    if (periodic) return {0, gap, false};
    if (n >= 2 && gap >= 2) return {1, gap, true};
    return {0, 1, false};
}

int shift_axis(const int32_t* b, int n, int L, int t, bool periodic, const ShiftAxis& ax, int s, int32_t* out) {
    if (periodic) {
        for (int k = 0; k < n; ++k) out[k] = ((b[k] - s) % L + L) % L;
        std::sort(out, out + n);
        return n;
    }
    if (!ax.grows) {
        std::copy(b, b + n, out);
        return n;
    }
    out[0] = 0;
    for (int k = 1; k < n; ++k) out[k] = b[k] - s;
    out[n] = L - t;
    return n + 1;
}

int check_base(const td_grid* g, const char* what) {
    if (g == nullptr || (g->wrap & ~(int)(TD_WRAP_X | TD_WRAP_Y)) != 0 ||
        !valid_axis(g->xs, g->cols, g->W, g->tile_w, (g->wrap & TD_WRAP_X) != 0) ||
        !valid_axis(g->ys, g->rows, g->H, g->tile_h, (g->wrap & TD_WRAP_Y) != 0)) {
        td_set_error("%s: null or malformed base plan", what);
        return TD_ERR_INVALID_ARG;
    }
    return TD_OK;
}

}  // namespace

extern "C" int td_grid_shift_bounds(const td_grid* base, int32_t out[4]) {
    int st = check_base(base, "grid_shift_bounds");
    if (st != TD_OK) return st;
    if (out == nullptr) {
        td_set_error("grid_shift_bounds: null output");
        return TD_ERR_INVALID_ARG;
    }
    const ShiftAxis ax = shift_axis_bounds(base->xs, base->cols, base->W, (base->wrap & TD_WRAP_X) != 0);
    const ShiftAxis ay = shift_axis_bounds(base->ys, base->rows, base->H, (base->wrap & TD_WRAP_Y) != 0);
    out[0] = ax.lo; out[1] = ax.hi; out[2] = ay.lo; out[3] = ay.hi;
    return TD_OK;
}

extern "C" int td_grid_shift(const td_grid* base, int shift_x, int shift_y, int tile_bs, td_grid* out) {
    int st = check_base(base, "grid_shift");
    if (st != TD_OK) return st;
    if (out == nullptr || tile_bs <= 0) {
        td_set_error("grid_shift: null output or tile_bs %d <= 0", tile_bs);
        return TD_ERR_INVALID_ARG;
    }
    const bool px = (base->wrap & TD_WRAP_X) != 0, py = (base->wrap & TD_WRAP_Y) != 0;
    const ShiftAxis ax = shift_axis_bounds(base->xs, base->cols, base->W, px);
    const ShiftAxis ay = shift_axis_bounds(base->ys, base->rows, base->H, py);
    if (shift_x < ax.lo || shift_x >= ax.hi || shift_y < ay.lo || shift_y >= ay.hi) {
        td_set_error("grid_shift: shift (%d, %d) outside [%d, %d) x [%d, %d)", shift_x, shift_y, ax.lo, ax.hi, ay.lo, ay.hi);
        return TD_ERR_INVALID_ARG;
    }
    if (base->cols + (ax.grows ? 1 : 0) > TD_MAX_GRID_DIM || base->rows + (ay.grows ? 1 : 0) > TD_MAX_GRID_DIM) {
        td_set_error("grid_shift: a %dx%d base plan gains a window row / column past TD_MAX_GRID_DIM=%d", base->rows, base->cols,
                     TD_MAX_GRID_DIM);
        return TD_ERR_UNSUPPORTED;
    }
    td_grid g;
    std::memset(&g, 0, sizeof(g));
    g.W = base->W; g.H = base->H;
    g.tile_w = base->tile_w; g.tile_h = base->tile_h;
    g.overlap = base->overlap;
    g.wrap = base->wrap;
    g.cols = shift_axis(base->xs, base->cols, base->W, base->tile_w, px, ax, shift_x, g.xs);
    g.rows = shift_axis(base->ys, base->rows, base->H, base->tile_h, py, ay, shift_y, g.ys);
    g.num_tiles = g.rows * g.cols;
    g.num_batches = ceil_div_py(g.num_tiles, tile_bs);                  // as td_grid_init
    g.tile_bs = ceil_div_py(g.num_tiles, g.num_batches);
    *out = g;
    return g.num_tiles;
}

extern "C" int td_rescale_factor(const float* weights, float* out, int64_t n) {
    if (weights == nullptr || out == nullptr || n < 0) {
        td_set_error("rescale_factor: bad args");
        return TD_ERR_INVALID_ARG;
    }
    for (int64_t i = 0; i < n; ++i) out[i] = 1.0f / weights[i];  // IEEE; inf where uncovered, like torch
    return TD_OK;
}
