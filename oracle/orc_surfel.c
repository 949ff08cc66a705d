/*
 * oracle/orc_surfel.c -- CPU ORACLE (test infrastructure, not product):
 * restatement of the reference's GLSL surfel passes (Core/Shaders) and their
 * host drivers (Core/Model/Model.cpp, ModelProjection.cpp, GlobalProjection.cpp,
 * Shaders/FillIn.cpp, FeedbackBuffer.cpp).  No OpenGL exists in this
 * environment, so these passes are "parity unpinned"; the raster / sampling
 * rules that GL leaves implementation-defined are fixed here in writing
 * (SURVEY.md Appendix A N1-N7, N14; DESIGN.md "parity rules").
 *
 * mat4*vec4 and dot products are evaluated left to right:
 *   ((m0*x + m1*y) + m2*z) + m3.
 */
#include "orc.h"
#include <math.h>
#include <string.h>
#include <stdlib.h>

#define MAX_POINT_SIZE 2047.0f   /* GL_ALIASED_POINT_SIZE_RANGE upper bound on NVIDIA (rule R-PS) */

static inline int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
static inline uint32_t fbits(float f) { union { float f; uint32_t u; } c; c.f = f; return c.u; }

static inline void xform(const float* T, const float* p, float* o)
{
    o[0] = ((T[0] * p[0] + T[1] * p[1]) + T[2] * p[2]) + T[3];
    o[1] = ((T[4] * p[0] + T[5] * p[1]) + T[6] * p[2]) + T[7];
    o[2] = ((T[8] * p[0] + T[9] * p[1]) + T[10] * p[2]) + T[11];
}
static inline void rot(const float* T, const float* n, float* o)
{
    o[0] = (T[0] * n[0] + T[1] * n[1]) + T[2] * n[2];
    o[1] = (T[4] * n[0] + T[5] * n[1]) + T[6] * n[2];
    o[2] = (T[8] * n[0] + T[9] * n[1]) + T[10] * n[2];
}
/* depth-tested key images are built by all threads: min over 64-bit keys is order-free, the winner is the one a sequential loop finds */
static inline void atomic_min_u64(uint64_t* p, uint64_t v)
{
    uint64_t o = __atomic_load_n(p, __ATOMIC_RELAXED);
    while (v < o && !__atomic_compare_exchange_n(p, &o, v, 1, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
}

static inline float dot3(const float* a, const float* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
static inline void normalize3(float* v)
{
    float l = sqrtf(dot3(v, v));
    v[0] /= l; v[1] /= l; v[2] /= l;
}
static inline void cross3(const float* a, const float* b, float* o)
{
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}

/* color_encoding.glsl:19-34; round(x) := floor(x + 0.5) */
static inline float encode_color(const float* c)
{
    int rgb = (int)floorf(c[0] * 255.0f + 0.5f);
    rgb = (rgb << 8) + (int)floorf(c[1] * 255.0f + 0.5f);
    rgb = (rgb << 8) + (int)floorf(c[2] * 255.0f + 0.5f);
    return (float)rgb;
}
static inline void decode_color(float c, float* col)
{
    int ci = (int)c;
    col[0] = (float)((ci >> 16) & 0xFF) / 255.0f;
    col[1] = (float)((ci >> 8) & 0xFF) / 255.0f;
    col[2] = (float)(ci & 0xFF) / 255.0f;
}

/* surfels.glsl:19-34 (cam.z = 1/fx, cam.w = 1/fy) */
static inline float get_radius(float depth, float norm_z, float ifx, float ify)
{
    float meanFocal = ((1.0f / fabsf(ifx)) + (1.0f / fabsf(ify))) / 2.0f;
    const float sqrt2 = 1.41421356237f;
    float radius = (depth / meanFocal) * sqrt2;
    float radius_n = radius / fabsf(norm_z);
    float r2 = 2.0f * radius;
    return r2 < radius_n ? r2 : radius_n;      /* min(a,b): b<a ? b : a, NaN -> 2*radius */
}
/* surfels.glsl:36-46 */
static inline float confidence(float x, float y, float weighting, float cx, float cy)
{
    float px = x - cx, py = y - cy;
    float radialDist = sqrtf(px * px + py * py) / 400.0f;
    return orc_expf((-(radialDist * radialDist) / 0.72f)) * weighting;
}

/* geometry.glsl:22-26 with nearest / clamp-to-edge sampling (N14) */
static inline void get_vertex(const float* depth, int W, int H, int tx, int ty, float x, float y,
                              orc_cam cam, float ifx, float ify, float* v)
{
    float z = depth[clampi(ty, 0, H - 1) * W + clampi(tx, 0, W - 1)];
    v[0] = (x - cam.cx) * z * ifx;
    v[1] = (y - cam.cy) * z * ify;
    v[2] = z;
}
/* geometry.glsl:29-41: central difference (float overload) */
static void get_normal_central(const float* depth, int W, int H, int tx, int ty, float x, float y,
                               orc_cam cam, float ifx, float ify, const float* vp, float* n)
{
    float xf[3], xb[3], yf[3], yb[3], dx[3], dy[3];
    get_vertex(depth, W, H, tx + 1, ty, x + 1, y, cam, ifx, ify, xf);
    get_vertex(depth, W, H, tx - 1, ty, x - 1, y, cam, ifx, ify, xb);
    get_vertex(depth, W, H, tx, ty + 1, x, y + 1, cam, ifx, ify, yf);
    get_vertex(depth, W, H, tx, ty - 1, x, y - 1, cam, ifx, ify, yb);
    for (int k = 0; k < 3; ++k) {
        dx[k] = ((xb[k] + vp[k]) / 2) - ((xf[k] + vp[k]) / 2);
        dy[k] = ((yb[k] + vp[k]) / 2) - ((yf[k] + vp[k]) / 2);
    }
    cross3(dx, dy, n);
    normalize3(n);
}
/* geometry.glsl:51-60: forward difference (int overload) */
static void get_normal_forward(const float* depth, int W, int H, int tx, int ty,
                               orc_cam cam, float ifx, float ify, const float* vp, float* n)
{
    float vx[3], vy[3], dx[3], dy[3];
    get_vertex(depth, W, H, tx + 1, ty, (float)(tx + 1), (float)ty, cam, ifx, ify, vx);
    get_vertex(depth, W, H, tx, ty + 1, (float)tx, (float)(ty + 1), cam, ifx, ify, vy);
    for (int k = 0; k < 3; ++k) { dx[k] = vx[k] - vp[k]; dy[k] = vy[k] - vp[k]; }
    cross3(dx, dy, n);
    normalize3(n);
}

/* ------------------------------------------------------------------------- */
/* index_map.vert/.frag; ModelProjection.cpp:100-152; rule N2                */
/* ------------------------------------------------------------------------- */
void orc_predict_indices(const float* surfels, int count, const float* pose, orc_cam cam,
                         int W, int H, float maxDepth, int time, int timeDelta,
                         uint32_t* idx, float* vertConf4, float* colorTime4, float* normRad4)
{
    float tinv[16];
    orc_pose_inverse(pose, tinv);
    size_t P = (size_t)W * H;
    uint64_t* key = (uint64_t*)malloc(P * sizeof(uint64_t));
    for (size_t i = 0; i < P; ++i) key[i] = ~0ull;
#pragma omp parallel for schedule(static)
    for (int id = 0; id < count; ++id) {
        const float* s = surfels + (size_t)id * 12;
        float ph[3];
        xform(tinv, s, ph);
        if (ph[2] > maxDepth || ph[2] <= 0 || (float)time - s[7] > (float)timeDelta) continue;
        float x = ((cam.fx * ph[0]) / ph[2]) + cam.cx;
        float y = ((cam.fy * ph[1]) / ph[2]) + cam.cy;
        float zn = ph[2] / maxDepth;
        if (!(zn < 1.0f)) continue;                     /* GL_LESS against the cleared 1.0 */
        float fx_ = floorf(x), fy_ = floorf(y);
        if (!(fx_ >= 0 && fy_ >= 0 && fx_ < (float)W && fy_ < (float)H)) continue;
        int px = (int)fx_, py = (int)fy_;
        uint64_t k = ((uint64_t)fbits(zn) << 32) | (uint32_t)id;
        atomic_min_u64(&key[py * W + px], k);
    }
#pragma omp parallel for schedule(static)
    for (size_t i = 0; i < P; ++i) {
        float* vc = vertConf4 + i * 4; float* ct = colorTime4 + i * 4; float* nr = normRad4 + i * 4;
        if (key[i] == ~0ull) {
            idx[i] = 0;
            for (int k = 0; k < 4; ++k) { vc[k] = 0; ct[k] = 0; nr[k] = 0; }
            continue;
        }
        uint32_t id = (uint32_t)(key[i] & 0xffffffffu);
        const float* s = surfels + (size_t)id * 12;
        float ph[3], n[3];
        xform(tinv, s, ph);
        rot(tinv, s + 8, n);
        normalize3(n);
        idx[i] = id;
        vc[0] = ph[0]; vc[1] = ph[1]; vc[2] = ph[2]; vc[3] = s[3];
        ct[0] = s[4]; ct[1] = s[5]; ct[2] = s[6]; ct[3] = s[7];
        nr[0] = n[0]; nr[1] = n[1]; nr[2] = n[2]; nr[3] = s[11];
    }
    free(key);
}

/* ------------------------------------------------------------------------- */
/* data.vert/.geom/.frag; Model.cpp:466-581; rules N1, N3                    */
/* ------------------------------------------------------------------------- */
static inline float angle_between(const float* a, const float* b)
{
    return orc_acosf(dot3(a, b) / (sqrtf(dot3(a, a)) * sqrtf(dot3(b, b))));
}

void orc_data_associate(const uint8_t* rgb3, const float* depthRaw, const float* depthFilt,
                        const uint8_t* mask, const uint32_t* idx, const float* vertConf4,
                        const float* normRad4, const float* pose, orc_cam cam, int W, int H,
                        float maxDepth, int time, float weighting, uint8_t maskID,
                        uint8_t* updateId, uint32_t* best, float* meas)
{
    const float ifx = 1.0f / cam.fx, ify = 1.0f / cam.fy;          /* Model.cpp:514-515 */
    const float ftime = (float)time;
#pragma omp parallel for schedule(static)
    for (int i = 0; i < W; ++i)
        for (int j = 0; j < H; ++j) {
            int p = i * H + j;                                      /* x-major, Model.cpp:179-183 */
            float tcx = (float)i / (float)W + 0.5f / (float)W;
            float tcy = (float)j / (float)H + 0.5f / (float)H;
            float x = tcx * (float)W, y = tcy * (float)H;
            float vl[3], vg[3], vf[3], nl[3], ng[3];
            get_vertex(depthRaw, W, H, i, j, x, y, cam, ifx, ify, vl);
            xform(pose, vl, vg);
            get_vertex(depthFilt, W, H, i, j, x, y, cam, ifx, ify, vf);
            const uint8_t* c8 = rgb3 + (size_t)(j * W + i) * 3;
            float col[3] = { (float)c8[0] / 255.0f, (float)c8[1] / 255.0f, (float)c8[2] / 255.0f };
            get_normal_central(depthFilt, W, H, i, j, x, y, cam, ifx, ify, vf, nl);
            rot(pose, nl, ng);
            float* m = meas + (size_t)p * 12;
            m[0] = vg[0]; m[1] = vg[1]; m[2] = vg[2]; m[3] = confidence(x, y, weighting, cam.cx, cam.cy);
            m[4] = encode_color(col); m[5] = 0; m[6] = ftime; m[7] = 0;
            m[8] = ng[0]; m[9] = ng[1]; m[10] = ng[2]; m[11] = get_radius(vf[2], nl[2], ifx, ify);
            updateId[p] = 0; best[p] = 0;

            int nb_ok = depthRaw[j * W + clampi(i - 1, 0, W - 1)] != 0 && depthRaw[clampi(j - 1, 0, H - 1) * W + i] != 0 &&
                        depthRaw[j * W + clampi(i + 1, 0, W - 1)] != 0 && depthRaw[clampi(j + 1, 0, H - 1) * W + i] != 0;
            if (((int)x) % 2 == time % 2 && ((int)y) % 2 == time % 2 && mask[j * W + i] == maskID && nb_ok &&
                vl[2] > 0 && vl[2] <= maxDepth) {
                int operation = 0;
                float bestDist = 1000;
                float xl = (x - cam.cx) * ifx, yl = (y - cam.cy) * ify;
                float lambda = sqrtf((xl * xl + yl * yl) + 1);
                float ray[3] = { xl, yl, 1 };
                uint32_t b = 0;
                for (int dx = -1; dx <= 1; ++dx)
                    for (int dy = -1; dy <= 1; ++dy) {
                        int q = clampi(j + dy, 0, H - 1) * W + clampi(i + dx, 0, W - 1);
                        uint32_t cur = idx[q];
                        if (cur > 0u) {
                            const float* vc = vertConf4 + (size_t)q * 4;
                            float zdiff = vc[2] - vl[2];
                            if (fabsf(zdiff * lambda) < 0.05f) {
                                float cr[3];
                                cross3(ray, vc, cr);
                                float dist = sqrtf(dot3(cr, cr));
                                const float* nr = normRad4 + (size_t)q * 4;
                                if (dist < bestDist && (fabsf(nr[2]) < 0.75f || fabsf(angle_between(nr, nl)) < 0.5f)) {
                                    operation = 1; bestDist = dist; b = cur;
                                }
                            }
                        }
                    }
                if (operation == 1) { updateId[p] = 1; m[7] = -1; best[p] = b; }
                else { updateId[p] = 2; m[7] = -2; }
            }
        }
}

/* update.vert:38-111, driven by Model.cpp:583-646; collisions: rule N4 */
void orc_fuse_update(float* surfels, int count, const uint8_t* updateId, const uint32_t* best,
                     const float* meas, int W, int H, int time)
{
    size_t P = (size_t)W * H;
    uint8_t* taken = (uint8_t*)calloc((size_t)(count > 0 ? count : 1), 1);
    for (size_t p = 0; p < P; ++p) {
        if (updateId[p] != 1) continue;
        uint32_t id = best[p];
        if ((int)id >= count || taken[id]) continue;
        taken[id] = 1;
        float* s = surfels + (size_t)id * 12;
        const float* m = meas + p * 12;
        float c_k = s[3], a = m[3];
        if (m[11] < (1.0f + 0.5f) * s[11]) {
            float d = c_k + a;
            for (int k = 0; k < 3; ++k) s[k] = ((c_k * s[k]) + (a * m[k])) / d;
            s[3] = d;
            float oc[3], nc[3], avg[3];
            decode_color(s[4], oc); decode_color(m[4], nc);
            for (int k = 0; k < 3; ++k) avg[k] = ((c_k * oc[k]) + (a * nc[k])) / d;
            s[4] = encode_color(avg);
            s[7] = (float)time;
            for (int k = 8; k < 12; ++k) s[k] = ((c_k * s[k]) + (a * m[k])) / d;
            normalize3(s + 8);
        } else {
            s[3] = c_k + a;
            s[7] = (float)time;
        }
    }
    free(taken);
}

/* ------------------------------------------------------------------------- */
/* copy_unstable.vert/.geom; Model.cpp:649-772; rules N3b, N5, N6            */
/* ------------------------------------------------------------------------- */
static int clean_vertex(const float* in, float* out, const uint32_t* idx, const float* vertConf4,
                        const float* colorTime4, const float* depthFilt, const uint8_t* mask,
                        const float* tinv, orc_cam cam, int W, int H, int time, int timeDelta,
                        float confThreshold, float outlierCoeff, uint8_t maskID)
{
    float v[12];
    memcpy(v, in, sizeof v);
    int test = 1;
    float lp[3], ln[3];
    xform(tinv, v, lp);
    float cols = (float)W, rows = (float)H;
    float x = ((cam.fx * lp[0]) / lp[2]) + cam.cx;
    float y = ((cam.fy * lp[1]) / lp[2]) + cam.cy;
    rot(tinv, v + 8, ln);
    normalize3(ln);
    float x_n = x / cols, y_n = y / rows;
    float stepX = 1.0f / cols, stepY = 1.0f / rows;
    const float scale = 1.0f;                                  /* ModelProjection::FACTOR */
    float ixs = stepX * 0.5f / scale, iys = stepY * 0.5f / scale;
    const float wm = 2;
    int count = 0, zCount = 0;
    float ftime = (float)time;
    if (ftime - v[7] < (float)timeDelta && lp[2] > 0 && x > 0 && y > 0 && x < cols && y < rows) {
        for (float i = x_n - (scale * ixs * wm); i < x_n + (scale * ixs * wm); i += ixs)
            for (float j = y_n - (scale * iys * wm); j < y_n + (scale * iys * wm); j += iys) {
                int tx = clampi((int)floorf(i * cols), 0, W - 1);
                int ty = clampi((int)floorf(j * rows), 0, H - 1);
                int q = ty * W + tx;
                uint32_t cur = idx[q];
                if (cur > 0u) {
                    const float* vc = vertConf4 + (size_t)q * 4;
                    const float* ct = colorTime4 + (size_t)q * 4;
                    float ddx = vc[0] - lp[0], ddy = vc[1] - lp[1];
                    if (ct[2] < v[6] && vc[3] > confThreshold && vc[2] > lp[2] && vc[2] - lp[2] < 0.01f &&
                        sqrtf(ddx * ddx + ddy * ddy) < v[11] * 1.4f)
                        count++;
                    if (ct[3] == ftime && vc[3] > confThreshold && vc[2] > lp[2] && vc[2] - lp[2] > 0.01f &&
                        fabsf(ln[2]) > 0.85f)
                        zCount++;
                }
            }
    }
    if (count > 8 || zCount > 4) test = 0;
    if (v[7] == -2) v[7] = ftime;
    if (v[7] == -1 || ((ftime - v[7]) > 20 && v[3] < confThreshold)) test = 0;
    if (v[7] > 0 && ftime - v[7] > (float)timeDelta) test = 1;

    /* sample at the continuous projection, nearest, clamp-to-edge; NaN -> texel 0 (rule R-CS) */
    float fxs = floorf(x), fys = floorf(y);
    int sx = (fxs != fxs) ? 0 : (fxs < 0 ? 0 : (fxs > (float)(W - 1) ? W - 1 : (int)fxs));
    int sy = (fys != fys) ? 0 : (fys < 0 ? 0 : (fys > (float)(H - 1) ? H - 1 : (int)fys));
    float wDepth = depthFilt[sy * W + sx];
    uint8_t maskValue = mask[sy * W + sx];
    if ((maskValue != maskID) && maskValue < 255 && (wDepth > lp[2] - 0.05f && wDepth < lp[2] + 0.05f)) {
        float f = (0.5f + 0.5f * (1 - outlierCoeff / 10.0f));
        if (maskValue == 0) v[3] *= f;
        else if (maskID == 0) v[3] *= 0.25f * f;
        else v[3] *= f;
    }
    if (test) memcpy(out, v, sizeof v);
    return test;
}

int orc_clean(const float* surfels, int count, const uint8_t* updateId, const float* meas,
              const uint32_t* idx, const float* vertConf4, const float* colorTime4,
              const float* depthFilt, const uint8_t* mask, const float* pose, orc_cam cam,
              int W, int H, int time, int timeDelta, float confThreshold, float outlierCoeff,
              uint8_t maskID, float* out, int capacity)
{
    float tinv[16];
    orc_pose_inverse(pose, tinv);
    /* The per-vertex test is independent of the others; only the ORDER of the survivors matters (N5).  Chunks of vertices are
     * evaluated by all threads into a scratch buffer, then copied out in order -- the same output as the single loop, including the
     * stop at `capacity` (vertices behind the stop have no side effects). */
    enum { CHUNK = 1 << 18 };
    float* tmp = (float*)malloc((size_t)CHUNK * 12 * sizeof(float));
    uint8_t* kept = (uint8_t*)malloc(CHUNK);
    int n = 0;
    size_t P = (size_t)W * H;
    const size_t total = (size_t)count + P;          /* old surfels, then the per-pixel new-vertex slots in x-major order */
    for (size_t base = 0; base < total && n < capacity; base += CHUNK) {
        const size_t m = total - base < (size_t)CHUNK ? total - base : (size_t)CHUNK;
#pragma omp parallel for schedule(static)
        for (size_t j = 0; j < m; ++j) {
            const size_t e = base + j;
            const float* in;
            if (e < (size_t)count) in = surfels + e * 12;
            else {
                const size_t p = e - (size_t)count;
                if (updateId[p] == 0) { kept[j] = 0; continue; }      /* merges (w=-1) are emitted into the buffer but always fail the test */
                in = meas + p * 12;
            }
            kept[j] = (uint8_t)clean_vertex(in, tmp + j * 12, idx, vertConf4, colorTime4, depthFilt, mask,
                                            tinv, cam, W, H, time, timeDelta, confThreshold, outlierCoeff, maskID);
        }
        for (size_t j = 0; j < m && n < capacity; ++j)
            if (kept[j]) { memcpy(out + (size_t)n * 12, tmp + j * 12, 12 * sizeof(float)); ++n; }
    }
    free(tmp); free(kept);
    return n;
}

/* ------------------------------------------------------------------------- */
/* splat.vert + combo_splat.frag / combo_splat_models.frag                   */
/* ------------------------------------------------------------------------- */
typedef struct { float pos[3], conf, n[3], rad, size, xw, yw; int ok; } splat_vs;

static void splat_vertex(const float* s, const float* tinv, orc_cam cam, int W, int H, float maxDepth,
                         float confThreshold, int time, int maxTime, int timeDelta, splat_vs* o)
{
    o->ok = 0;
    float ph[3];
    xform(tinv, s, ph);
    if (ph[2] > maxDepth || ph[2] < 0 || s[3] < confThreshold || (float)time - s[7] > (float)timeDelta || s[7] > (float)maxTime) return;
    o->pos[0] = ph[0]; o->pos[1] = ph[1]; o->pos[2] = ph[2]; o->conf = s[3];
    rot(tinv, s + 8, o->n);
    normalize3(o->n);
    o->rad = s[11];
    float x1[3] = { o->n[1] - o->n[2], -o->n[0], o->n[0] }, y1[3];
    normalize3(x1);
    for (int k = 0; k < 3; ++k) x1[k] = x1[k] * o->rad * 1.41421356f;
    cross3(o->n, x1, y1);
    float px[4], py[4];
    for (int q = 0; q < 4; ++q) {
        const float* d = (q == 0 || q == 3) ? x1 : y1;
        float sg = (q < 2) ? 1.0f : -1.0f;
        float p[3] = { ph[0] + sg * d[0], ph[1] + sg * d[1], ph[2] + sg * d[2] };
        px[q] = ((cam.fx * p[0]) / p[2]) + cam.cx;
        py[q] = ((cam.fy * p[1]) / p[2]) + cam.cy;
    }
    float xmin = fminf(px[0], fminf(px[1], fminf(px[2], px[3]))), xmax = fmaxf(px[0], fmaxf(px[1], fmaxf(px[2], px[3])));
    float ymin = fminf(py[0], fminf(py[1], fminf(py[2], py[3]))), ymax = fmaxf(py[0], fmaxf(py[1], fmaxf(py[2], py[3])));
    float sz = fmaxf(0.0f, fmaxf(fabsf(xmax - xmin), fabsf(ymax - ymin)));
    if (!(sz >= 1.0f)) sz = 1.0f;                  /* GL clamps to the supported range [1, MAX] */
    if (sz > MAX_POINT_SIZE) sz = MAX_POINT_SIZE;
    o->size = sz;
    o->xw = ((cam.fx * ph[0]) / ph[2]) + cam.cx;
    o->yw = ((cam.fy * ph[1]) / ph[2]) + cam.cy;
    /* point clipping by centre against the view volume (GL spec 2.20; rule R-PC) */
    if (!(o->xw >= 0 && o->xw <= (float)W && o->yw >= 0 && o->yw <= (float)H)) return;
    if (!(ph[2] / maxDepth <= 1.0f)) return;
    o->ok = 1;
}

/* fragment: returns 0 if discarded; corrected position in cp */
static inline int splat_fragment(const splat_vs* v, orc_cam cam, float fcx, float fcy, float* cp)
{
    float l[3] = { (fcx - cam.cx) / cam.fx, (fcy - cam.cy) / cam.fy, 1.0f };
    normalize3(l);
    float t = dot3(v->pos, v->n) / dot3(l, v->n);
    cp[0] = t * l[0]; cp[1] = t * l[1]; cp[2] = t * l[2];
    float sqrRad = v->rad * v->rad;
    float d[3] = { cp[0] - v->pos[0], cp[1] - v->pos[1], cp[2] - v->pos[2] };
    if (dot3(d, d) > sqrRad) return 0;
    return 1;
}

static void splat_range(const splat_vs* v, int W, int H, int* x0, int* x1, int* y0, int* y1)
{
    /* pixel centres c with  xw - s/2 <= c < xw + s/2  (rule R-PR) */
    float h = v->size * 0.5f;
    float lo = ceilf(v->xw - h - 0.5f), hi = ceilf(v->xw + h - 0.5f) - 1.0f;
    *x0 = lo < 0 ? 0 : (int)lo; *x1 = hi > (float)(W - 1) ? W - 1 : (int)hi;
    lo = ceilf(v->yw - h - 0.5f); hi = ceilf(v->yw + h - 0.5f) - 1.0f;
    *y0 = lo < 0 ? 0 : (int)lo; *y1 = hi > (float)(H - 1) ? H - 1 : (int)hi;
}

void orc_splat_extent(const float* surfel, const float* pose, orc_cam cam, int W, int H, float maxDepth, float confThreshold,
                      int time, int maxTime, int timeDelta, float* out)
{
    float tinv[16];
    orc_pose_inverse(pose, tinv);
    splat_vs v;
    memset(&v, 0, sizeof v);
    splat_vertex(surfel, tinv, cam, W, H, maxDepth, confThreshold, time, maxTime, timeDelta, &v);
    int x0 = 0, x1 = -1, y0 = 0, y1 = -1;
    if (v.ok) splat_range(&v, W, H, &x0, &x1, &y0, &y1);
    const float o[16] = { (float)v.ok, v.size, v.xw, v.yw, (float)x0, (float)x1, (float)y0, (float)y1,
                          v.pos[0], v.pos[1], v.pos[2], v.n[0], v.n[1], v.n[2], v.rad, v.conf };
    memcpy(out, o, sizeof o);
}

static void splat_keys(const float* surfels, int count, const float* tinv, orc_cam cam, int W, int H,
                       float maxDepth, float confThreshold, int time, int maxTime, int timeDelta,
                       uint32_t drawBase, uint64_t* key)
{
#pragma omp parallel for schedule(dynamic, 4096)
    for (int id = 0; id < count; ++id) {
        splat_vs v;
        splat_vertex(surfels + (size_t)id * 12, tinv, cam, W, H, maxDepth, confThreshold, time, maxTime, timeDelta, &v);
        if (!v.ok) continue;
        int x0, x1, y0, y1;
        splat_range(&v, W, H, &x0, &x1, &y0, &y1);
        for (int py = y0; py <= y1; ++py)
            for (int px = x0; px <= x1; ++px) {
                float cp[3];
                if (!splat_fragment(&v, cam, (float)px + 0.5f, (float)py + 0.5f, cp)) continue;
                float fd = (cp[2] / (2 * maxDepth)) + 0.5f;
                if (!(fd >= 0.0f && fd < 1.0f)) continue;          /* depth clamp + GL_LESS vs cleared 1.0; NaN fails */
                uint64_t k = ((uint64_t)fbits(fd) << 32) | (uint32_t)(drawBase + (uint32_t)id);
                atomic_min_u64(&key[py * W + px], k);
            }
    }
}

/* ModelProjection.cpp:187-268 */
void orc_combined_predict(const float* surfels, int count, const float* pose, orc_cam cam,
                          int W, int H, float maxDepth, float confThreshold, int time, int maxTime,
                          int timeDelta, uint8_t* image4, float* vertexConf4, float* normalRad4,
                          uint16_t* timeTex)
{
    float tinv[16];
    orc_pose_inverse(pose, tinv);
    size_t P = (size_t)W * H;
    uint64_t* key = (uint64_t*)malloc(P * sizeof(uint64_t));
    for (size_t i = 0; i < P; ++i) key[i] = ~0ull;
    splat_keys(surfels, count, tinv, cam, W, H, maxDepth, confThreshold, time, maxTime, timeDelta, 0, key);
#pragma omp parallel for schedule(static)
    for (int py = 0; py < H; ++py)
        for (int px = 0; px < W; ++px) {
            size_t i = (size_t)py * W + px;
            uint8_t* im = image4 + i * 4; float* vc = vertexConf4 + i * 4; float* nr = normalRad4 + i * 4;
            if (key[i] == ~0ull) {
                for (int k = 0; k < 4; ++k) { im[k] = 0; vc[k] = 0; nr[k] = 0; }
                timeTex[i] = 0;
                continue;
            }
            uint32_t id = (uint32_t)(key[i] & 0xffffffffu);
            const float* s = surfels + (size_t)id * 12;
            splat_vs v;
            splat_vertex(s, tinv, cam, W, H, maxDepth, confThreshold, time, maxTime, timeDelta, &v);
            float cp[3], fcx = (float)px + 0.5f, fcy = (float)py + 0.5f;
            splat_fragment(&v, cam, fcx, fcy, cp);
            float col[3];
            decode_color(s[4], col);
            for (int k = 0; k < 3; ++k) im[k] = (uint8_t)(int)floorf(col[k] * 255.0f + 0.5f);
            im[3] = 255;
            float z = cp[2];
            vc[0] = (fcx - cam.cx) * z * (1.f / cam.fx);
            vc[1] = (fcy - cam.cy) * z * (1.f / cam.fy);
            vc[2] = z; vc[3] = v.conf;
            nr[0] = v.n[0]; nr[1] = v.n[1]; nr[2] = v.n[2]; nr[3] = v.rad;
            timeTex[i] = (uint16_t)(uint32_t)s[6];
        }
    free(key);
}

/* GlobalProjection.cpp:43-107 */
void orc_global_projection_begin(int W, int H, uint64_t* keys)
{
    for (size_t i = 0; i < (size_t)W * H; ++i) keys[i] = ~0ull;
}
void orc_global_projection_add(const float* surfels, int count, const float* pose, orc_cam cam,
                               int W, int H, float maxDepth, float confThreshold, int time,
                               int maxTime, int timeDelta, uint32_t drawBase, uint64_t* keys)
{
    float tinv[16];
    orc_pose_inverse(pose, tinv);
    splat_keys(surfels, count, tinv, cam, W, H, maxDepth, confThreshold, time, maxTime, timeDelta, drawBase, keys);
}

/* ------------------------------------------------------------------------- */
/* fill_{vertex,normal,rgb}.frag; FillIn.cpp; Model.cpp:976-984              */
/* ------------------------------------------------------------------------- */
void orc_fill_in(const float* vertexConf4, const float* normalRad4, const uint8_t* image4,
                 const float* depthFilt, const uint8_t* rgb3, orc_cam cam, int W, int H,
                 int ptVN, int ptImg, float* fillVertex4, float* fillNormal4, uint8_t* fillImage4)
{
    const float ifx = 1.0f / cam.fx, ify = 1.0f / cam.fy;
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            size_t i = (size_t)y * W + x;
            const float* sv = vertexConf4 + i * 4; const float* sn = normalRad4 + i * 4; const uint8_t* si = image4 + i * 4;
            float vp[3];
            get_vertex(depthFilt, W, H, x, y, (float)x, (float)y, cam, ifx, ify, vp);
            if (sv[2] == 0 || ptVN) { fillVertex4[i * 4] = vp[0]; fillVertex4[i * 4 + 1] = vp[1]; fillVertex4[i * 4 + 2] = vp[2]; fillVertex4[i * 4 + 3] = 1; }
            else memcpy(fillVertex4 + i * 4, sv, 4 * sizeof(float));
            if (sn[2] == 0 || ptVN) {
                float n[3];
                get_normal_forward(depthFilt, W, H, x, y, cam, ifx, ify, vp, n);
                fillNormal4[i * 4] = n[0]; fillNormal4[i * 4 + 1] = n[1]; fillNormal4[i * 4 + 2] = n[2]; fillNormal4[i * 4 + 3] = 1;
            } else memcpy(fillNormal4 + i * 4, sn, 4 * sizeof(float));
            float sum = ((float)si[0] / 255.0f + (float)si[1] / 255.0f) + (float)si[2] / 255.0f;
            if (sum == 0 || ptImg) { fillImage4[i * 4] = rgb3[i * 3]; fillImage4[i * 4 + 1] = rgb3[i * 3 + 1]; fillImage4[i * 4 + 2] = rgb3[i * 3 + 2]; fillImage4[i * 4 + 3] = 255; }
            else memcpy(fillImage4 + i * 4, si, 4);
        }
}

/* resize.frag + GPUResize::image (Resize.cpp:43-75) + MaskFusion.cpp:630-648:
 * dest (W/20 x H/20), source texel (20i+10, 20j+10) (texel-edge sample, nearest) */
int orc_requires_fill_in(const uint8_t* image4, int W, int H, float ratio)
{
    int dw = W / 20, dh = H / 20, sum = 0;
    for (int j = 0; j < dh; ++j)
        for (int i = 0; i < dw; ++i) {
            int sx = clampi(i * 20 + 10, 0, W - 1), sy = clampi(j * 20 + 10, 0, H - 1);
            const uint8_t* p = image4 + ((size_t)sy * W + sx) * 4;
            sum += (p[0] > 0 && p[1] > 0 && p[2] > 0);
        }
    return (float)sum / (float)(dh * dw) < ratio;
}

/* ------------------------------------------------------------------------- */
/* vertex_feedback.vert/.geom (FeedbackBuffer.cpp:78-128) + init_unstable.vert */
/* (Model.cpp:240-285): raw stream supplies position+colour, filtered stream  */
/* supplies normal+radius, paired by emission index; count = raw stream.      */
/* ------------------------------------------------------------------------- */
int orc_init_model(const uint8_t* rgb3, const float* depthRaw, const float* depthFilt,
                   orc_cam cam, int W, int H, int time, float maxDepth, float* out, int capacity)
{
    const float ifx = 1.0f / cam.fx, ify = 1.0f / cam.fy;
    int nraw = 0, nfil = 0;
    for (int pass = 0; pass < 2; ++pass) {
        const float* depth = pass == 0 ? depthRaw : depthFilt;
        int n = 0;
        for (int i = 0; i < W; ++i)
            for (int j = 0; j < H; ++j) {
                float tcx = (float)(((double)((float)i / (float)W)) + 1.0 / (double)(2 * (float)W));   /* FeedbackBuffer.cpp:44-49 */
                float tcy = (float)(((double)((float)j / (float)H)) + 1.0 / (double)(2 * (float)H));
                float x = tcx * (float)W, y = tcy * (float)H;
                float vp[3], nl[3];
                get_vertex(depth, W, H, i, j, x, y, cam, ifx, ify, vp);
                if (vp[2] <= 0 || vp[2] > maxDepth) continue;
                if (n >= capacity) continue;
                float* o = out + (size_t)n * 12;
                if (pass == 0) {
                    const uint8_t* c8 = rgb3 + (size_t)(j * W + i) * 3;
                    float col[3] = { (float)c8[0] / 255.0f, (float)c8[1] / 255.0f, (float)c8[2] / 255.0f };
                    o[0] = vp[0]; o[1] = vp[1]; o[2] = vp[2]; o[3] = confidence(x, y, 1.0f, cam.cx, cam.cy);
                    o[4] = encode_color(col); o[5] = 0; o[6] = 1; o[7] = (float)time;
                    o[8] = o[9] = o[10] = o[11] = 0;
                } else {
                    get_normal_central(depth, W, H, i, j, x, y, cam, ifx, ify, vp, nl);
                    o[8] = nl[0]; o[9] = nl[1]; o[10] = nl[2]; o[11] = get_radius(vp[2], nl[2], ifx, ify);
                }
                ++n;
            }
        if (pass == 0) nraw = n; else nfil = n;
    }
    (void)nfil;
    return nraw;
}
