// mf_surfel.cu -- surfel-map kernels (sm_90a).  These replace the reference's OpenGL
// passes; there is no rasteriser here.
//   predictIndices  <- index_map.vert/.frag,            ModelProjection.cpp:100-152
//   associate       <- data.vert/.geom/.frag,           Model.cpp:466-581
//   fuseUpdate      <- update.vert,                     Model.cpp:583-646
//   clean           <- copy_unstable.vert/.geom,        Model.cpp:649-772
//   combinedPredict <- splat.vert + combo_splat.frag,   ModelProjection.cpp:187-268
//   fillIn          <- fill_{vertex,normal,rgb}.frag,   Shaders/FillIn.cpp
//   initModel       <- vertex_feedback.* + init_unstable.vert, Model.cpp:240-285
//
// Surfel store: three float4 planes (position|conf, colour|.|initTime|lastTime,
// normal|radius) -> every pass streams 16-byte coalesced loads (the reference's VBO is
// 48-byte AoS).  Depth-tested rasterisation is a 64-bit atomicMin on
// (depth bits << 32 | surfel id): nearest fragment wins, ties go to the lowest id, which
// is the GL_LESS + draw-order rule (N2).  Keys are reset by the resolve kernel that
// consumes them, so no per-pass clear of per-pixel or per-surfel state is ever issued
// (the reference clears 3 x texDim^2 x 16 B of update maps on every fuse).
#include "mf_common.cuh"
#include "mf_kernels.h"
#include "mf_host.h"

namespace mfb {

#define MAX_POINT_SIZE 2047.0f

// ---------------------------------------------------------------------------------------
// index map
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_index_project(const float4* __restrict__ pos, const float4* __restrict__ col,
                                                       const uint32_t* __restrict__ countPtr, const DevPose* __restrict__ dpose, Cam cam, int W, int H,
                                                       float maxDepth, float ftime, float ftimeDelta,
                                                       unsigned long long* __restrict__ key)
{
    const Rt tinv = dpose->tinv;
    const uint32_t count = *countPtr;
    for (uint32_t id = blockIdx.x * blockDim.x + threadIdx.x; id < count; id += gridDim.x * blockDim.x) {
        float4 p = ldStream(pos + id);
        float lastTime = ldStream(col + id).w;
        float3 ph = xform(tinv, make_float3(p.x, p.y, p.z));
        if (ph.z > maxDepth || ph.z <= 0 || ftime - lastTime > ftimeDelta) continue;
        float x = ((cam.fx * ph.x) / ph.z) + cam.cx;
        float y = ((cam.fy * ph.y) / ph.z) + cam.cy;
        float zn = ph.z / maxDepth;
        if (!(zn < 1.0f)) continue;
        float fx_ = floorf(x), fy_ = floorf(y);
        if (!(fx_ >= 0 && fy_ >= 0 && fx_ < (float)W && fy_ < (float)H)) continue;
        unsigned long long k = ((unsigned long long)__float_as_uint(zn) << 32) | id;
        unsigned long long* dst = key + ((int)fy_ * W + (int)fx_);
        if (k < *dst) atomicMin(dst, k);
    }
}

__global__ void k_index_resolve(const float4* __restrict__ pos, const float4* __restrict__ col, const float4* __restrict__ nrm,
                                const DevPose* __restrict__ dpose, int P, unsigned long long* __restrict__ key, uint32_t* __restrict__ idx,
                                float4* __restrict__ vertConf, float4* __restrict__ colorTime, float4* __restrict__ normRad,
                                float4* __restrict__ cleanTex, float cleanConf, float cleanTime)
{
    // cleanTex: what the window of the clean pass (copy_unstable.vert:86-113) reads per texel, packed into ONE 16-byte word:
    //   (x, y, z | sign bit: conf > confThreshold,  initTime | sign bit: lastTime == time);  all zero = empty texel (or surfel 0, N2).
    // z > 0 for every drawn surfel and initTime >= 0, so both sign bits are free; the two tests they carry are the only uses the
    // window makes of the confidence and of the last-seen time, evaluated here with the thresholds of the clean call that follows
    // (Model::clean falls back to the three index-map images when it is called with other thresholds).  Three images cost three
    // sectors per tap, the 32-byte record of round 1 one; 16 bytes let a thread hold its whole 3x3 window in registers and issue the
    // nine loads together.
    const Rt tinv = dpose->tinv;
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    unsigned long long k = key[i];
    if (k == KEY_EMPTY) {
        idx[i] = 0;
        float4 z = make_float4(0, 0, 0, 0);
        vertConf[i] = z; colorTime[i] = z; normRad[i] = z;
        if (cleanTex) cleanTex[i] = z;
        return;
    }
    key[i] = KEY_EMPTY;
    uint32_t id = (uint32_t)(k & 0xffffffffull);
    float4 p = pos[id], c = col[id], n = nrm[id];
    float3 ph = xform(tinv, make_float3(p.x, p.y, p.z));
    float3 nn = normalize3(rotate(tinv, make_float3(n.x, n.y, n.z)));
    idx[i] = id;
    vertConf[i] = make_float4(ph.x, ph.y, ph.z, p.w);
    colorTime[i] = c;
    normRad[i] = make_float4(nn.x, nn.y, nn.z, n.w);
    if (cleanTex) {
        const uint32_t zb = (__float_as_uint(ph.z) & 0x7fffffffu) | (p.w > cleanConf ? 0x80000000u : 0u);
        const uint32_t tb = (__float_as_uint(c.z) & 0x7fffffffu) | (c.w == cleanTime ? 0x80000000u : 0u);
        cleanTex[i] = id != 0u ? make_float4(ph.x, ph.y, __uint_as_float(zb), __uint_as_float(tb)) : make_float4(0, 0, 0, 0);
    }
}

// ---------------------------------------------------------------------------------------
// frame-side vertex helpers (geometry.glsl)
// ---------------------------------------------------------------------------------------
MF_D float3 getVertex(const float* __restrict__ depth, int W, int H, int tx, int ty, float x, float y, Cam cam, float ifx, float ify)
{
    float z = depth[clampi(ty, 0, H - 1) * W + clampi(tx, 0, W - 1)];
    return make_float3((x - cam.cx) * z * ifx, (y - cam.cy) * z * ify, z);
}
MF_D float3 normalCentral(const float* __restrict__ depth, int W, int H, int tx, int ty, float x, float y, Cam cam, float ifx, float ify, float3 vp)
{
    float3 xf = getVertex(depth, W, H, tx + 1, ty, x + 1, y, cam, ifx, ify);
    float3 xb = getVertex(depth, W, H, tx - 1, ty, x - 1, y, cam, ifx, ify);
    float3 yf = getVertex(depth, W, H, tx, ty + 1, x, y + 1, cam, ifx, ify);
    float3 yb = getVertex(depth, W, H, tx, ty - 1, x, y - 1, cam, ifx, ify);
    float3 dx = make_float3(((xb.x + vp.x) / 2) - ((xf.x + vp.x) / 2), ((xb.y + vp.y) / 2) - ((xf.y + vp.y) / 2), ((xb.z + vp.z) / 2) - ((xf.z + vp.z) / 2));
    float3 dy = make_float3(((yb.x + vp.x) / 2) - ((yf.x + vp.x) / 2), ((yb.y + vp.y) / 2) - ((yf.y + vp.y) / 2), ((yb.z + vp.z) / 2) - ((yf.z + vp.z) / 2));
    return normalize3(cross3(dx, dy));
}
MF_D float3 normalForward(const float* __restrict__ depth, int W, int H, int tx, int ty, Cam cam, float ifx, float ify, float3 vp)
{
    float3 vx = getVertex(depth, W, H, tx + 1, ty, (float)(tx + 1), (float)ty, cam, ifx, ify);
    float3 vy = getVertex(depth, W, H, tx, ty + 1, (float)tx, (float)(ty + 1), cam, ifx, ify);
    return normalize3(cross3(sub3(vx, vp), sub3(vy, vp)));
}

// ---------------------------------------------------------------------------------------
// data association: one thread per pixel (row-major => coalesced frame reads); results are
// stored at the x-major order index p = x*H + y that the reference's draw order defines.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_associate(const uchar4* __restrict__ rgb, const float* __restrict__ depthRaw,
                                                   const float* __restrict__ depthFilt, const uint8_t* __restrict__ mask,
                                                   const uint32_t* __restrict__ idx, const float4* __restrict__ vertConf,
                                                   const float4* __restrict__ normRad, const DevPose* __restrict__ dpose, Cam cam, int W, int H,
                                                   float maxDepth, int time, float weightMultiplier, uint8_t maskID,
                                                   uint8_t* __restrict__ flag, uint32_t* __restrict__ best,
                                                   float4* __restrict__ m0, float4* __restrict__ m1, float4* __restrict__ m2,
                                                   uint32_t* __restrict__ slot)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= W || j >= H) return;
    const int p = i * H + j;
    const float ifx = 1.0f / cam.fx, ify = 1.0f / cam.fy;
    float tcx = (float)i / (float)W + 0.5f / (float)W;
    float tcy = (float)j / (float)H + 0.5f / (float)H;
    float x = tcx * (float)W, y = tcy * (float)H;
    uint8_t f = 0;
    float3 vl = getVertex(depthRaw, W, H, i, j, x, y, cam, ifx, ify);
    bool cand = ((int)x) % 2 == time % 2 && ((int)y) % 2 == time % 2 && mask[j * W + i] == maskID && vl.z > 0 && vl.z <= maxDepth;
    if (cand) {
        cand = depthRaw[j * W + clampi(i - 1, 0, W - 1)] != 0 && depthRaw[clampi(j - 1, 0, H - 1) * W + i] != 0 &&
               depthRaw[j * W + clampi(i + 1, 0, W - 1)] != 0 && depthRaw[clampi(j + 1, 0, H - 1) * W + i] != 0;
    }
    if (cand) {
        const Rt pose = dpose->pose;
        const float weighting = dpose->fusionW * weightMultiplier;          // Model::computeFusionWeight (Model.cpp:449-464)
        float3 vg = xform(pose, vl);
        float3 vf = getVertex(depthFilt, W, H, i, j, x, y, cam, ifx, ify);
        float3 nl = normalCentral(depthFilt, W, H, i, j, x, y, cam, ifx, ify, vf);
        float3 ng = rotate(pose, nl);
        uchar4 c8 = rgb[j * W + i];
        float enc = encodeColor((float)c8.x / 255.0f, (float)c8.y / 255.0f, (float)c8.z / 255.0f);
        float conf = surfelConfidence(x, y, weighting, cam.cx, cam.cy);
        float rad = surfelRadius(vf.z, nl.z, ifx, ify);

        float bestDist = 1000;
        float xl = (x - cam.cx) * ifx, yl = (y - cam.cy) * ify;
        float lambda = sqrtf((xl * xl + yl * yl) + 1);
        float3 ray = make_float3(xl, yl, 1);
        uint32_t b = 0; int operation = 0;
        for (int dx = -1; dx <= 1; ++dx)
            for (int dy = -1; dy <= 1; ++dy) {
                int q = clampi(j + dy, 0, H - 1) * W + clampi(i + dx, 0, W - 1);
                uint32_t cur = idx[q];
                if (cur > 0u) {
                    float4 vc = vertConf[q];
                    float zdiff = vc.z - vl.z;
                    if (fabsf(zdiff * lambda) < 0.05f) {
                        float3 cr = cross3(ray, make_float3(vc.x, vc.y, vc.z));
                        float dist = sqrtf(dot3(cr, cr));
                        float4 nr = normRad[q];
                        if (dist < bestDist) {
                            float3 a = make_float3(nr.x, nr.y, nr.z);
                            bool okn = fabsf(nr.z) < 0.75f ||
                                       fabsf(det_acosf(dot3(a, nl) / (sqrtf(dot3(a, a)) * sqrtf(dot3(nl, nl))))) < 0.5f;
                            if (okn) { operation = 1; bestDist = dist; b = cur; }
                        }
                    }
                }
            }
        f = operation ? 1 : 2;
        m0[p] = make_float4(vg.x, vg.y, vg.z, conf);
        m1[p] = make_float4(enc, 0.f, (float)time, operation ? -1.f : -2.f);
        m2[p] = make_float4(ng.x, ng.y, ng.z, rad);
        best[p] = b;
        if (operation) atomicMin(slot + b, (uint32_t)p);        // N4: first pixel in draw order wins
    }
    flag[p] = f;
}

// winners update their surfel in place (the reference rewrites the whole VBO; only the
// <= P/4 associated surfels change, so the contents are identical)
__global__ void k_fuse_update(const uint8_t* __restrict__ flag, const uint32_t* __restrict__ best,
                              const float4* __restrict__ m0, const float4* __restrict__ m1, const float4* __restrict__ m2,
                              const uint32_t* __restrict__ slot, int P, int time,
                              float4* __restrict__ pos, float4* __restrict__ col, float4* __restrict__ nrm)
{
    int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P || flag[p] != 1) return;
    uint32_t id = best[p];
    if (slot[id] != (uint32_t)p) return;
    float4 sp = pos[id], sc = col[id], sn = nrm[id];
    float4 np_ = m0[p], nc = m1[p], nn = m2[p];
    float c_k = sp.w, a = np_.w;
    if (nn.w < (1.0f + 0.5f) * sn.w) {
        float d = c_k + a;
        sp = make_float4(((c_k * sp.x) + (a * np_.x)) / d, ((c_k * sp.y) + (a * np_.y)) / d, ((c_k * sp.z) + (a * np_.z)) / d, d);
        float3 oc = decodeColor(sc.x), ncl = decodeColor(nc.x);
        sc.x = encodeColor(((c_k * oc.x) + (a * ncl.x)) / d, ((c_k * oc.y) + (a * ncl.y)) / d, ((c_k * oc.z) + (a * ncl.z)) / d);
        sc.w = (float)time;
        float4 avg = make_float4(((c_k * sn.x) + (a * nn.x)) / d, ((c_k * sn.y) + (a * nn.y)) / d, ((c_k * sn.z) + (a * nn.z)) / d,
                                 ((c_k * sn.w) + (a * nn.w)) / d);
        float3 u = normalize3(make_float3(avg.x, avg.y, avg.z));
        sn = make_float4(u.x, u.y, u.z, avg.w);
    } else {
        sp.w = c_k + a;
        sc.w = (float)time;
    }
    pos[id] = sp; col[id] = sc; nrm[id] = sn;
}

// release the update slots taken this frame (self-cleaning; runs after k_fuse_update)
__global__ void k_slot_release(const uint8_t* __restrict__ flag, const uint32_t* __restrict__ best, int P, uint32_t* __restrict__ slot)
{
    int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P || flag[p] != 1) return;
    slot[best[p]] = 0xffffffffu;
}

// ---------------------------------------------------------------------------------------
// clean: per-vertex test (copy_unstable.vert) + ordered compaction (N5)
// ---------------------------------------------------------------------------------------
struct CleanParams {
    Rt tinv; Cam cam; int W, H; int time; float ftimeDelta; float confThreshold; float outlierCoeff; uint8_t maskID;
};

// ---- clean, restructured for dense execution -------------------------------------------------
// Only surfels that project into the image need the index-map window and they are scattered through
// the store: evaluated inline per thread the window code ran with ~9 of 32 lanes active, and a
// warp-cooperative variant was instruction bound.  So each block (1) projects its
// 512 surfels, (2) compacts the ones that need a window into shared memory, (3) runs the window code
// densely, one compacted entry per thread, (4) hands the counts back to the owning threads.
struct CleanEntry { float xn, yn, lx, ly, lz, init, rad, lnz; };

// window of copy_unstable.vert:86-113 for one surfel.  The shader walks a 4x4 (5 on rounding) grid of
// half-texel steps; the taps land on 2-3 distinct texels per axis and the per-tap tests depend on the texel
// alone: run the literal float loops for the texel columns/rows, visit each DISTINCT texel once, weight by
// its multiplicity (same counts as the tap loop, ~4x fewer loads).
// window texels: the packed 16-byte records (PACKED) or, when the clean call's thresholds differ from the ones the records were
// written with, the three index-map images themselves
struct CleanTexels { const float4* packed; const float4* vertConf; const float4* colorTime; const uint32_t* idx; };
template <bool PACKED>
MF_D void cleanWindow(const CleanEntry& e, const CleanParams& P, const CleanTexels& tx, int& count, int& zCount)
{
    const int W = P.W, H = P.H;
    const float cols = (float)W, rows = (float)H, ftime = (float)P.time;
    const float stepX = 1.0f / cols, stepY = 1.0f / rows;
    const float scale = 1.0f, wm = 2;
    const float ixs = stepX * 0.5f / scale, iys = stepY * 0.5f / scale;
    int txs[5], tys[5]; int nx = 0, ny = 0;
#pragma unroll
    for (int k = 0; k < 5; ++k) { txs[k] = -1; tys[k] = -1; }
    for (float i = e.xn - (scale * ixs * wm); i < e.xn + (scale * ixs * wm); i += ixs) {
        int t = clampi((int)floorf(i * cols), 0, W - 1);
#pragma unroll
        for (int k = 0; k < 5; ++k) if (k == nx) txs[k] = t;
        ++nx;
    }
    for (float j = e.yn - (scale * iys * wm); j < e.yn + (scale * iys * wm); j += iys) {
        int t = clampi((int)floorf(j * rows), 0, H - 1);
#pragma unroll
        for (int k = 0; k < 5; ++k) if (k == ny) tys[k] = t;
        ++ny;
    }
    // unused slots hold -1 and never match a texel
    int mxs[5], mys[5];
#pragma unroll
    for (int a = 0; a < 5; ++a) {
        mxs[a] = 0; mys[a] = 0;
#pragma unroll
        for (int c = 0; c < 5; ++c) { mxs[a] += (txs[c] == txs[a]) ? 1 : 0; mys[a] += (tys[c] == tys[a]) ? 1 : 0; }
    }
    // The tap coordinates are monotone and span two texels: at most three DISTINCT columns / rows, equal ones adjacent.
    // Compact them (texel, multiplicity) so that the loads of a whole window row can be issued together: walked one texel at a
    // time every tap paid a full L2 round trip before the next address was even formed.
    int ux[3] = {0, 0, 0}, wx[3] = {0, 0, 0}, uy[3] = {0, 0, 0}, wy[3] = {0, 0, 0};
    int nux = 0, nuy = 0;
#pragma unroll
    for (int a = 0; a < 5; ++a) {
        if (!(txs[a] < 0 || (a > 0 && txs[a] == txs[a - 1]))) {
#pragma unroll
            for (int k = 0; k < 3; ++k) if (k == nux) { ux[k] = txs[a]; wx[k] = mxs[a]; }
            ++nux;
        }
        if (!(tys[a] < 0 || (a > 0 && tys[a] == tys[a - 1]))) {
#pragma unroll
            for (int k = 0; k < 3; ++k) if (k == nuy) { uy[k] = tys[a]; wy[k] = mys[a]; }
            ++nuy;
        }
    }
    count = 0; zCount = 0;
    if (PACKED) {
        // the whole window at once: nine independent 16-byte loads (slots beyond nux / nuy repeat texel 0 with weight 0), one L2 round trip
        float4 t[3][3];
#pragma unroll
        for (int b = 0; b < 3; ++b)
#pragma unroll
            for (int k = 0; k < 3; ++k) t[b][k] = __ldg(tx.packed + (uy[b] * W + ux[k]));
#pragma unroll
        for (int b = 0; b < 3; ++b)
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const uint32_t zb = __float_as_uint(t[b][k].z), tb = __float_as_uint(t[b][k].w);
                if (b >= nuy || k >= nux || (zb & 0x7fffffffu) == 0u) continue;     // empty texel (or surfel 0, N2)
                const float mz = __uint_as_float(zb & 0x7fffffffu), initT = __uint_as_float(tb & 0x7fffffffu);
                const bool confOK = (zb >> 31) != 0u, lastNow = (tb >> 31) != 0u;
                const float ddx = t[b][k].x - e.lx, ddy = t[b][k].y - e.ly;
                if (initT < e.init && confOK && mz > e.lz && mz - e.lz < 0.01f && sqrtf(ddx * ddx + ddy * ddy) < e.rad * 1.4f)
                    count += wx[k] * wy[b];
                if (lastNow && confOK && mz > e.lz && mz - e.lz > 0.01f && e.lnz > 0.85f)
                    zCount += wx[k] * wy[b];
            }
        return;
    }
#pragma unroll
    for (int b = 0; b < 3; ++b) {
        if (b >= nuy) break;
        float4 mc[3], tt[3]; uint32_t oc[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {                        // slots beyond nux repeat column 0 (weight 0): the loads are unconditional
            const int q = uy[b] * W + ux[k];
            mc[k] = __ldg(tx.vertConf + q); tt[k] = __ldg(tx.colorTime + q); oc[k] = __ldg(tx.idx + q);
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            if (k >= nux || oc[k] == 0u) continue;           // idx == 0: empty texel (or surfel 0, N2)
            const float initT = tt[k].z, lastT = tt[k].w;
            const float ddx = mc[k].x - e.lx, ddy = mc[k].y - e.ly;
            if (initT < e.init && mc[k].w > P.confThreshold && mc[k].z > e.lz && mc[k].z - e.lz < 0.01f && sqrtf(ddx * ddx + ddy * ddy) < e.rad * 1.4f)
                count += wx[k] * wy[b];
            if (lastT == ftime && mc[k].w > P.confThreshold && mc[k].z > e.lz && mc[k].z - e.lz > 0.01f && e.lnz > 0.85f)
                zCount += wx[k] * wy[b];
        }
    }
}

// everything of copy_unstable.vert after the window (:128-157)
MF_D bool cleanFinish(float4& vp, float4& vc, float x, float y, float lpz, int count, int zCount, const CleanParams& P,
                      const float* __restrict__ depthFilt, const uint8_t* __restrict__ mask)
{
    const int W = P.W, H = P.H;
    const float ftime = (float)P.time;
    bool test = true;
    if (count > 8 || zCount > 4) test = false;
    if (vc.w == -2) vc.w = ftime;
    if (vc.w == -1 || ((ftime - vc.w) > 20 && vp.w < P.confThreshold)) test = false;
    if (vc.w > 0 && ftime - vc.w > P.ftimeDelta) test = true;
    float fxs = floorf(x), fys = floorf(y);
    int sx = (fxs != fxs) ? 0 : (fxs < 0 ? 0 : (fxs > (float)(W - 1) ? W - 1 : (int)fxs));
    int sy = (fys != fys) ? 0 : (fys < 0 ? 0 : (fys > (float)(H - 1) ? H - 1 : (int)fys));
    float wDepth = depthFilt[sy * W + sx];
    uint8_t maskValue = mask[sy * W + sx];
    if ((maskValue != P.maskID) && maskValue < 255 && (wDepth > lpz - 0.05f && wDepth < lpz + 0.05f)) {
        float f = (0.5f + 0.5f * (1 - P.outlierCoeff / 10.0f));
        if (maskValue == 0) vp.w *= f;
        else if (P.maskID == 0) vp.w *= 0.25f * f;
        else vp.w *= f;
    }
    return test;
}

#define SCAN_BLOCK 512
// clean, pass 1a: stream the whole store once (old surfels, then the new vertices emitted by the association pass).
// A vertex that does not project into the image needs no index-map window: it is finished here.  The others are
// only REGISTERED in a device-wide candidate list; pass 1b works that list densely.
// (An in-kernel window ran with 9/32 lanes active; a block-compacted variant was still latency bound at 2 blocks/SM.)
#define CAND_BUF 2048
__global__ void __launch_bounds__(256, 8) k_clean_p1(float4* __restrict__ pos, float4* __restrict__ col, const uint32_t* __restrict__ countPtr,
                                                  const uint8_t* __restrict__ aflag, float4* __restrict__ m0, float4* __restrict__ m1, int Ppix,
                                                  CleanParams P, const DevPose* __restrict__ dpose, const float* __restrict__ depthFilt, const uint8_t* __restrict__ mask,
                                                  uint8_t* __restrict__ keep, uint32_t* __restrict__ cand, uint32_t* __restrict__ candCount,
                                                  unsigned long long* __restrict__ indexKey, float indexMaxDepth)
{
    // indexKey != nullptr: this pass ALSO is the index-map projection of Model::predictIndices that precedes Model::clean in the frame
    // (MaskFusion.cpp:550-562: same store, same pose, same time gate): one 32-byte-per-surfel stream instead of two.  The index map is
    // resolved after this kernel and read by pass 2 only.  A surfel that is drawn into the index map but needs no window (x or y exactly
    // 0, time gate at equality) is finished by pass 2 as well (flag bit 31): its confidence must not change before the resolve reads it.
    // candidates are staged per block in shared memory and flushed in chunks: one device-wide atomic per ~2k candidates
    // (a warp-aggregated global append put ~130k returning atomics on ONE L2 address)
    // ... and, round 2, per WARP: a warp owns CAND_BUF / 8 slots, appends with a ballot and flushes on its own (one device-wide atomic
    // per ~220 candidates, coalesced 128-byte copies): no block barrier in the streaming loop (two per round stall it
    // when every surfel of a dense map is a candidate).  The order of the list is irrelevant to pass 2.
    __shared__ uint32_t sBuf[8][CAND_BUF / 8];
    P.tinv = dpose->tinv;
    const uint32_t count = *countPtr;
    const uint32_t total = count + (uint32_t)Ppix;
    const float cols = (float)P.W, rows = (float)P.H, ftime = (float)P.time;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t staged = 0;                                                 // warp-uniform: entries waiting in this warp's slots
    auto flush = [&]() {
        uint32_t gbase = 0;
        if (lane == 0) gbase = atomicAdd(candCount, staged);
        gbase = __shfl_sync(0xffffffffu, gbase, 0);
        for (uint32_t i = lane; i < staged; i += 32) cand[gbase + i] = sBuf[warp][i];
        __syncwarp();
        staged = 0;
    };
    // the next round's two planes stream in behind this round's arithmetic and block-wide staging (two barriers per round exposed the
    // full DRAM latency of every round otherwise)
    const uint32_t stride = gridDim.x * blockDim.x;
    float4 vpN = make_float4(0, 0, 0, 0), vcN = vpN;
    { const uint32_t e0 = blockIdx.x * blockDim.x + threadIdx.x; if (e0 < count) { vpN = pos[e0]; vcN = col[e0]; } }
    for (uint32_t base = blockIdx.x * blockDim.x; base < total; base += stride) {
        const uint32_t e = base + threadIdx.x;
        bool valid = false, need = false, noWindow = false;
        const bool isOld = e < count;
        float4 vp = vpN, vc = vcN;
        if (e + stride < count) { vpN = pos[e + stride]; vcN = col[e + stride]; }
        if (isOld) valid = true;
        else if (e < total) { uint32_t p = e - count; if (aflag[p] == 2) { vp = m0[p]; vc = m1[p]; valid = true; } }
        if (valid) {
            float3 lp = xform(P.tinv, make_float3(vp.x, vp.y, vp.z));
            float x = ((P.cam.fx * lp.x) / lp.z) + P.cam.cx;
            float y = ((P.cam.fy * lp.y) / lp.z) + P.cam.cy;
            need = ftime - vc.w < P.ftimeDelta && lp.z > 0 && x > 0 && y > 0 && x < cols && y < rows;
            if (indexKey && isOld && !(lp.z > indexMaxDepth || lp.z <= 0 || ftime - vc.w > P.ftimeDelta)) {      // k_index_project, verbatim
                const float zn = lp.z / indexMaxDepth;
                const float fx_ = floorf(x), fy_ = floorf(y);
                if (zn < 1.0f && fx_ >= 0 && fy_ >= 0 && fx_ < cols && fy_ < rows) {
                    const unsigned long long k = ((unsigned long long)__float_as_uint(zn) << 32) | e;
                    unsigned long long* dst = indexKey + ((int)fy_ * P.W + (int)fx_);
                    if (k < *dst) atomicMin(dst, k);
                    if (!need) { need = true; noWindow = true; }
                }
            }
            if (!need) {
                const float w0 = vp.w, t0 = vc.w;
                bool k = cleanFinish(vp, vc, x, y, lp.z, 0, 0, P, depthFilt, mask);
                if (isOld) { if (vp.w != w0) pos[e].w = vp.w; if (vc.w != t0) col[e].w = vc.w; }
                else { uint32_t p = e - count; m0[p].w = vp.w; m1[p].w = vc.w; }
                keep[e] = k ? 1 : 0;
            }
        } else if (e < total) keep[e] = 0;
        const unsigned nb = __ballot_sync(0xffffffffu, need);
        if (nb) {
            if (staged + 32 > CAND_BUF / 8) flush();                    // warp uniform
            if (need) sBuf[warp][staged + __popc(nb & ((1u << lane) - 1))] = noWindow ? (e | 0x80000000u) : e;
            staged += (uint32_t)__popc(nb);
            __syncwarp();
        }
    }
    if (staged) flush();
}

// clean, pass 1b: one thread per candidate: index-map window (copy_unstable.vert:86-113) + the rest of the shader
template <bool PACKED>
__global__ void __launch_bounds__(256, 4) k_clean_p2(float4* __restrict__ pos, float4* __restrict__ col, const float4* __restrict__ nrm,
                                                  const uint32_t* __restrict__ countPtr, float4* __restrict__ m0, float4* __restrict__ m1,
                                                  const float4* __restrict__ m2, CleanParams P, const DevPose* __restrict__ dpose, CleanTexels cleanTex,
                                                  const float* __restrict__ depthFilt, const uint8_t* __restrict__ mask, uint8_t* __restrict__ keep,
                                                  const uint32_t* __restrict__ cand, const uint32_t* __restrict__ candCount)
{
    P.tinv = dpose->tinv;
    const uint32_t count = *countPtr, n = *candCount;
    const float cols = (float)P.W, rows = (float)P.H;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint32_t ce_ = cand[j];
        const bool noWindow = (ce_ >> 31) != 0;                        // drawn into the index map by pass 1 but outside the window's domain
        const uint32_t e = ce_ & 0x7fffffffu;
        const bool isOld = e < count;
        const uint32_t p = e - count;
        float4 vp, vc, vn;
        if (isOld) { vp = pos[e]; vc = col[e]; vn = nrm[e]; } else { vp = m0[p]; vc = m1[p]; vn = m2[p]; }
        const float w0 = vp.w, t0 = vc.w;
        float3 lp = xform(P.tinv, make_float3(vp.x, vp.y, vp.z));
        float x = ((P.cam.fx * lp.x) / lp.z) + P.cam.cx;
        float y = ((P.cam.fy * lp.y) / lp.z) + P.cam.cy;
        float3 ln = normalize3(rotate(P.tinv, make_float3(vn.x, vn.y, vn.z)));
        CleanEntry ce; ce.xn = x / cols; ce.yn = y / rows; ce.lx = lp.x; ce.ly = lp.y; ce.lz = lp.z; ce.init = vc.z; ce.rad = vn.w; ce.lnz = fabsf(ln.z);
        int c1 = 0, c2 = 0;
        if (!noWindow) cleanWindow<PACKED>(ce, P, cleanTex, c1, c2);
        bool k = cleanFinish(vp, vc, x, y, lp.z, c1, c2, P, depthFilt, mask);
        if (isOld) { if (vp.w != w0) pos[e].w = vp.w; if (vc.w != t0) col[e].w = vc.w; }
        else { m0[p].w = vp.w; m1[p].w = vc.w; }
        keep[e] = k ? 1 : 0;
    }
}

// per-512-element keep counts for the ordered compaction: one WARP per sub-block (16 flag bytes per lane, no block barriers;
// the block-per-sub-block version paid two barriers and a serial 16-term sum per 512 flags)
__global__ void __launch_bounds__(256) k_keep_block_sums(const uint8_t* __restrict__ keep, const uint32_t* __restrict__ countPtr, int Ppix,
                                                         uint32_t* __restrict__ blockSums, uint32_t* __restrict__ candCount, uint32_t* __restrict__ ticket)
{
    const uint32_t total = *countPtr + (uint32_t)Ppix;
    const uint32_t nblk = (total + SCAN_BLOCK - 1) / SCAN_BLOCK;
    if (blockIdx.x == 0 && threadIdx.x == 0) { *candCount = 0; *ticket = 0; }       // self-cleaning: ready for the next clean / the compaction below
    const uint32_t lane = threadIdx.x & 31, gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t blk = gw; blk < nblk; blk += nw) {
        const uint32_t e0 = blk * SCAN_BLOCK + lane * 16;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (e0 < total) v = *reinterpret_cast<const uint4*>(keep + e0);                           // flags are 0 / 1 bytes; the buffer is a multiple of 16 bytes
        if (e0 < total && total - e0 < 16) {                                                      // flags beyond `total` were never written
            const uint32_t r = total - e0;
            uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) { const uint32_t lo = (uint32_t)q * 4; w[q] = r <= lo ? 0u : (r - lo >= 4 ? w[q] : (w[q] & ((1u << (8 * (r - lo))) - 1u))); }
            v = make_uint4(w[0], w[1], w[2], w[3]);
        }
        uint32_t c = __popc(v.x & 0x01010101u) + __popc(v.y & 0x01010101u) + __popc(v.z & 0x01010101u) + __popc(v.w & 0x01010101u);
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) c += __shfl_xor_sync(0xffffffffu, c, off);
        if (lane == 0) blockSums[blk] = c;
    }
}

// pass 2: exclusive scan of the block sums (single block: every thread owns a run of consecutive sums, the 1024 run totals are
// scanned with shuffles) -> block offsets, new count, and the first sub-block that holds a removal (everything before it stays in place)
__global__ void __launch_bounds__(1024) k_scan_block_sums(uint32_t* __restrict__ blockSums, const uint32_t* __restrict__ countPtr,
                                                          int extra, uint32_t capacity, uint32_t* __restrict__ newCount, uint32_t* __restrict__ firstMoved)
{
    const uint32_t total = *countPtr + (uint32_t)extra;
    const uint32_t nblk = (total + SCAN_BLOCK - 1) / SCAN_BLOCK;
    __shared__ uint32_t wtot[32];
    __shared__ uint32_t sFirst;
    if (threadIdx.x == 0) sFirst = nblk;
    __syncthreads();
    const uint32_t per = (nblk + 1023) / 1024;
    const uint32_t b0 = threadIdx.x * per, b1 = min(b0 + per, nblk);
    uint32_t run = 0, first = 0xffffffffu;
    for (uint32_t i = b0; i < b1; ++i) { const uint32_t v = blockSums[i]; run += v; if (v != SCAN_BLOCK && first == 0xffffffffu) first = i; }
    if (first != 0xffffffffu) atomicMin(&sFirst, first);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = run;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= off) incl += t; }
    if (lane == 31) wtot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = wtot[lane], wi = w;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, wi, off); if (lane >= off) wi += t; }
        wtot[lane] = wi - w;                                         // exclusive prefix of the warp totals
        if (lane == 31) { *newCount = wi < capacity ? wi : capacity; }
    }
    __syncthreads();
    uint32_t offs = wtot[warp] + incl - run;
    for (uint32_t i = b0; i < b1; ++i) { const uint32_t v = blockSums[i]; blockSums[i] = offs; offs += v; }
    if (threadIdx.x == 0) { firstMoved[0] = sFirst; firstMoved[1] = nblk; }      // [1]: read back by the host for its in-place / ping-pong choice
}

// pass 3: ordered scatter of the survivors (old surfels in buffer order, then new vertices
// in x-major pixel order) into the other buffer
__global__ void __launch_bounds__(SCAN_BLOCK) k_clean_scatter(const float4* __restrict__ pos, const float4* __restrict__ col, const float4* __restrict__ nrm,
                                                              const uint32_t* __restrict__ countPtr, const float4* __restrict__ m0,
                                                              const float4* __restrict__ m1, const float4* __restrict__ m2, int Ppix,
                                                              const uint8_t* __restrict__ keep, const uint32_t* __restrict__ blockOffs,
                                                              uint32_t capacity, float4* __restrict__ opos, float4* __restrict__ ocol,
                                                              float4* __restrict__ onrm)
{
    const uint32_t count = *countPtr;
    const uint32_t total = count + (uint32_t)Ppix;
    const uint32_t nblk = (total + SCAN_BLOCK - 1) / SCAN_BLOCK;
    __shared__ uint32_t wsum[SCAN_BLOCK / 32];
    for (uint32_t blk = blockIdx.x; blk < nblk; blk += gridDim.x) {
        uint32_t e = blk * SCAN_BLOCK + threadIdx.x;
        bool k = e < total && keep[e];
        unsigned bal = __ballot_sync(0xffffffffu, k);
        int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        if (lane == 0) wsum[warp] = __popc(bal);
        __syncthreads();
        uint32_t woff = 0;
        for (int w = 0; w < warp; ++w) woff += wsum[w];
        uint32_t dst = blockOffs[blk] + woff + __popc(bal & ((1u << lane) - 1));
        if (k && dst < capacity) {
            float4 a, b, c;
            if (e < count) { a = ldStream(pos + e); b = ldStream(col + e); c = ldStream(nrm + e); }
            else { uint32_t p = e - count; a = m0[p]; b = m1[p]; c = m2[p]; }
            stStream(opos + dst, a); stStream(ocol + dst, b); stStream(onrm + dst, c);
        }
        __syncthreads();
    }
}

// pass 3, in place: Model::clean's ordered copy moves a survivor DOWN by the number of removals before it, so everything in front of
// the first removal already sits where it belongs: only the tail behind it is touched (the ping-pong copy above rewrites the whole
// store, 96 B per surfel, although removals concern the young surfels at its end).  Sub-blocks of 512 entries are handed out in
// ascending order by a ticket, starting at the first one that holds a removal.  A sub-block (1) loads its survivors into registers,
// (2) publishes `loaded[blk] = epoch` (release), (3) waits until the (at most two, lower) sub-blocks whose SOURCE range its
// destination range overlaps have published theirs, (4) stores.  Waits only ever point to lower tickets, whose owners are running
// and publish before they wait: no deadlock whatever the residency.  Same output order as the ping-pong copy, bit for bit.
__global__ void __launch_bounds__(SCAN_BLOCK) k_clean_compact(float4* __restrict__ pos, float4* __restrict__ col, float4* __restrict__ nrm,
                                                              const uint32_t* __restrict__ countPtr, const float4* __restrict__ m0,
                                                              const float4* __restrict__ m1, const float4* __restrict__ m2, int Ppix,
                                                              const uint8_t* __restrict__ keep, const uint32_t* __restrict__ blockOffs,
                                                              uint32_t capacity, uint32_t* __restrict__ ticket, uint32_t* __restrict__ loaded,
                                                              const uint32_t* __restrict__ firstMoved, uint32_t epoch)
{
    const uint32_t count = *countPtr;
    const uint32_t total = count + (uint32_t)Ppix;
    const uint32_t nblk = (total + SCAN_BLOCK - 1) / SCAN_BLOCK;
    const uint32_t first = *firstMoved;
    __shared__ uint32_t wsum[SCAN_BLOCK / 32];
    __shared__ uint32_t sBlk[2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // tickets are drawn one iteration ahead: the atomic's round trip hides behind the current sub-block's loads
    if (threadIdx.x == 0) sBlk[0] = first + atomicAdd(ticket, 1u);
    __syncthreads();
    for (uint32_t it = 0;; ++it) {
        const uint32_t blk = sBlk[it & 1];
        if (blk >= nblk) break;                                      // block uniform
        if (threadIdx.x == 0) sBlk[(it + 1) & 1] = first + atomicAdd(ticket, 1u);
        const uint32_t e = blk * SCAN_BLOCK + threadIdx.x;
        const bool k = e < total && keep[e];
        const unsigned bal = __ballot_sync(0xffffffffu, k);
        if (lane == 0) wsum[warp] = __popc(bal);
        __syncthreads();
        uint32_t woff = 0, nb = 0;
#pragma unroll
        for (int w = 0; w < SCAN_BLOCK / 32; ++w) { const uint32_t c = wsum[w]; if (w < warp) woff += c; nb += c; }
        const uint32_t off = blockOffs[blk];
        const uint32_t dst = off + woff + __popc(bal & ((1u << lane) - 1));
        const bool isOld = e < count;
        const bool move = k && dst < capacity && !(isOld && dst == e);
        float4 a = make_float4(0, 0, 0, 0), b = a, c = a;
        if (move) {
            if (isOld) { a = __ldcg(pos + e); b = __ldcg(col + e); c = __ldcg(nrm + e); }      // coherent loads: the planes are written by this very kernel
            else { const uint32_t p = e - count; a = m0[p]; b = m1[p]; c = m2[p]; }
        }
        // The barrier below CONSUMES the loaded words (a predicate no compiler can fold): no thread passes it before every load of the block
        // has returned its value, i.e. has been performed -- a later store to those addresses by another block cannot change what was read.
        // (A __threadfence per thread did the same job at several hundred cycles per iteration.)
        const unsigned probe = __float_as_uint(a.x) & __float_as_uint(b.y) & __float_as_uint(c.z);
        __syncthreads_or(probe == 0x7fedcba9u);
        if (threadIdx.x == 0) {
            asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(loaded + blk), "r"(epoch) : "memory");
            if (nb) {
                const uint32_t s0 = off / SCAN_BLOCK, s1 = (off + nb - 1) / SCAN_BLOCK;
                for (uint32_t s = s0; s <= s1 && s < blk; ++s) {
                    if (s < first) continue;                         // cannot happen (off >= first * 512); kept as a guard
                    unsigned v;
                    do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(loaded + s) : "memory"); } while (v != epoch);
                }
            }
        }
        __syncthreads();                                             // also: the next ticket (sBlk) is visible, wsum may be rewritten
        if (move) { stStream(pos + dst, a); stStream(col + dst, b); stStream(nrm + dst, c); }
    }
}

// ---------------------------------------------------------------------------------------
// splat prediction (combinedPredict) and model-ID projection
// ---------------------------------------------------------------------------------------
struct SplatVS { float3 pos; float conf; float3 n; float rad, size, xw, yw; bool ok; };

MF_D SplatVS splatVertex(float4 p, float4 c, float4 nr, const Rt& tinv, Cam cam, int W, int H, float maxDepth,
                         float confThreshold, float ftime, float fmaxTime, float ftimeDelta)
{
    SplatVS o; o.ok = false;
    float3 ph = xform(tinv, make_float3(p.x, p.y, p.z));
    if (ph.z > maxDepth || ph.z < 0 || p.w < confThreshold || ftime - c.w > ftimeDelta || c.w > fmaxTime) return o;
    o.pos = ph; o.conf = p.w;
    o.n = normalize3(rotate(tinv, make_float3(nr.x, nr.y, nr.z)));
    o.rad = nr.w;
    float3 x1 = normalize3(make_float3(o.n.y - o.n.z, -o.n.x, o.n.x));
    x1 = make_float3(x1.x * o.rad * 1.41421356f, x1.y * o.rad * 1.41421356f, x1.z * o.rad * 1.41421356f);
    float3 y1 = cross3(o.n, x1);
    float px[4], py[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        float3 d = (q == 0 || q == 3) ? x1 : y1;
        float sg = (q < 2) ? 1.0f : -1.0f;
        float3 pp = make_float3(ph.x + sg * d.x, ph.y + sg * d.y, ph.z + sg * d.z);
        px[q] = ((cam.fx * pp.x) / pp.z) + cam.cx;
        py[q] = ((cam.fy * pp.y) / pp.z) + cam.cy;
    }
    float xmin = fminf(px[0], fminf(px[1], fminf(px[2], px[3]))), xmax = fmaxf(px[0], fmaxf(px[1], fmaxf(px[2], px[3])));
    float ymin = fminf(py[0], fminf(py[1], fminf(py[2], py[3]))), ymax = fmaxf(py[0], fmaxf(py[1], fmaxf(py[2], py[3])));
    float sz = fmaxf(0.0f, fmaxf(fabsf(xmax - xmin), fabsf(ymax - ymin)));
    if (!(sz >= 1.0f)) sz = 1.0f;
    if (sz > MAX_POINT_SIZE) sz = MAX_POINT_SIZE;
    o.size = sz;
    o.xw = ((cam.fx * ph.x) / ph.z) + cam.cx;
    o.yw = ((cam.fy * ph.y) / ph.z) + cam.cy;
    if (!(o.xw >= 0 && o.xw <= (float)W && o.yw >= 0 && o.yw <= (float)H)) return o;
    if (!(ph.z / maxDepth <= 1.0f)) return o;
    o.ok = true;
    return o;
}

// viewing ray of the pixel centre (combo_splat.frag:39-45).  It depends on the camera alone: k_ray_table evaluates it once
// per context, the rasteriser reads it back (two IEEE divisions, a square root and three more divisions per FRAGMENT otherwise).
MF_D float3 pixelRay(Cam cam, float fcx, float fcy)
{
    return normalize3(make_float3((fcx - cam.cx) / cam.fx, (fcy - cam.cy) / cam.fy, 1.0f));
}
__global__ void k_ray_table(Cam cam, int W, int H, float4* __restrict__ tab)
{
    int px = blockIdx.x * blockDim.x + threadIdx.x, py = blockIdx.y * blockDim.y + threadIdx.y;
    if (px >= W || py >= H) return;
    float3 l = pixelRay(cam, (float)px + 0.5f, (float)py + 0.5f);
    tab[py * W + px] = make_float4(l.x, l.y, l.z, 0.f);
}

MF_D bool splatFragmentRay(const SplatVS& v, float3 l, float3& cp)
{
    float t = dot3(v.pos, v.n) / dot3(l, v.n);
    cp = make_float3(t * l.x, t * l.y, t * l.z);
    float sqrRad = v.rad * v.rad;
    float3 d = sub3(cp, v.pos);
    return !(dot3(d, d) > sqrRad);
}
MF_D bool splatFragment(const SplatVS& v, Cam cam, float fcx, float fcy, float3& cp) { return splatFragmentRay(v, pixelRay(cam, fcx, fcy), cp); }

MF_D void splatRange(const SplatVS& v, int W, int H, int& x0, int& x1, int& y0, int& y1)
{
    float h = v.size * 0.5f;
    float lo = ceilf(v.xw - h - 0.5f), hi = ceilf(v.xw + h - 0.5f) - 1.0f;
    x0 = lo < 0 ? 0 : (int)lo; x1 = hi > (float)(W - 1) ? W - 1 : (int)hi;
    lo = ceilf(v.yw - h - 0.5f); hi = ceilf(v.yw + h - 0.5f) - 1.0f;
    y0 = lo < 0 ? 0 : (int)lo; y1 = hi > (float)(H - 1) ? H - 1 : (int)hi;
}

#define SPLAT_SEG 8
#ifndef SPLAT_BS
#define SPLAT_BS 128               // surfels (= threads) per block round: smaller rounds interleave the load phase of one block with the raster phase of another
#endif
#ifndef SPLAT_MIN_BLOCKS
#define SPLAT_MIN_BLOCKS 8             // 56 registers, no spills; 9 blocks per SM fit.  Measured (k_splat_project, ms; H100 80GB HBM3, 400 W limit): 8 blocks
#endif                                 // 0.257; 12 (40 registers, 28 B of spills) 0.303; 16 (32 registers, 76 B; shared memory holds 13) 0.364;
                                       // SPLAT_BS 64 / 16 blocks 0.270; SPLAT_BS 256 / 4 blocks 0.286
#define SPLAT_Q 64                 // per-warp queue of exact-path fragments: a drain takes 32, so at most 31 + 32 are pending

// one drawable surfel of a round as the raster phase reads it; pn = dot3(pos, n) is the numerator of the ray parameter
struct __align__(16) SplatEntry { float px, py, pz, pn, nx, ny, nz, rad; int x0, y0, w; uint32_t id; };

// exact path of a fragment that passed the pre-tests (combo_splat.frag): IEEE ray parameter and disc test, depth range, and the
// (depth, id) key into the key image.  atomicMin does not depend on the order of the fragments.  A stale (larger) key from L1 only
// lets more fragments reach the atomic.
MF_D void splatExact(const SplatEntry& e, int pix, const float4* __restrict__ rayTab, unsigned long long* __restrict__ key, float maxDepth)
{
    SplatVS sv; sv.pos = make_float3(e.px, e.py, e.pz); sv.n = make_float3(e.nx, e.ny, e.nz); sv.rad = e.rad;
    const float4 l4 = __ldg(rayTab + pix);
    float3 cp;
    if (!splatFragmentRay(sv, make_float3(l4.x, l4.y, l4.z), cp)) return;
    const float fd = (cp.z / (2 * maxDepth)) + 0.5f;
    if (!(fd >= 0.0f && fd < 1.0f)) return;
    const unsigned long long k = ((unsigned long long)__float_as_uint(fd) << 32) | e.id;
    if (k < key[pix]) atomicMin(key + pix, k);
}

__global__ void __launch_bounds__(SPLAT_BS, SPLAT_MIN_BLOCKS) k_splat_project(const float4* __restrict__ pos, const float4* __restrict__ col, const float4* __restrict__ nrm,
                                                       const uint32_t* __restrict__ countPtr, const DevPose* __restrict__ dpose, Cam cam, int W, int H,
                                                       float maxDepth, float confThreshold, float ftime, float fmaxTime, float ftimeDelta,
                                                       uint32_t drawBase, const float4* __restrict__ rayTab, unsigned long long* __restrict__ key)
{
    // Row-segment rasterisation.  A block projects SPLAT_BS surfels per round and compacts the drawable ones into shared memory.
    // Their point sprites (1 .. 2047^2 pixels) are cut into UNITS of up to SPLAT_SEG consecutive pixels of one sprite row; the units
    // are numbered by an exclusive prefix sum and walked by all threads, unit u belonging to the entry found by binary search.
    // Balanced whatever the mix of far (1 px) and near (large) surfels; the search and the unit -> (row, x range) arithmetic are paid
    // once per SPLAT_SEG fragments, the pixel ray comes from the table.
    // With ~100 fragments per pixel almost every fragment loses the depth test or misses its disc.  The fragment loop only runs
    // conservative pre-tests in fast arithmetic; a fragment that can still win goes to a per-warp queue (pixel << 8 | entry slot),
    // and the warp drains 32 queued fragments at a time through the IEEE path (splatExact) with all lanes.  The divisions of that
    // path stay out of the loop, which then needs no local memory.
    // Rounds alternate between two entry / offset buffers: round r + 2 overwrites round r's buffer only after both barriers of
    // round r + 1, which every thread reaches after its raster of round r, so a round needs no barrier at its end.  The next
    // round's positions stream into shared memory (one bulk copy, completion on an mbarrier) behind this round's raster.
    constexpr int NW = SPLAT_BS / 32;
    static_assert(SPLAT_BS % 32 == 0 && SPLAT_BS <= 256, "the queue packs the entry slot into 8 bits");
    __shared__ SplatEntry ent[2][SPLAT_BS];
    __shared__ int offs[2][SPLAT_BS];
    __shared__ __align__(16) float4 spos[SPLAT_BS];
    __shared__ uint32_t queue[NW][SPLAT_Q];
    __shared__ int wtot[NW], wcnt[NW];
    __shared__ Rt tinv;
    __shared__ float inv2md;
    __shared__ __align__(8) unsigned long long bar;
    const uint32_t count = *countPtr;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t stride = gridDim.x * SPLAT_BS;
    const unsigned barAddr = (unsigned)__cvta_generic_to_shared(&bar);
    const unsigned sposAddr = (unsigned)__cvta_generic_to_shared(spos);
    // one bulk copy of the positions of the round starting at surfel b (16-byte aligned source, destination and size)
    auto fetch = [&](uint32_t b) {
        const unsigned bytes = min((uint32_t)SPLAT_BS, count - b) * 16u;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(barAddr), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(sposAddr), "l"(pos + b), "r"(bytes), "r"(barAddr) : "memory");
    };
    if (threadIdx.x < 12) tinv.m[threadIdx.x] = dpose->tinv.m[threadIdx.x];
    if (threadIdx.x == 0) {
        inv2md = 1.0f / (2 * maxDepth);
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(barAddr));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        if (blockIdx.x * SPLAT_BS < count) fetch(blockIdx.x * SPLAT_BS);
    }
    __syncthreads();
    unsigned parity = 0;
    for (uint32_t base = blockIdx.x * SPLAT_BS; base < count; base += stride, parity ^= 1u) {
        const uint32_t id = base + threadIdx.x;
        SplatVS v; v.ok = false;
        int x0 = 0, x1 = -1, y0 = 0, y1 = -1;
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "SPLAT_WAIT:\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
            "@!p bra SPLAT_WAIT;\n\t}" ::"r"(barAddr), "r"(parity) : "memory");
        if (id < count) {
            const float4 p = spos[threadIdx.x];
            // cheap rejects before touching the other two planes
            float3 ph = xform(tinv, make_float3(p.x, p.y, p.z));
            // ... including the point-clipping test on the projected centre (same arithmetic as splatVertex), which most
            // surfels of a large map fail: the basis / extent maths below then only runs for surfels inside the view
            const float cxw = ((cam.fx * ph.x) / ph.z) + cam.cx, cyw = ((cam.fy * ph.y) / ph.z) + cam.cy;
            if (!(ph.z > maxDepth || ph.z < 0 || p.w < confThreshold) && cxw >= 0 && cxw <= (float)W && cyw >= 0 && cyw <= (float)H) {
                float4 c = ldStream(col + id), nr = ldStream(nrm + id);
                v = splatVertex(p, c, nr, tinv, cam, W, H, maxDepth, confThreshold, ftime, fmaxTime, ftimeDelta);
                if (v.ok) splatRange(v, W, H, x0, x1, y0, y1);
            }
        }
        const bool draw = v.ok && x1 >= x0 && y1 >= y0;
        const int nunit = draw ? (y1 - y0 + 1) * ((x1 - x0 + SPLAT_SEG) / SPLAT_SEG) : 0;
        // block exclusive scans: unit offsets and compact slots
        int incl = nunit;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        unsigned db = __ballot_sync(0xffffffffu, draw);
        if (lane == 31) wtot[warp] = incl;
        if (lane == 0) wcnt[warp] = __popc(db);
        __syncthreads();
        // every thread has read its position: the next round's positions may overwrite them
        if (threadIdx.x == 0 && base + stride < count) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            fetch(base + stride);
        }
        SplatEntry* __restrict__ E = ent[parity];
        int* __restrict__ O = offs[parity];
        int fbase = 0, sbase = 0, total = 0, nent = 0;
#pragma unroll
        for (int w = 0; w < NW; ++w) { if (w < warp) { fbase += wtot[w]; sbase += wcnt[w]; } total += wtot[w]; nent += wcnt[w]; }
        if (draw) {
            const int slot = sbase + __popc(db & ((1u << lane) - 1));
            SplatEntry e; e.px = v.pos.x; e.py = v.pos.y; e.pz = v.pos.z; e.pn = dot3(v.pos, v.n); e.nx = v.n.x; e.ny = v.n.y; e.nz = v.n.z; e.rad = v.rad;
            e.x0 = x0; e.y0 = y0; e.w = x1 - x0 + 1; e.id = drawBase + id;
            E[slot] = e;
            O[slot] = fbase + incl - nunit;
        }
        __syncthreads();
        // gridDim.y > 1 (small stores): the blocks of a column redo the (cheap) vertex stage of the same surfels and share their units --
        // an object model has ~50 blocks' worth of surfels, and the units of a few large sprites kept one SM busy while the others idled
        uint32_t* __restrict__ q = queue[warp];
        int qn = 0;
        for (int ub = threadIdx.x - lane + blockIdx.y * SPLAT_BS; ub < total; ub += SPLAT_BS * gridDim.y) {
            const int u = ub + lane;
            int slot = 0, pix = 0, n = 0;
            if (u < total) {
                int lo = 0, hi = nent - 1;                       // last entry with offs[e] <= u
                while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (O[mid] <= u) lo = mid; else hi = mid - 1; }
                slot = lo;
                const int t = u - O[slot], w = E[slot].w, x0e = E[slot].x0;
                const int nseg = (w + SPLAT_SEG - 1) / SPLAT_SEG;
                const int row = t / nseg, xs = x0e + (t - row * nseg) * SPLAT_SEG;
                n = min(SPLAT_SEG, x0e + w - xs);
                pix = (E[slot].y0 + row) * W + xs;
            }
            const int nmax = __reduce_max_sync(0xffffffffu, n);
            for (int i = 0; i < nmax; ++i, ++pix) {
                bool cand = false;
                if (i < n) {
                    // Conservative pre-tests in fast arithmetic: an approximate ray parameter (error < 1e-6 relative, margins 10x larger)
                    // recognises the fragments that are clearly behind the current winner or clearly outside the disc.
                    const float4 pp = *reinterpret_cast<const float4*>(&E[slot].px), nr = *reinterpret_cast<const float4*>(&E[slot].nx);
                    const float4 l4 = __ldg(rayTab + pix);
                    const unsigned long long cur = key[pix];
                    const float ta = __fdividef(pp.w, dot3(make_float3(l4.x, l4.y, l4.z), make_float3(nr.x, nr.y, nr.z)));
                    cand = cur == KEY_EMPTY || !(__fmaf_rn(ta * l4.z, inv2md, 0.5f) > __uint_as_float((unsigned)(cur >> 32)) * 1.00001f);
                    if (cand) {
                        const float ax = __fmaf_rn(ta, l4.x, -pp.x), ay = __fmaf_rn(ta, l4.y, -pp.y), az = __fmaf_rn(ta, l4.z, -pp.z);
                        const float re = nr.w + 8e-6f * fabsf(ta);
                        cand = !(__fmaf_rn(ax, ax, __fmaf_rn(ay, ay, az * az)) > re * re * 1.0001f);
                    }
                }
                const unsigned m = __ballot_sync(0xffffffffu, cand);
                if (cand) q[qn + __popc(m & ((1u << lane) - 1))] = (uint32_t)pix << 8 | (uint32_t)slot;
                qn += __popc(m);
                if (qn >= 32) {
                    qn -= 32;
                    __syncwarp();
                    const uint32_t it = q[qn + lane];
                    __syncwarp();
                    splatExact(E[it & 255u], (int)(it >> 8), rayTab, key, maxDepth);
                }
            }
        }
        __syncwarp();
        if (lane < qn) {
            const uint32_t it = q[lane];
            splatExact(E[it & 255u], (int)(it >> 8), rayTab, key, maxDepth);
        }
    }
}

// resolve the winning surfel per pixel -> colour, vertex, normal, time; fill-in of holes
// from the raw frame (fill_*.frag) and the 1/20 sub-sampled "is the prediction mostly
// black" counter of MaskFusion::requiresFillIn are fused into the same pass.
__global__ void k_splat_resolve(const float4* __restrict__ pos, const float4* __restrict__ col, const float4* __restrict__ nrm,
                                const DevPose* __restrict__ dpose, Cam cam, int W, int H, float maxDepth, float confThreshold, float ftime, float fmaxTime,
                                float ftimeDelta, const float4* __restrict__ rayTab, unsigned long long* __restrict__ key,
                                uchar4* __restrict__ image, float4* __restrict__ vertexConf, float4* __restrict__ normalRad,
                                uint16_t* __restrict__ timeTex,
                                int doFill, const float* __restrict__ depthFilt, const uchar4* __restrict__ rgb, int ptVN, int ptImg,
                                uchar4* __restrict__ fillImage, float4* __restrict__ fillVertex, float4* __restrict__ fillNormal,
                                uint32_t* __restrict__ nonBlackSamples)
{
    const Rt tinv = dpose->tinv;
    int px = blockIdx.x * blockDim.x + threadIdx.x, py = blockIdx.y * blockDim.y + threadIdx.y;
    if (px >= W || py >= H) return;
    int i = py * W + px;
    unsigned long long k = key[i];
    uchar4 im = make_uchar4(0, 0, 0, 0);
    float4 vc = make_float4(0, 0, 0, 0), nr = vc;
    uint16_t tt = 0;
    if (k != KEY_EMPTY) {
        key[i] = KEY_EMPTY;
        uint32_t id = (uint32_t)(k & 0xffffffffull);
        float4 p = pos[id], c = col[id], n = nrm[id];
        SplatVS v = splatVertex(p, c, n, tinv, cam, W, H, maxDepth, confThreshold, ftime, fmaxTime, ftimeDelta);
        float3 cp; float fcx = (float)px + 0.5f, fcy = (float)py + 0.5f;
        const float4 l4 = __ldg(rayTab + i);
        splatFragmentRay(v, make_float3(l4.x, l4.y, l4.z), cp);
        float3 cl = decodeColor(c.x);
        im = make_uchar4((uint8_t)(int)floorf(cl.x * 255.0f + 0.5f), (uint8_t)(int)floorf(cl.y * 255.0f + 0.5f),
                         (uint8_t)(int)floorf(cl.z * 255.0f + 0.5f), 255);
        float z = cp.z;
        vc = make_float4((fcx - cam.cx) * z * (1.f / cam.fx), (fcy - cam.cy) * z * (1.f / cam.fy), z, v.conf);
        nr = make_float4(v.n.x, v.n.y, v.n.z, v.rad);
        tt = (uint16_t)(uint32_t)c.z;
    }
    image[i] = im; vertexConf[i] = vc; normalRad[i] = nr; timeTex[i] = tt;
    if (nonBlackSamples && (px % 20) == 10 && (py % 20) == 10 && px / 20 < W / 20 && py / 20 < H / 20) {
        if (im.x > 0 && im.y > 0 && im.z > 0) atomicAdd(nonBlackSamples, 1u);
    }
    if (doFill) {
        const float ifx = 1.0f / cam.fx, ify = 1.0f / cam.fy;
        float3 vp = getVertex(depthFilt, W, H, px, py, (float)px, (float)py, cam, ifx, ify);
        fillVertex[i] = (vc.z == 0 || ptVN) ? make_float4(vp.x, vp.y, vp.z, 1.f) : vc;
        if (nr.z == 0 || ptVN) {
            float3 n = normalForward(depthFilt, W, H, px, py, cam, ifx, ify, vp);
            fillNormal[i] = make_float4(n.x, n.y, n.z, 1.f);
        } else fillNormal[i] = nr;
        float sum = ((float)im.x / 255.0f + (float)im.y / 255.0f) + (float)im.z / 255.0f;
        fillImage[i] = (sum == 0 || ptImg) ? rgb[i] : im;
    }
}

// ---------------------------------------------------------------------------------------
// first-frame initialisation: two ordered streams (raw: position+colour, filtered:
// normal+radius) compacted in x-major order and paired by emission index.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SCAN_BLOCK) k_init_flags(const float* __restrict__ depthRaw, const float* __restrict__ depthFilt,
                                                           int W, int H, float maxDepth, uint8_t* __restrict__ fr, uint8_t* __restrict__ ff,
                                                           uint32_t* __restrict__ sumR, uint32_t* __restrict__ sumF)
{
    const int P = W * H;
    __shared__ uint32_t ws[2][SCAN_BLOCK / 32];
    int p = blockIdx.x * SCAN_BLOCK + threadIdx.x;
    bool kr = false, kf = false;
    if (p < P) {
        int i = p / H, j = p - i * H;
        float zr = depthRaw[j * W + i], zf = depthFilt[j * W + i];
        kr = !(zr <= 0 || zr > maxDepth);
        kf = !(zf <= 0 || zf > maxDepth);
        fr[p] = kr; ff[p] = kf;
    }
    unsigned br = __ballot_sync(0xffffffffu, kr), bf = __ballot_sync(0xffffffffu, kf);
    if ((threadIdx.x & 31) == 0) { ws[0][threadIdx.x >> 5] = __popc(br); ws[1][threadIdx.x >> 5] = __popc(bf); }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t a = 0, b = 0;
        for (int w = 0; w < SCAN_BLOCK / 32; ++w) { a += ws[0][w]; b += ws[1][w]; }
        sumR[blockIdx.x] = a; sumF[blockIdx.x] = b;
    }
}

__global__ void __launch_bounds__(SCAN_BLOCK) k_init_scatter(const uchar4* __restrict__ rgb, const float* __restrict__ depthRaw,
                                                             const float* __restrict__ depthFilt, Cam cam, int W, int H, int time,
                                                             const uint8_t* __restrict__ fr, const uint8_t* __restrict__ ff,
                                                             const uint32_t* __restrict__ offR, const uint32_t* __restrict__ offF,
                                                             uint32_t capacity, float4* __restrict__ pos, float4* __restrict__ col,
                                                             float4* __restrict__ nrm)
{
    const int P = W * H;
    __shared__ uint32_t ws[2][SCAN_BLOCK / 32];
    int p = blockIdx.x * SCAN_BLOCK + threadIdx.x;
    bool kr = p < P && fr[p], kf = p < P && ff[p];
    unsigned br = __ballot_sync(0xffffffffu, kr), bf = __ballot_sync(0xffffffffu, kf);
    int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { ws[0][warp] = __popc(br); ws[1][warp] = __popc(bf); }
    __syncthreads();
    uint32_t wr = 0, wf = 0;
    for (int w = 0; w < warp; ++w) { wr += ws[0][w]; wf += ws[1][w]; }
    if (p >= P) return;
    int i = p / H, j = p - i * H;
    const float ifx = 1.0f / cam.fx, ify = 1.0f / cam.fy;
    float tcx = (float)(((double)((float)i / (float)W)) + 1.0 / (double)(2 * (float)W));   // FeedbackBuffer.cpp:44-49
    float tcy = (float)(((double)((float)j / (float)H)) + 1.0 / (double)(2 * (float)H));
    float x = tcx * (float)W, y = tcy * (float)H;
    if (kr) {
        uint32_t dst = offR[blockIdx.x] + wr + __popc(br & ((1u << lane) - 1));
        if (dst < capacity) {
            float3 vp = getVertex(depthRaw, W, H, i, j, x, y, cam, ifx, ify);
            uchar4 c8 = rgb[j * W + i];
            pos[dst] = make_float4(vp.x, vp.y, vp.z, surfelConfidence(x, y, 1.0f, cam.cx, cam.cy));
            col[dst] = make_float4(encodeColor((float)c8.x / 255.0f, (float)c8.y / 255.0f, (float)c8.z / 255.0f), 0.f, 1.f, (float)time);
        }
    }
    if (kf) {
        uint32_t dst = offF[blockIdx.x] + wf + __popc(bf & ((1u << lane) - 1));
        if (dst < capacity) {
            float3 vp = getVertex(depthFilt, W, H, i, j, x, y, cam, ifx, ify);
            float3 nl = normalCentral(depthFilt, W, H, i, j, x, y, cam, ifx, ify, vp);
            nrm[dst] = make_float4(nl.x, nl.y, nl.z, surfelRadius(vp.z, nl.z, ifx, ify));
        }
    }
}

// generic exclusive scan of one array of block sums (used by the init path, 2 arrays)
__global__ void __launch_bounds__(1024) k_scan_small(uint32_t* __restrict__ a, int n, uint32_t capacity, uint32_t* __restrict__ total)
{
    __shared__ uint32_t sh[1024];
    __shared__ uint32_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        int i = base + threadIdx.x;
        uint32_t v = i < n ? a[i] : 0;
        sh[threadIdx.x] = v;
        __syncthreads();
        for (int off = 1; off < 1024; off <<= 1) {
            uint32_t t = threadIdx.x >= off ? sh[threadIdx.x - off] : 0;
            __syncthreads();
            sh[threadIdx.x] += t;
            __syncthreads();
        }
        uint32_t incl = sh[threadIdx.x];
        if (i < n) a[i] = carry + incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry += incl;
        __syncthreads();
    }
    if (threadIdx.x == 0 && total) *total = carry < capacity ? carry : capacity;
}

__global__ void k_fill_u32(uint32_t* p, uint32_t v, size_t n)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}
__global__ void k_fill_u64(unsigned long long* p, unsigned long long v, size_t n)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}
__global__ void k_zero_f4(float4* p, uint32_t from, uint32_t to)
{
    uint32_t i = from + blockIdx.x * blockDim.x + threadIdx.x;
    if (i < to) p[i] = make_float4(0, 0, 0, 0);
}

// AoS (12 floats) <-> planes, for the C-ABI download/upload (Model::downloadMap layout)
__global__ void k_planes_to_aos(const float4* __restrict__ pos, const float4* __restrict__ col, const float4* __restrict__ nrm, uint32_t n, float4* __restrict__ out)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[(size_t)i * 3] = pos[i]; out[(size_t)i * 3 + 1] = col[i]; out[(size_t)i * 3 + 2] = nrm[i];
}
__global__ void k_aos_to_planes(const float4* __restrict__ in, uint32_t n, float4* __restrict__ pos, float4* __restrict__ col, float4* __restrict__ nrm)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    pos[i] = in[(size_t)i * 3]; col[i] = in[(size_t)i * 3 + 1]; nrm[i] = in[(size_t)i * 3 + 2];
}

// ------------------------------ host launchers ----------------------------------------
int num_sms()
{
    static PerDevice<int> sms([](int dev) {
        int n = 0;
        cudaCheck(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev), "cudaDeviceGetAttribute");
        return n;
    });
    return sms.get();
}
static inline int persistentBlocks(int perSM) { return num_sms() * perSM; }

// host-driven pose (constructor, overridePose, updateStaticPose, C-ABI set_pose) -> device-resident DevPose; matrices by value
struct Pose2 { float p[16], l[16]; };
__global__ void k_set_pose(DevPose* d, Pose2 in)
{
    if (threadIdx.x == 0 && blockIdx.x == 0) derivePose(d, in.p, in.l);
}
void launch_set_pose(DevPose* d, const float* pose16, const float* lastPose16, Enq q)
{
    Pose2 in;
    for (int k = 0; k < 16; ++k) { in.p[k] = pose16[k]; in.l[k] = lastPose16[k]; }
    launch(q, nullptr, k_set_pose, 1, 32, 0, d, in);
}

void launch_fill_u32(uint32_t* p, uint32_t v, size_t n, Enq q) { if (n) launch(q, nullptr, k_fill_u32, (unsigned)((n + 255) / 256), 256, 0, p, v, n); }
void launch_fill_u64(uint64_t* p, uint64_t v, size_t n, Enq q) { if (n) launch(q, nullptr, k_fill_u64, (unsigned)((n + 255) / 256), 256, 0, (unsigned long long*)p, v, n); }

void launch_predict_indices(const SurfelPlanes& sp, const uint32_t* count, const DevPose* tinv, Cam cam, int W, int H, float maxDepth, int time,
                            int timeDelta, uint64_t* key, uint32_t* idx, float4* vertConf, float4* colorTime, float4* normRad, float4* cleanTex, float cleanConf, Enq q)
{
    launch(q, "k_index_project", k_index_project, persistentBlocks(8), 256, 0, sp.pos, sp.col, count, tinv, cam, W, H, maxDepth, (float)time, (float)timeDelta,
           (unsigned long long*)key);
    int P = W * H;
    launch(q, "k_index_resolve", k_index_resolve, (P + 255) / 256, 256, 0, sp.pos, sp.col, sp.nrm, tinv, P, (unsigned long long*)key, idx, vertConf, colorTime, normRad, cleanTex, cleanConf, (float)time);
}

void launch_associate(const uchar4* rgb, const float* depthRaw, const float* depthFilt, const uint8_t* mask, const uint32_t* idx,
                      const float4* vertConf, const float4* normRad, const DevPose* pose, Cam cam, int W, int H, float maxDepth, int time,
                      float weighting, uint8_t maskID, uint8_t* flag, uint32_t* best, float4* const* meas, uint32_t* slot, Enq q)
{
    dim3 b(32, 8), g((W + 31) / 32, (H + 7) / 8);
    launch(q, "k_associate", k_associate, g, b, 0, rgb, depthRaw, depthFilt, mask, idx, vertConf, normRad, pose, cam, W, H, maxDepth, time, weighting, maskID,
           flag, best, meas[0], meas[1], meas[2], slot);
}

void launch_fuse_update(const uint8_t* flag, const uint32_t* best, float4* const* meas, uint32_t* slot, int P, int time,
                        const SurfelPlanes& sp, Enq q)
{
    launch(q, "k_fuse_update", k_fuse_update, (P + 255) / 256, 256, 0, flag, best, meas[0], meas[1], meas[2], slot, P, time, sp.pos, sp.col, sp.nrm);
    launch(q, "k_slot_release", k_slot_release, (P + 255) / 256, 256, 0, flag, best, P, slot);
}

void launch_clean(const SurfelPlanes& src, const SurfelPlanes& dst, const uint32_t* count, uint32_t* newCount, uint32_t capacity,
                  const uint8_t* aflag, float4* const* meas, const DevPose* tinv, Cam cam, int W, int H, int time, int timeDelta, float confThreshold,
                  float outlierCoeff, uint8_t maskID, const CleanWindowImages& win,
                  const float* depthFilt, const uint8_t* mask, uint8_t* keep, uint32_t* blockSums, uint32_t* cand, uint32_t* candCount, Enq q,
                  const CleanInPlace& inplace, const IndexFused* fused)
{
    const CleanTexels texels{win.packed, win.vertConf, win.colorTime, win.idx};
    CleanParams P;
    P.tinv = Rt{};                          // filled from the device-resident pose inside the kernels
    P.cam = cam; P.W = W; P.H = H; P.time = time; P.ftimeDelta = (float)timeDelta; P.confThreshold = confThreshold;
    P.outlierCoeff = outlierCoeff; P.maskID = maskID;
    int Ppix = W * H;
    int blocks = persistentBlocks(4);
    launch(q, "k_clean_p1", k_clean_p1, persistentBlocks(8), 256, 0, src.pos, src.col, count, aflag, meas[0], meas[1], Ppix, P, tinv, depthFilt, mask, keep, cand, candCount,
           fused ? (unsigned long long*)fused->key : nullptr, fused ? fused->maxDepth : 0.f);
    if (fused) {           // Model::predictIndices, second half: the index map of the store as clean sees it
        launch(q, "k_index_resolve", k_index_resolve, (Ppix + 255) / 256, 256, 0, src.pos, src.col, src.nrm, tinv, Ppix, (unsigned long long*)fused->key, fused->idx,
               fused->vertConf, fused->colorTime, fused->normRad, fused->cleanTex, confThreshold, (float)time);
    }
    launch(q, "k_clean_p2", texels.packed ? k_clean_p2<true> : k_clean_p2<false>, persistentBlocks(8), 256, 0, src.pos, src.col, src.nrm, count, meas[0], meas[1], meas[2],
           P, tinv, texels, depthFilt, mask, keep, cand, candCount);
    launch(q, "k_keep_block_sums", k_keep_block_sums, persistentBlocks(8), 256, 0, keep, count, Ppix, blockSums, candCount, inplace.ticket);
    launch(q, "k_scan_block_sums", k_scan_block_sums, 1, 1024, 0, blockSums, count, Ppix, capacity, newCount, inplace.firstMoved);
    if (!inplace.pingPong) {
        launch(q, "k_clean_compact", k_clean_compact, blocks, SCAN_BLOCK, 0, src.pos, src.col, src.nrm, count, meas[0], meas[1], meas[2], Ppix, keep, blockSums, capacity,
               inplace.ticket, inplace.loaded, inplace.firstMoved, inplace.epoch);
    } else {
        launch(q, "k_clean_scatter", k_clean_scatter, blocks, SCAN_BLOCK, 0, src.pos, src.col, src.nrm, count, meas[0], meas[1], meas[2], Ppix, keep, blockSums, capacity,
               dst.pos, dst.col, dst.nrm);
    }
}

void launch_ray_table(Cam cam, int W, int H, float4* tab, Enq q)
{
    dim3 b(32, 8), g((W + 31) / 32, (H + 7) / 8);
    launch(q, nullptr, k_ray_table, g, b, 0, cam, W, H, tab);
}

// grid of the splat rasteriser: for large stores a persistent grid of as many blocks as the SMs hold at once; for a small store (an object
// model: a few thousand surfels) one column of blocks per SPLAT_BS surfels of CAPACITY is cheap to over-provision, and 8 blocks share the
// units of each column (gridDim.y)
static dim3 splatGrid(uint32_t capacity, int W, int H)
{
    if ((size_t)W * H > (1u << 24)) throw CudaError{"splat rasteriser: more than 2^24 pixels (its exact-path queue keeps 24-bit pixel indices)"};
    static PerDevice<int> perSM([](int) {
        int n = 0;
        cudaCheck(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_splat_project, SPLAT_BS, 0), "k_splat_project occupancy");
        if (n < 1) throw CudaError{"k_splat_project does not fit on an SM"};
        return n;
    });
    const int persistent = persistentBlocks(perSM.get());
    if (capacity == 0 || capacity >= (1u << 20)) return dim3(persistent);
    const int cols = (int)std::min<uint32_t>((capacity + SPLAT_BS - 1) / SPLAT_BS, (uint32_t)persistent);
    return dim3(cols, 8);
}
void launch_combined_predict(const SurfelPlanes& sp, const uint32_t* count, const DevPose* tinv, Cam cam, int W, int H, float maxDepth,
                             float confThreshold, int time, int maxTime, int timeDelta, const float4* rayTab, uint64_t* key, uchar4* image, float4* vertexConf,
                             float4* normalRad, uint16_t* timeTex, int doFill, const float* depthFilt, const uchar4* rgb, int ptVN, int ptImg,
                             uchar4* fillImage, float4* fillVertex, float4* fillNormal, uint32_t* nonBlackSamples, Enq q, uint32_t capacity)
{
    launch(q, "k_splat_project", k_splat_project, splatGrid(capacity, W, H), SPLAT_BS, 0, sp.pos, sp.col, sp.nrm, count, tinv, cam, W, H, maxDepth, confThreshold, (float)time,
           (float)maxTime, (float)timeDelta, 0u, rayTab, (unsigned long long*)key);
    if (nonBlackSamples) cudaMemsetAsync(nonBlackSamples, 0, sizeof(uint32_t), q.s);
    dim3 b(32, 8), g((W + 31) / 32, (H + 7) / 8);
    launch(q, "k_splat_resolve", k_splat_resolve, g, b, 0, sp.pos, sp.col, sp.nrm, tinv, cam, W, H, maxDepth, confThreshold, (float)time, (float)maxTime,
           (float)timeDelta, rayTab, (unsigned long long*)key, image, vertexConf, normalRad, timeTex, doFill, depthFilt, rgb,
           ptVN, ptImg, fillImage, fillVertex, fillNormal, nonBlackSamples);
}

void launch_init_model(const uchar4* rgb, const float* depthRaw, const float* depthFilt, Cam cam, int W, int H, int time, float maxDepth,
                       uint8_t* fr, uint8_t* ff, uint32_t* sumR, uint32_t* sumF, uint32_t capacity, const SurfelPlanes& sp, uint32_t* count,
                       Enq q)
{
    int P = W * H, nb = (P + SCAN_BLOCK - 1) / SCAN_BLOCK;
    launch(q, "k_zero_f4", k_zero_f4, (P + 255) / 256, 256, 0, sp.nrm, 0, (uint32_t)(P < (int)capacity ? P : (int)capacity));
    launch(q, "k_init_flags", k_init_flags, nb, SCAN_BLOCK, 0, depthRaw, depthFilt, W, H, maxDepth, fr, ff, sumR, sumF);
    launch(q, "k_scan_small", k_scan_small, 1, 1024, 0, sumR, nb, capacity, count);
    launch(q, "k_scan_small", k_scan_small, 1, 1024, 0, sumF, nb, capacity, nullptr);
    launch(q, "k_init_scatter", k_init_scatter, nb, SCAN_BLOCK, 0, rgb, depthRaw, depthFilt, cam, W, H, time, fr, ff, sumR, sumF, capacity, sp.pos, sp.col, sp.nrm);
}

void launch_planes_to_aos(const SurfelPlanes& sp, uint32_t n, float4* out, Enq q) { if (n) launch(q, nullptr, k_planes_to_aos, (n + 255) / 256, 256, 0, sp.pos, sp.col, sp.nrm, n, out); }
void launch_aos_to_planes(const float4* in, uint32_t n, const SurfelPlanes& sp, Enq q) { if (n) launch(q, nullptr, k_aos_to_planes, (n + 255) / 256, 256, 0, in, n, sp.pos, sp.col, sp.nrm); }

}  // namespace mfb

namespace mfb {
// splat projection into a caller-owned key image (GlobalProjection: all models share one key image)
void launch_splat_project_only(const SurfelPlanes& sp, const uint32_t* count, const DevPose* tinv, Cam cam, int W, int H, float maxDepth, float confThreshold,
                               int time, int maxTime, int timeDelta, uint32_t drawBase, const float4* rayTab, uint64_t* key, Enq q, uint32_t capacity)
{
    launch(q, "k_splat_project_ids", k_splat_project, splatGrid(capacity, W, H), SPLAT_BS, 0, sp.pos, sp.col, sp.nrm, count, tinv, cam, W, H, maxDepth, confThreshold,
           (float)time, (float)maxTime, (float)timeDelta, drawBase, rayTab, (unsigned long long*)key);
}
}  // namespace mfb
