// mf_frame.cu -- per-frame preprocessing kernels (sm_90a):
//   depth bilateral filter        <- Core/Shaders/depth_bilateral_metric.frag:30-76 (MaskFusion::filterDepth)
//   depth / intensity pyramids    <- Core/Cuda/cudafuncs.cu:333-364, 534-564
//   vertex + normal maps (fused)  <- Core/Cuda/cudafuncs.cu:109-189 (Model::generateCUDATextures, Model.cpp:350-389)
//   intensity, Sobel, clouds      <- Core/Cuda/cudafuncs.cu:602-751
//   model-map preparation (fused) <- RGBDOdometry::initICPModel, RGBDOdometry.cpp:153-185
// Layout: maps are float4 per pixel (x,y,z,0), invalid == NaN in x (reference: planar
// 3*rows x cols, NaN in the x plane); all loads are 16-byte, coalesced along rows.
#include "mf_common.cuh"
#include "mf_kernels.h"
#include "mf_host.h"

namespace mfb {

__global__ void k_unpack_rgb(const uint8_t* __restrict__ rgb3, uchar4* __restrict__ out, int P)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    out[i] = make_uchar4(rgb3[i * 3], rgb3[i * 3 + 1], rgb3[i * 3 + 2], 255);
}

// 13x13 bilateral, one thread per pixel, (32+12)x(8+12) depth tile staged in shared memory.
// Accumulation order (cy outer, cx inner, ascending) is part of the parity contract.
#define BIL_R 6
#define BIL_BX 32
#define BIL_BY 8
#define BIL_BW (BIL_BX + 16)             // 48 floats per staged row
#define BIL_XO 2                         // the halo's first column sits at index 2 of the staged row (x0 = 32 bx - 6 = (32 bx - 8) + 2)
// the filter of one pixel from the staged tile: tile[ty][BIL_XO + tx] holds depth(x0 + tx, y0 + ty), zero outside the image
MF_D void bilateralPixel(const float (*tile)[BIL_BW], float* __restrict__ out, int W, int H, int x0, int y0)
{
    const int x = blockIdx.x * BIL_BX + threadIdx.x, y = blockIdx.y * BIL_BY + threadIdx.y;
    if (x >= W || y >= H) return;
    const float value = tile[threadIdx.y + BIL_R][BIL_XO + threadIdx.x + BIL_R];
    if (value <= 0.03f) { out[y * W + x] = 0.0f; return; }
    const float sigma_space2_inv_half = 0.024691358f, sigma_color2_inv_half = 555.556f;
    const int D = 2 * BIL_R + 1;
    const int tx = min(x - D / 2 + D, W), ty = min(y - D / 2 + D, H);
    float sum1 = 0.f, sum2 = 0.f;
    if (x >= BIL_R && y >= BIL_R && x + BIL_R < W && y + BIL_R < H) {
        // whole window inside the image (97 % of the pixels at 640x480): fixed trip counts, the row fully unrolled, the spatial term of a
        // tap a compile-time constant per column.  Same operations on the same operands in the same order as the general loop below
        // (dx, dy are small integers: (float)x - (float)cx == (float)(x - cx) exactly), so the result is the same bit pattern.
        for (int iy = 0; iy < D; ++iy) {
            const float dy = (float)(BIL_R - iy);
            const float dy2 = dy * dy;
            const float* row = &tile[threadIdx.y + iy][BIL_XO + threadIdx.x];
#pragma unroll
            for (int ix = 0; ix < D; ++ix) {
                const float tmp = row[ix];
                const float dx = (float)(BIL_R - ix);
                const float space2 = dx * dx + dy2;
                const float dc = value - tmp;
                const float color2 = dc * dc;
                const float weight = det_expf(-(space2 * sigma_space2_inv_half + color2 * sigma_color2_inv_half));
                sum1 += tmp * weight;
                sum2 += weight;
            }
        }
        out[y * W + x] = sum1 / sum2;
        return;
    }
    for (int cy = max(y - D / 2, 0); cy < ty; ++cy) {
        const float dy = (float)y - (float)cy;
        const float* row = tile[cy - y0] + BIL_XO;
        for (int cx = max(x - D / 2, 0); cx < tx; ++cx) {
            float tmp = row[cx - x0];
            float dx = (float)x - (float)cx;
            float space2 = dx * dx + dy * dy;
            float dc = value - tmp;
            float color2 = dc * dc;
            float weight = det_expf(-(space2 * sigma_space2_inv_half + color2 * sigma_color2_inv_half));
            sum1 += tmp * weight;
            sum2 += weight;
        }
    }
    out[y * W + x] = sum1 / sum2;
}

// The halo tile is staged by the bulk-copy engine.  One cp.async.bulk (global -> shared, completion on an mbarrier) per tile ROW: 20 rows of 48 floats, the 16-byte aligned superset
// [32 bx - 8, 32 bx + 40) of the 44 columns the filter reads (bulk copies need 16-byte aligned source, destination and size; the halo
// starts 6 pixels left of the block).  Rows above / below the image and the column ranges left / right of it are zero-filled by the
// threads themselves (disjoint shared-memory words: no proxy ordering needed); everything else arrives without a single load instruction
// or bounds branch in the kernel.  The descriptor-based 2-D tensor copy of round 2a (zero fill by the copy engine) trapped in this kernel;
// the descriptor-free form does the same job.  Needs 16-byte aligned rows: W % 4 == 0 and a 16-byte aligned image (launch_bilateral checks).
__global__ void __launch_bounds__(BIL_BX* BIL_BY) k_bilateral(const float* __restrict__ depth, float* __restrict__ out, int W, int H)
{
    __shared__ __align__(128) float tile[BIL_BY + 2 * BIL_R][BIL_BW];
    __shared__ __align__(8) unsigned long long bar;
    const int x0 = blockIdx.x * BIL_BX - BIL_R, y0 = blockIdx.y * BIL_BY - BIL_R;
    const int xs = blockIdx.x * BIL_BX - 8;                        // first staged column (may be negative)
    const int c0 = max(xs, 0), c1 = min(xs + BIL_BW, W);           // columns that exist in the image
    const int tid = threadIdx.y * BIL_BX + threadIdx.x;
    const unsigned barAddr = (unsigned)__cvta_generic_to_shared(&bar);
    const int r0 = max(y0, 0), r1 = min(y0 + BIL_BY + 2 * BIL_R, H);   // rows that exist
    const unsigned rowBytes = (unsigned)(c1 - c0) * 4u;
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(barAddr));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(barAddr), "r"(rowBytes * (unsigned)(r1 - r0)) : "memory");
    __syncthreads();                                               // the transaction count is armed before any copy can complete
    if (tid < BIL_BY + 2 * BIL_R) {
        const int gy = y0 + tid;
        if (gy >= r0 && gy < r1) {
            const unsigned dst = (unsigned)__cvta_generic_to_shared(&tile[tid][c0 - xs]);
            const float* src = depth + (size_t)gy * W + c0;
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(dst), "l"(src), "r"(rowBytes), "r"(barAddr) : "memory");
        }
    }
    // zero fill of what lies outside the image (words no copy writes)
    for (int t = tid; t < (BIL_BY + 2 * BIL_R) * BIL_BW; t += BIL_BX * BIL_BY) {
        const int ty = t / BIL_BW, tx = t - ty * BIL_BW;
        const int gx = xs + tx, gy = y0 + ty;
        if (gx < c0 || gx >= c1 || gy < r0 || gy >= r1) tile[ty][tx] = 0.0f;
    }
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "BILB_WAIT:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n\t"
        "@p bra BILB_DONE;\n\t"
        "bra BILB_WAIT;\n\t"
        "BILB_DONE:\n\t}" ::"r"(barAddr) : "memory");
    __syncthreads();                                               // the zero fill of the other threads
    bilateralPixel(tile, out, W, H, x0, y0);
}

__constant__ float c_gauss5[25] = {1, 4, 6, 4, 1, 4, 16, 24, 16, 4, 6, 24, 36, 24, 6, 4, 16, 24, 16, 4, 1, 4, 6, 4, 1};

// NaN-skipping 5x5 Gaussian decimation; window clamp excludes the last row/column and
// the weight sum is an int, exactly as the reference (rule N9).


// Two pyramid levels in ONE launch: a block owns a PY_TX x PY_TY tile of the coarse level; it first evaluates the (2*PY_TX+3) x
// (2*PY_TY+3) patch of the middle level that tile reads (same arithmetic as the single-level kernels, straight from the fine
// level), keeps it in shared memory, writes the part it owns, then decimates the patch.  Bit-identical outputs, half the launches
// (these images are 76 800 / 19 200 pixels: the launches, not the arithmetic, were the cost -- 8 of them per frame).
#define PY_TX 8                          // 8x8 coarse tiles: 600 blocks per 640x480 image, all resident at once (16x8: 150 blocks, one per SM, three serial patch rounds)
#define PY_TY 8
struct PyrF {
    typedef float T;
    static __device__ __forceinline__ bool ok(float v) { return !isnan(v); }
    static __device__ __forceinline__ float val(float v) { return v; }
    static __device__ __forceinline__ float fin(float sum, int count) { return sum / (float)count; }
};
struct PyrU8 {
    typedef uint8_t T;
    static __device__ __forceinline__ bool ok(uint8_t v) { return v > 0; }
    static __device__ __forceinline__ float val(uint8_t v) { return (float)v; }
    static __device__ __forceinline__ uint8_t fin(float sum, int count) { float r = sum / (float)count; return (r != r) ? 0 : (uint8_t)(int)r; }
};
template <typename TR, typename Src>
MF_D typename TR::T pyrPixel(Src src, int sw, int sh, int x, int y)
{
    const int D = 5;
    int tx = min(2 * x - D / 2 + D, sw - 1), ty = min(2 * y - D / 2 + D, sh - 1);
    float sum = 0; int count = 0;
    for (int cy = max(0, 2 * y - D / 2); cy < ty; ++cy)
        for (int cx = max(0, 2 * x - D / 2); cx < tx; ++cx) {
            typename TR::T v = src(cx, cy);
            if (TR::ok(v)) {
                float g = c_gauss5[(ty - cy - 1) * 5 + (tx - cx - 1)];
                sum += TR::val(v) * g;
                count = (int)((float)count + g);
            }
        }
    return TR::fin(sum, count);
}
template <typename TR>
MF_D void pyrdown2Body(const typename TR::T* __restrict__ src, int sw, int sh, typename TR::T* __restrict__ dst1, typename TR::T* __restrict__ dst2)
{
    typedef typename TR::T T;
    constexpr int MW = 2 * PY_TX + 3, MH = 2 * PY_TY + 3;
    __shared__ T mid[MH][MW + 1];
    const int w1 = sw / 2, h1 = sh / 2, w2 = w1 / 2, h2 = h1 / 2;
    const int X0 = blockIdx.x * PY_TX, Y0 = blockIdx.y * PY_TY;              // coarse tile origin
    const int mx0 = 2 * X0 - 2, my0 = 2 * Y0 - 2;                            // middle-level patch origin
    for (int t = threadIdx.x; t < MW * MH; t += blockDim.x) {
        const int py = t / MW, px = t - py * MW;
        const int x = mx0 + px, y = my0 + py;
        T v = T(0);
        if (x >= 0 && y >= 0 && x < w1 && y < h1) {
            v = pyrPixel<TR>([&](int cx, int cy) { return src[cy * sw + cx]; }, sw, sh, x, y);
            if (px >= 2 && px < 2 + 2 * PY_TX && py >= 2 && py < 2 + 2 * PY_TY) dst1[y * w1 + x] = v;      // owned part of the middle level
        }
        mid[py][px] = v;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < PY_TX * PY_TY; t += blockDim.x) {
        const int ly = t / PY_TX, lx = t - ly * PY_TX;
        const int x = X0 + lx, y = Y0 + ly;
        if (x < w2 && y < h2) dst2[y * w2 + x] = pyrPixel<TR>([&](int cx, int cy) { return mid[cy - my0][cx - mx0]; }, w1, h1, x, y);
    }
}
template <typename TR>
__global__ void __launch_bounds__(256) k_pyrdown2(const typename TR::T* __restrict__ src, int sw, int sh, typename TR::T* __restrict__ dst1,
                                                  typename TR::T* __restrict__ dst2)
{
    pyrdown2Body<TR>(src, sw, sh, dst1, dst2);
}
// depth (float) and intensity (u8) pyramids of the same image size in one launch: blockIdx.z picks the image
__global__ void __launch_bounds__(256) k_pyrdown2_pair(const float* __restrict__ srcF, float* __restrict__ dstF1, float* __restrict__ dstF2,
                                                       const uint8_t* __restrict__ srcU, uint8_t* __restrict__ dstU1, uint8_t* __restrict__ dstU2, int sw, int sh)
{
    if (blockIdx.z == 0) pyrdown2Body<PyrF>(srcF, sw, sh, dstF1, dstF2);
    else pyrdown2Body<PyrU8>(srcU, sw, sh, dstU1, dstU2);
}

// three pyramid levels of one per-pixel kernel in a single launch: blockIdx.z = level
struct Maps3 { const float* depth[3]; float4* vmap[3]; float4* nmap[3]; float4* cloud[3]; const uint8_t* img[3]; short2* grad[3]; uint8_t* valid[3]; float minScale[3]; };

// depth -> vertex map + forward-difference normal map in ONE pass (the three vertices a
// normal needs are rebuilt from depth; saves the vmap round trip through HBM).
MF_D void vmapNmapPixel(const float* __restrict__ depth, int W, int H, Cam cam, float cutoff, float4* __restrict__ vmap, float4* __restrict__ nmap, int u, int v);
__global__ void k_vmap_nmap3(Maps3 m, int W0, int H0, Cam cam0, float cutoff)
{
    const int l = blockIdx.z, W = W0 >> l, H = H0 >> l;
    int u = blockIdx.x * blockDim.x + threadIdx.x, v = blockIdx.y * blockDim.y + threadIdx.y;
    if (u >= W || v >= H) return;
    vmapNmapPixel(m.depth[l], W, H, camLevel(cam0, l), cutoff, m.vmap[l], m.nmap[l], u, v);
}
MF_D void vmapNmapPixel(const float* __restrict__ depth, int W, int H, Cam cam, float cutoff, float4* __restrict__ vmap, float4* __restrict__ nmap, int u, int v)
{
    const float fx_inv = 1.f / cam.fx, fy_inv = 1.f / cam.fy;
    auto vert = [&](int uu, int vv, float3& o) -> bool {
        float z = depth[vv * W + uu];
        if (z > 0.0f && z < cutoff) {
            o = make_float3(z * ((float)uu - cam.cx) * fx_inv, z * ((float)vv - cam.cy) * fy_inv, z);
            return true;
        }
        return false;
    };
    float3 v00, v01, v10;
    bool ok00 = vert(u, v, v00);
    vmap[v * W + u] = ok00 ? make_float4(v00.x, v00.y, v00.z, 0.f) : make_float4(qnanf(), 0.f, 0.f, 0.f);
    float4 n = make_float4(qnanf(), 0.f, 0.f, 0.f);
    if (ok00 && u != W - 1 && v != H - 1 && vert(u + 1, v, v01) && vert(u, v + 1, v10)) {
        float3 c = cross3(sub3(v01, v00), sub3(v10, v00));
        float len = sqrtf((c.x * c.x + c.y * c.y) + c.z * c.z);
        n = make_float4(c.x / len, c.y / len, c.z / len, 0.f);
    }
    nmap[v * W + u] = n;
}

__global__ void k_intensity(const uchar4* __restrict__ img, int P, uint8_t* __restrict__ out)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    uchar4 s = img[i];
    float v = ((float)s.x * 0.114f + (float)s.y * 0.299f) + (float)s.z * 0.587f;   // cudafuncs.cu:634
    out[i] = (uint8_t)(int)v;
}

// model-side intensity: source image picked on the device like k_model_maps (Model::initICP, Model.cpp:391-409)
__global__ void k_intensity_select(const uchar4* __restrict__ imgPred, const uchar4* __restrict__ imgFill, const uint32_t* __restrict__ nonBlack,
                                   float denom, int forceFill, int P, uint8_t* __restrict__ out)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const bool fill = forceFill || (nonBlack && ((float)(*nonBlack) / denom < 0.75f));
    uchar4 s = fill ? imgFill[i] : imgPred[i];
    float v = ((float)s.x * 0.114f + (float)s.y * 0.299f) + (float)s.z * 0.587f;
    out[i] = (uint8_t)(int)v;
}

__constant__ float c_sobx[9] = {0.52201f, 0.00000f, -0.52201f, 0.79451f, -0.00000f, -0.79451f, 0.52201f, 0.00000f, -0.52201f};
__constant__ float c_soby[9] = {0.52201f, 0.79451f, 0.52201f, 0.00000f, 0.00000f, 0.00000f, -0.52201f, -0.79451f, -0.52201f};
// + the pose-independent half of residualKernel (reduce.cu:821-845): a pixel can enter the photometric term only if its 4x4
// neighbourhood of intensities is non-zero and its own gradient magnitude passes the level's gate.  Frame-side, shared by all
// models and all Gauss-Newton iterations (the tracker used to re-derive it per model per level).
MF_D void sobelPixel(const uint8_t* __restrict__ src, int W, int H, short2* __restrict__ grad, float minScale, uint8_t* __restrict__ rgbValid, int x, int y);
__global__ void k_sobel3(Maps3 m, int W0, int H0)
{
    const int l = blockIdx.z, W = W0 >> l, H = H0 >> l;
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H) return;
    sobelPixel(m.img[l], W, H, m.grad[l], m.minScale[l], m.valid[l], x, y);
}
MF_D void sobelPixel(const uint8_t* __restrict__ src, int W, int H, short2* __restrict__ grad, float minScale, uint8_t* __restrict__ rgbValid, int x, int y)
{
    float dxv = 0, dyv = 0; int k = 8;
    for (int j = max(y - 1, 0); j <= min(y + 1, H - 1); ++j)
        for (int i = max(x - 1, 0); i <= min(x + 1, W - 1); ++i) {
            float s = (float)src[j * W + i];
            dxv += s * c_sobx[k];
            dyv += s * c_soby[k];
            --k;
        }
    const short2 g = make_short2((short)(int)dxv, (short)(int)dyv);
    grad[y * W + x] = g;
    bool valid = false;
    if (x < W - 5 && y < H - 1) {
        valid = true;
        for (int u = max(y - 2, 0); u < min(y + 2, H); ++u)
            for (int v = max(x - 2, 0); v < min(x + 2, W); ++v) valid = valid && (src[u * W + v] > 0);
        if (valid) {
            float mTwo = (float)(((int)g.x * (int)g.x) + ((int)g.y * (int)g.y));
            valid = mTwo >= minScale;
        }
    }
    rgbValid[y * W + x] = valid ? 1 : 0;
}

// ---- model-map preparation ------------------------------------------------------------
// One thread per level-1 pixel; the four threads of a level-2 pixel sit in adjacent lanes.
// Each thread reads its 2x2 block of the predicted (or fill-in) RGBA32F maps and emits
// level 0 (x4), level 1 and -- by quad shuffle -- level 2 of the transformed model maps,
// plus the level-0 depth used by the photometric term (verticesToDepth).
// Arithmetic order follows copyMaps -> resizeMap x2 -> tranformMaps of the reference.
struct V3 { float x, y, z; bool ok; };
MF_D float4 packv(float3 v, bool ok) { return ok ? make_float4(v.x, v.y, v.z, 0.f) : make_float4(qnanf(), qnanf(), qnanf(), 0.f); }

__global__ void k_model_maps(const float4* __restrict__ srcV_pred, const float4* __restrict__ srcN_pred,
                             const float4* __restrict__ srcV_fill, const float4* __restrict__ srcN_fill,
                             const uint32_t* __restrict__ nonBlack, float denom, int W, int H, const DevPose* __restrict__ dpose, float maxDepthRGB,
                             float4* __restrict__ v0, float4* __restrict__ n0, float4* __restrict__ v1, float4* __restrict__ n1,
                             float4* __restrict__ v2, float4* __restrict__ n2, float* __restrict__ depth0)
{
    const Rt pose = dpose->pose;
    const int W1 = W / 2, H1 = H / 2, W2 = W / 4, H2 = H / 4;
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    int q = t >> 2, sub = t & 3;
    bool active = q < W2 * H2;
    int qx = active ? q % W2 : 0, qy = active ? q / W2 : 0;
    int x1 = 2 * qx + (sub & 1), y1 = 2 * qy + (sub >> 1);
    // MaskFusion::requiresFillIn (MaskFusion.cpp:630-648) evaluated on the device: no host round trip
    const bool fill = nonBlack && ((float)(*nonBlack) / denom < 0.75f);
    const float4* srcV = fill ? srcV_fill : srcV_pred;
    const float4* srcN = fill ? srcN_fill : srcN_pred;
    float3 sv = make_float3(0, 0, 0), sn = make_float3(0, 0, 0);
    bool bad = false;
    if (active) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            int x = 2 * x1 + (k & 1), y = 2 * y1 + (k >> 1);
            float4 a = srcV[y * W + x], b = srcN[y * W + x];
            bool ok = !(a.z == 0.0f);
            float3 vv = make_float3(a.x, a.y, a.z), nn = make_float3(b.x, b.y, b.z);
            // level 0: copyMaps + tranformMaps (a NaN normal inside a valid vertex stays NaN)
            bool nok = ok && !isnan(nn.x);
            bool vok = ok && !isnan(vv.x);
            v0[y * W + x] = packv(xform(pose, vv), vok);
            n0[y * W + x] = packv(rotate(pose, nn), nok);
            depth0[y * W + x] = (a.z > maxDepthRGB || a.z <= 0) ? qnanf() : a.z;      // cudafuncs.cu:602-613
            bad = bad || !vok || !nok;
            // ((a+b)+c)+d accumulation order of resizeMapKernel
            sv = (k == 0) ? vv : add3(sv, vv);
            sn = (k == 0) ? nn : add3(sn, nn);
        }
    }
    // NOTE: vertex and normal validity coincide (both derive from vsrc.z != 0) except for NaN
    // normals stored inside valid vertices; the reference tests each map's own x plane.
    float3 a1v = make_float3(sv.x / 4, sv.y / 4, sv.z / 4);
    float3 a1n = make_float3(sn.x / 4, sn.y / 4, sn.z / 4);
    bool badV = bad, badN = bad;
    if (active) {
        // recompute exact per-map validity
        badV = false; badN = false;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            int x = 2 * x1 + (k & 1), y = 2 * y1 + (k >> 1);
            float4 a = srcV[y * W + x], b = srcN[y * W + x];
            bool ok = !(a.z == 0.0f);
            badV = badV || !ok || isnan(a.x);
            badN = badN || !ok || isnan(b.x);
        }
    }
    float3 a1nn = normalize3(a1n);
    if (active) {
        v1[y1 * W1 + x1] = packv(xform(pose, a1v), !badV);
        n1[y1 * W1 + x1] = packv(rotate(pose, a1nn), !badN);
    }
    // level 2: average of the four (untransformed) level-1 values held by the quad's lanes
    const unsigned full = 0xffffffffu;
    int base = (threadIdx.x & 31) & ~3;
    float3 s2v, s2n; bool b2v = false, b2n = false;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        float3 pv = make_float3(__shfl_sync(full, a1v.x, base + k), __shfl_sync(full, a1v.y, base + k), __shfl_sync(full, a1v.z, base + k));
        float3 pn = make_float3(__shfl_sync(full, a1nn.x, base + k), __shfl_sync(full, a1nn.y, base + k), __shfl_sync(full, a1nn.z, base + k));
        b2v = b2v || __shfl_sync(full, (int)badV, base + k);
        b2n = b2n || __shfl_sync(full, (int)badN, base + k);
        s2v = (k == 0) ? pv : add3(s2v, pv);
        s2n = (k == 0) ? pn : add3(s2n, pn);
    }
    if (active && sub == 0) {
        float3 a2v = make_float3(s2v.x / 4, s2v.y / 4, s2v.z / 4);
        float3 a2n = normalize3(make_float3(s2n.x / 4, s2n.y / 4, s2n.z / 4));
        v2[qy * W2 + qx] = packv(xform(pose, a2v), !b2v);
        n2[qy * W2 + qx] = packv(rotate(pose, a2n), !b2n);
    }
}

// float4 map -> reference planar layout (for read-back through the C ABI)
__global__ void k_map_to_planar(const float4* __restrict__ m, int P, float* __restrict__ out)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    float4 v = m[i];
    out[i] = v.x; out[P + i] = v.y; out[2 * P + i] = v.z;
}

__global__ void k_project_points3(Maps3 m, int W0, int H0, Cam cam0)
{
    const int l = blockIdx.z, W = W0 >> l, H = H0 >> l;
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H) return;
    const Cam cam = camLevel(cam0, l);
    float z = m.depth[l][y * W + x];
    float ifx = 1.0f / cam.fx, ify = 1.0f / cam.fy;
    // .w: the 1.0 / cloudPoint.z of rgbKernel (reduce.cu:574, a double-precision reciprocal rounded to float), which depends on the map alone:
    // evaluated here once per frame instead of once per photometric row in each of the 19 Gauss-Newton iterations
    m.cloud[l][y * W + x] = make_float4(((float)x - cam.cx) * z * ifx, ((float)y - cam.cy) * z * ify, z, (float)(1.0 / (double)z));
}

// ------------------------------ host launchers ----------------------------------------
static inline dim3 grid2(int w, int h, dim3 b) { return dim3((w + b.x - 1) / b.x, (h + b.y - 1) / b.y); }

void launch_unpack_rgb(const uint8_t* rgb3, uchar4* out, int P, Enq q) { launch(q, nullptr, k_unpack_rgb, (P + 255) / 256, 256, 0, rgb3, out, P); }
void launch_bilateral(const float* depth, float* out, int W, int H, Enq q)
{
    // the bulk copies need 16-byte aligned rows (MaskFusion rejects W % 4 != 0; the raw depth sits 16-byte aligned in its frame buffer)
    if (W % 4 != 0 || ((uintptr_t)depth & 15) != 0) throw CudaError{"bilateral filter: depth rows must be 16-byte aligned (W % 4 == 0, aligned image)"};
    dim3 b(BIL_BX, BIL_BY);
    launch(q, "k_bilateral", k_bilateral, grid2(W, H, b), b, 0, depth, out, W, H);
}
void launch_pyrdown2_f(const float* src, int sw, int sh, float* dst1, float* dst2, Enq q)
{
    dim3 g((sw / 4 + PY_TX - 1) / PY_TX, (sh / 4 + PY_TY - 1) / PY_TY);
    launch(q, "k_pyrdown2_f", k_pyrdown2<PyrF>, g, 256, 0, src, sw, sh, dst1, dst2);
}
void launch_pyrdown2_pair(const float* srcF, float* dstF1, float* dstF2, const uint8_t* srcU, uint8_t* dstU1, uint8_t* dstU2, int sw, int sh, Enq q)
{
    dim3 g((sw / 4 + PY_TX - 1) / PY_TX, (sh / 4 + PY_TY - 1) / PY_TY, 2);
    launch(q, "k_pyrdown2_pair", k_pyrdown2_pair, g, 256, 0, srcF, dstF1, dstF2, srcU, dstU1, dstU2, sw, sh);
}
void launch_pyrdown2_u8(const uint8_t* src, int sw, int sh, uint8_t* dst1, uint8_t* dst2, Enq q)
{
    dim3 g((sw / 4 + PY_TX - 1) / PY_TX, (sh / 4 + PY_TY - 1) / PY_TY);
    launch(q, "k_pyrdown2_u8", k_pyrdown2<PyrU8>, g, 256, 0, src, sw, sh, dst1, dst2);
}
void launch_vmap_nmap3(const float* const* depth, int W, int H, Cam cam, float cutoff, float4* const* vmap, float4* const* nmap, Enq q)
{
    Maps3 m = {};
    for (int l = 0; l < 3; ++l) { m.depth[l] = depth[l]; m.vmap[l] = vmap[l]; m.nmap[l] = nmap[l]; }
    dim3 b(32, 8), g = grid2(W, H, b); g.z = 3;
    launch(q, "k_vmap_nmap3", k_vmap_nmap3, g, b, 0, m, W, H, cam, cutoff);
}
void launch_sobel3(const uint8_t* const* img, int W, int H, short2* const* grad, uint8_t* const* rgbValid, Enq q)
{
    Maps3 m = {};
    for (int l = 0; l < 3; ++l) { m.img[l] = img[l]; m.grad[l] = grad[l]; m.valid[l] = rgbValid[l]; m.minScale[l] = track_min_scale(l); }
    dim3 b(32, 8), g = grid2(W, H, b); g.z = 3;
    launch(q, "k_sobel3", k_sobel3, g, b, 0, m, W, H);
}
void launch_project_points3(const float* const* depth, int W, int H, Cam cam, float4* const* cloud, Enq q)
{
    Maps3 m = {};
    for (int l = 0; l < 3; ++l) { m.depth[l] = depth[l]; m.cloud[l] = cloud[l]; }
    dim3 b(32, 8), g = grid2(W, H, b); g.z = 3;
    launch(q, "k_project_points3", k_project_points3, g, b, 0, m, W, H, cam);
}
void launch_intensity(const uchar4* img, int P, uint8_t* out, Enq q) { launch(q, nullptr, k_intensity, (P + 255) / 256, 256, 0, img, P, out); }
void launch_intensity_select(const uchar4* imgPred, const uchar4* imgFill, const uint32_t* nonBlack, float denom, int forceFill, int P, uint8_t* out, Enq q)
{
    launch(q, "k_intensity_select", k_intensity_select, (P + 255) / 256, 256, 0, imgPred, imgFill, nonBlack, denom, forceFill, P, out);
}
void launch_model_maps(const float4* srcVp, const float4* srcNp, const float4* srcVf, const float4* srcNf, const uint32_t* nonBlack, float denom,
                       int W, int H, const DevPose* pose, float maxDepthRGB, float4* const* v, float4* const* n, float* depth0, Enq q)
{
    int threads = (W / 4) * (H / 4) * 4;
    launch(q, "k_model_maps", k_model_maps, (threads + 127) / 128, 128, 0, srcVp, srcNp, srcVf, srcNf, nonBlack, denom, W, H, pose, maxDepthRGB,
           v[0], n[0], v[1], n[1], v[2], n[2], depth0);
}
// validity bitmask of a model's normal maps, three levels in one launch (blockIdx.y = level): the tracker tests the bit of the pixel a
// frame vertex projects to BEFORE gathering the model vertex / normal there.  An object model covers a few per cent of the image, so
// nearly every projection of a frame pixel lands on an invalid texel: the ICP correspondence test (reduce.cu:330-360) would reject it on
// isnan(normal) after two 16-byte gathers; the bit says the same thing from shared memory.
__global__ void k_valid_bits3(const float4* __restrict__ n0, const float4* __restrict__ n1, const float4* __restrict__ n2, int N0,
                              uint32_t* __restrict__ b0, uint32_t* __restrict__ b1, uint32_t* __restrict__ b2)
{
    const int l = blockIdx.y;
    const float4* n = l == 0 ? n0 : l == 1 ? n1 : n2;
    uint32_t* b = l == 0 ? b0 : l == 1 ? b1 : b2;
    const int N = N0 >> (2 * l);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if ((i & ~31) >= N) return;
    const bool ok = i < N && !isnan(n[i].x);
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if ((threadIdx.x & 31) == 0) b[i >> 5] = m;
}
void launch_valid_bits3(const float4* const* nmap, int W, int H, uint32_t* const* bits, Enq q)
{
    const int N0 = W * H;
    dim3 g((N0 + 255) / 256, 3);
    launch(q, "k_valid_bits3", k_valid_bits3, g, 256, 0, nmap[0], nmap[1], nmap[2], N0, bits[0], bits[1], bits[2]);
}
void launch_map_to_planar(const float4* m, int P, float* out, Enq q) { launch(q, nullptr, k_map_to_planar, (P + 255) / 256, 256, 0, m, P, out); }

}  // namespace mfb
