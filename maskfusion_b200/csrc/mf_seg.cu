// mf_seg.cu -- geometric depth-edge segmentation kernels (sm_90a)
//   edge-ness (concavity + distance) <- computeGeometricSegmentation_Kernel, Core/Cuda/segmentation.cu:122-177
//   threshold / invert               <- segmentation.cu:257-269
//   binary close                     <- dilate_Kernel / erode_Kernel, segmentation.cu:217-255, host :334-354
// Edge-ness and threshold are fused (one pass over the level-0 tracking maps, which is what
// the reference feeds it: MfSegmentation.cpp:149-151, REUSE_FILTERED_MAPS).
#include "mf_common.cuh"
#include "mf_kernels.h"
#include "mf_host.h"
#include <math.h>
#include <stdlib.h>

namespace mfb {

__global__ void k_geometric_edges(const float4* __restrict__ vmap, const float4* __restrict__ nmap, int W, int H, float wD, float wC,
                                  float thr, float* __restrict__ edge, uint8_t* __restrict__ binary)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H) return;
    float e = 1.0f;
    if (!(x < 1 || x >= W - 1 || y < 1 || y >= H - 1)) {
        float4 v4 = vmap[y * W + x], n4 = nmap[y * W + x];
        float3 v = make_float3(v4.x, v4.y, v4.z), n = make_float3(n4.x, n4.y, n4.z);
        if (!(v.z <= 0.0f)) {
            float c = 0.0f, d = 0.0f;
            const int ox[8] = {-1, 0, 1, -1, 1, -1, 0, 1}, oy[8] = {-1, -1, -1, 0, 0, 1, 1, 1};
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                float4 a = vmap[(y + oy[k]) * W + x + ox[k]], b = nmap[(y + oy[k]) * W + x + ox[k]];
                float3 dd = make_float3(a.x - v.x, a.y - v.y, a.z - v.z);
                float dn = dot3(dd, n);
                float ct = (dn < 0) ? 0.0f : 1 - dot3(make_float3(b.x, b.y, b.z), n);
                c = fmaxf(ct, c);
                d = fmaxf(fabsf(dn), d);
            }
            c = fmaxf(c, 0.0f);
            c *= wC; d *= wD;
            e = fminf(1.0f, c > d ? c : d);
        }
    }
    edge[y * W + x] = e;
    binary[y * W + x] = e > thr ? 255 : 0;
}

__global__ void k_morph(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int W, int H, int r, int dilate)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H) return;
    int x1 = max(x - r, 0), y1 = max(y - r, 0), x2 = min(x + r, W - 1), y2 = min(y + r, H - 1);
    uint8_t res = dilate ? 0 : 255;
    for (int cy = y1; cy <= y2; ++cy)
        for (int cx = x1; cx <= x2; ++cx) {
            if (cy == y && cx == x) continue;
            uint8_t v = in[cy * W + cx];
            if (dilate && v == 255) res = 255;
            if (!dilate && v == 0) res = 0;
        }
    out[y * W + x] = res;
}
__global__ void k_invert(const uint8_t* __restrict__ in, int n, uint8_t* __restrict__ out)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (uint8_t)(255 - in[i]);
}

// gray-level dilate / erode with OpenCV's elliptic structuring element (cv::getStructuringElement(MORPH_ELLIPSE, (2r+1)^2)):
// row dy of the element spans columns -hw[dy+r] .. +hw[dy+r]; taps outside the image are ignored (morphologyDefaultBorderValue).
// One step of cv::morphologyEx(MORPH_CLOSE) on the mask-id image (MfSegmentation.cpp:424-426).
struct EllipseRows { int r; int hw[33]; };
__global__ void k_morph_ellipse(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int W, int H, EllipseRows e, int dilate,
                                const FrameHdr* __restrict__ onlyIfMasks)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H) return;
    if (onlyIfMasks && onlyIfMasks->nMasks == 0) { out[y * W + x] = in[y * W + x]; return; }     // the reference closes only inside `if (nMasks)` (:420-426)
    int best = dilate ? 0 : 255;
    for (int dy = -e.r; dy <= e.r; ++dy) {
        const int yy = y + dy;
        if (yy < 0 || yy >= H) continue;
        const int hw = e.hw[dy + e.r];
        const int x1 = max(x - hw, 0), x2 = min(x + hw, W - 1);
        for (int xx = x1; xx <= x2; ++xx) {
            const int v = in[yy * W + xx];
            best = dilate ? max(best, v) : min(best, v);
        }
    }
    out[y * W + x] = (uint8_t)best;
}
// closes `data` in place (buf: scratch of the same size): dilate x iterations, then erode x iterations
void launch_morph_close_ellipse(uint8_t* data, uint8_t* buf, int W, int H, int radius, int iterations, const FrameHdr* onlyIfMasks, Enq q)
{
    if (iterations <= 0) return;
    if (radius < 0 || radius > 16) throw CudaError{"morphMaskRadius must be in 0..16"};
    EllipseRows e; e.r = radius;
    const double inv_r2 = radius ? 1.0 / ((double)radius * radius) : 0.0;
    for (int i = 0; i < 2 * radius + 1; ++i) {
        const int dy = i - radius;
        e.hw[i] = (int)lrint(radius * sqrt((double)(radius * radius - dy * dy) * inv_r2));     // cv::getStructuringElement, MORPH_ELLIPSE
    }
    dim3 b(32, 8), g((W + 31) / 32, (H + 7) / 8);
    uint8_t* src = data; uint8_t* dst = buf;
    for (int pass = 0; pass < 2; ++pass)
        for (int i = 0; i < iterations; ++i) {
            launch(q, "k_morph_ellipse", k_morph_ellipse, g, b, 0, src, dst, W, H, e, pass == 0, onlyIfMasks);
            uint8_t* t = src; src = dst; dst = t;
        }
    // an even number of passes: the result is back in `data`
}

void launch_geometric_edges(const float4* vmap, const float4* nmap, int W, int H, float wD, float wC, float thr, float* edge, uint8_t* binary, Enq q)
{
    dim3 b(32, 8), g((W + 31) / 32, (H + 7) / 8);
    launch(q, "k_geometric_edges", k_geometric_edges, g, b, 0, vmap, nmap, W, H, wD, wC, thr, edge, binary);
}
void launch_morph_close_invert(uint8_t* data, uint8_t* buf, int W, int H, int radius, int iterations, uint8_t* inverted, Enq q)
{
    dim3 b(32, 8), g((W + 31) / 32, (H + 7) / 8);
    for (int i = 0; i < iterations; ++i) {
        launch(q, "k_morph", k_morph, g, b, 0, data, buf, W, H, radius, 1);
        launch(q, "k_morph", k_morph, g, b, 0, buf, data, W, H, radius, 0);
    }
    launch(q, "k_invert", k_invert, (W * H + 255) / 256, 256, 0, data, W * H, inverted);
}

}  // namespace mfb

// =======================================================================================
// GPU replacement of the CPU tail of MfSegmentation::performSegmentation
// (Core/Segmentation/MfSegmentation.cpp:208-538; SURVEY 8(f)-2).  The reference downloads the
// edge mask and runs ~15 single-threaded full-image sweeps + OpenCV connected components; here
// the sweeps are kernels and only two tiny tables (per-mask pixel counts, mask x model overlaps)
// visit the host for the mask->model vote.
// Component numbering is arbitrary (atomic counter): the reference's results do not depend on it.
// =======================================================================================
namespace mfb {

// ---- 4-connected components: union-find with atomicMin (root = smallest pixel index) ----
MF_D int ccFind(const int* L, int x)       // (no __restrict__: L is being modified by other threads' atomics while we walk it)
{
    int p = L[x];
    while (p != x) { x = p; p = L[x]; }
    return x;
}
MF_D void ccUnion(int* L, int a, int b)
{
    while (true) {
        a = ccFind(L, a); b = ccFind(L, b);
        if (a == b) return;
        if (a < b) { int t = a; a = b; b = t; }        // a > b: hook the larger root under the smaller
        int old = atomicMin(&L[a], b);
        if (old == a) return;
        a = old;
    }
}
// Two-level union-find (a single global pass over all pixels hooks every root through L2 atomics):
//   k_cc_tile   : one 32x16 tile per CTA, union-find in SHARED memory over the tile's pixels (left / up neighbours inside the tile);
//                 every pixel leaves with the GLOBAL index of its tile-local root (roots are the smallest index, and local raster order is
//                 global raster order inside a tile, so the invariant "root = smallest pixel index of the set" holds for the global pass)
//   k_cc_border : only the pixels on a tile's left / top edge union with their neighbour across the edge, in global memory
#define CC_TW 32
#define CC_TH 16
__global__ void __launch_bounds__(CC_TW * CC_TH) k_cc_tile(const uint8_t* __restrict__ img, int W, int H, int* __restrict__ L, int* __restrict__ area, uint32_t* counter)
{
    __shared__ int sl[CC_TW * CC_TH];
    __shared__ uint8_t sf[CC_TW * CC_TH];
    const int tx = threadIdx.x & (CC_TW - 1), ty = threadIdx.x / CC_TW, t = threadIdx.x;
    const int x = blockIdx.x * CC_TW + tx, y = blockIdx.y * CC_TH + ty;
    const bool in = x < W && y < H;
    const int i = y * W + x;
    if (blockIdx.x == 0 && blockIdx.y == 0 && t == 0) *counter = 0;
    const uint8_t f = in ? img[i] : 0;
    sf[t] = f; sl[t] = t;
    __syncthreads();
    if (f) {
        if (tx > 0 && sf[t - 1]) ccUnion(sl, t, t - 1);
        if (ty > 0 && sf[t - CC_TW]) ccUnion(sl, t, t - CC_TW);
    }
    __syncthreads();
    if (in) {
        int r = -1;
        if (f) { const int lr = ccFind(sl, t); r = (blockIdx.y * CC_TH + lr / CC_TW) * W + blockIdx.x * CC_TW + (lr & (CC_TW - 1)); }
        L[i] = r;
        area[i] = 0;
    }
}
__global__ void k_cc_border(const uint8_t* __restrict__ img, int W, int H, int* L)
{
    // thread k < nV: a pixel on a vertical tile edge (column multiple of CC_TW); else one on a horizontal edge (row multiple of CC_TH)
    const int nCols = (W - 1) / CC_TW, nRows = (H - 1) / CC_TH;
    const int nV = nCols * H, nH = nRows * W;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < nV) {
        const int y = k / nCols, x = (k - y * nCols + 1) * CC_TW, i = y * W + x;
        if (img[i] && img[i - 1]) ccUnion(L, i, i - 1);
    } else if (k < nV + nH) {
        const int q = k - nV, r = q / W, x = q - r * W, y = (r + 1) * CC_TH, i = y * W + x;
        if (img[i] && img[i - W]) ccUnion(L, i, i - W);
    }
}
// roots get a dense id 1..n-1 (0 = background/edge); area is accumulated per dense id
__global__ void k_cc_number(int* __restrict__ L, int P, int* __restrict__ dense, uint32_t* counter, int* __restrict__ box)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    if (L[i] == i) {
        const int d = (int)atomicAdd(counter, 1u) + 1;
        dense[i] = d;
        box[4 * d] = 0x7fffffff; box[4 * d + 1] = 0x7fffffff; box[4 * d + 2] = -1; box[4 * d + 3] = -1;     // left, top, right, bottom of the component
    }
}
// Integer histogram update with one atomic per distinct bin per warp: neighbouring pixels mostly hit the same bin (one component /
// one model covers most of the image), and 300 k atomics on ONE address serialise (k_seg_hist, k_mask_overlap and this kernel were
// bound by them).  key < 0: this lane adds nothing.  All 32 lanes must call.  Sums of integers: order-free, results identical.
MF_D void warpAggAdd(int* __restrict__ bins, int key)
{
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    if (key >= 0 && (int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&bins[key], __popc(peers));
}
// labels + per-component area and bounding box (the `stats` of cv::connectedComponentsWithStats, MfSegmentation.cpp:239), one atomic per
// distinct component per warp
__global__ void k_cc_relabel(const int* __restrict__ L, const int* __restrict__ dense, int P, int W, int* __restrict__ lab, int* __restrict__ area,
                             int* __restrict__ box)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int l = 0, key = -1;
    if (i < P && L[i] >= 0) { l = dense[ccFind(L, i)]; key = l; }
    const int y = i / W, x = i - y * W;
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    const int mnx = __reduce_min_sync(peers, x), mxx = __reduce_max_sync(peers, x), mny = __reduce_min_sync(peers, y), mxy = __reduce_max_sync(peers, y);
    if (key >= 0 && (int)(threadIdx.x & 31) == __ffs(peers) - 1) {
        atomicAdd(&area[key], __popc(peers));
        atomicMin(&box[4 * key], mnx); atomicMin(&box[4 * key + 1], mny); atomicMax(&box[4 * key + 2], mxx); atomicMax(&box[4 * key + 3], mxy);
    }
    if (i < P) lab[i] = l;
}
// one Jacobi sweep of the edge-removal loop (MfSegmentation.cpp:243-291): reads the previous labels only
__global__ void k_remove_edges(const int* __restrict__ labIn, int* __restrict__ labOut, const float* __restrict__ depth,
                               const int* __restrict__ area, int W, int H)
{
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H) return;
    int i = y * W + x;
    int c = labIn[i];
    if (x >= 1 && x < W - 1 && y >= 1 && y < H - 1 && (c == 0 || area[c] < 50)) {
        float d = depth[i];
        const int oy[8] = {-1, -1, -1, 0, 0, 1, 1, 1}, ox[8] = {-1, 0, 1, -1, 1, -1, 0, 1};
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            int j = (y + oy[k]) * W + x + ox[k];
            int n = labIn[j];
            if (n != 0 && fabsf(depth[j] - d) < 0.008 && area[n] > 50) { c = n; break; }
        }
    }
    labOut[i] = c;
}
__global__ void k_seg_hist(const int* __restrict__ lab, const uint8_t* __restrict__ projID, const uint8_t* __restrict__ mask, int P,
                           const uint8_t* __restrict__ idToIndex, int nModels, const FrameHdr* __restrict__ hdr, int* __restrict__ compModel, int* __restrict__ compMask)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int nMasks = hdr->nMasks;
    const bool in = i < P;
    const int c = in ? lab[i] : 0;
    warpAggAdd(compModel, in ? c * nModels + (int)idToIndex[projID[i]] : -1);
    if (nMasks) warpAggAdd(compMask, in ? c * nMasks + (int)mask[i] : -1);
}
// the two component histograms are sized for the worst case (P/2 + 2 components x 64 models / 256 masks: memory is not the
// constraint: 0.6 GB at 1280x720 on an 80 GB part); only the rows this frame uses are cleared, the counts come from the device
__global__ void k_clear_hist(const uint32_t* __restrict__ ccCounter, const FrameHdr* __restrict__ hdr, int nModels, int* __restrict__ compModel, int* __restrict__ compMask)
{
    const size_t nC = (size_t)*ccCounter + 1, nA = nC * nModels, nB = nC * hdr->nMasks;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nA + nB; i += (size_t)gridDim.x * blockDim.x) {
        if (i < nA) compModel[i] = 0; else compMask[i - nA] = 0;
    }
}
__global__ void k_component_map(const uint32_t* __restrict__ ccCounter, const int* __restrict__ area, const int* __restrict__ compModel, const int* __restrict__ compMask,
                                int nModels, const FrameHdr* __restrict__ hdr, const uint8_t* __restrict__ indexToId, int minMappedComponentSize,
                                int* __restrict__ mapToMask, int* __restrict__ absorb, int* __restrict__ maskPixels)
{
    const int nComponents = (int)*ccCounter + 1, nMasks = hdr->nMasks;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < nComponents; c += gridDim.x * blockDim.x) {
        int m2m = 0, ab = 0;
        if (c >= 1) {
            int csize = area[c];
            if (nMasks && csize > minMappedComponentSize) {
                int t = (int)(0.65f * csize);
                for (int m = 1; m < nMasks; ++m)
                    if (compMask[(size_t)c * nMasks + m] > t) { m2m = m; atomicAdd(&maskPixels[m], csize); }
            }
            int best = compModel[(size_t)c * nModels], bi = 0;
            for (int m = 1; m < nModels; ++m) { int v = compModel[(size_t)c * nModels + m]; if (v > best) { best = v; bi = m; } }
            int id = indexToId[bi];
            if (id > 0 && best > 0.6f * csize) ab = id;
        }
        mapToMask[c] = m2m; absorb[c] = ab;
    }
}
// mask -> model vote of MfSegmentation.cpp:433-492 on the device (one thread: the "first new label wins" rule is sequential; the
// tables are <= 256 x 64 entries).  maskToID persists across frames like the member of the reference class.
__global__ void k_vote(const FrameHdr* __restrict__ hdr, VoteParams vp, const int* __restrict__ maskPixels, const unsigned* __restrict__ maskOverlap,
                       const uint32_t* __restrict__ ccCounter, uint8_t* __restrict__ maskToID, FrameResult* __restrict__ res)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const int nMasks = hdr->nMasks;
    int hasNew = 0, newClass = -1;
    if (nMasks) {
        for (int midx = 1; midx < nMasks; ++midx) { maskToID[midx] = 0; if (hdr->classIDs[midx] == vp.personClassID) maskToID[midx] = 255; }
        for (int midx = 1; midx < nMasks; ++midx) {
            if (maskToID[midx] == 255) continue;
            int bestModelIndex = 0; unsigned bestOverlap = 0;
            const int maskClassID = hdr->classIDs[midx];
            for (int j = 1; j < vp.nModels; ++j) { unsigned o = maskOverlap[(size_t)j * 256 + midx]; if (o > bestOverlap) { bestOverlap = o; bestModelIndex = j; } }
            const bool matches = vp.modelClass[bestModelIndex] == maskClassID;
            if (bestOverlap < vp.minMaskModelOverlap * maskPixels[midx]) bestModelIndex = 0;
            if (bestModelIndex != 0 && matches) maskToID[midx] = vp.modelID[bestModelIndex];
            else if (!hasNew && vp.allowNew && (unsigned)maskPixels[midx] > vp.minNew && (unsigned)maskPixels[midx] < vp.maxNew && bestModelIndex == 0) {
                maskToID[midx] = vp.nextModelID; hasNew = 1; newClass = maskClassID;
            } else maskToID[midx] = 255;
        }
    }
    res->hasNewLabel = hasNew; res->newClassID = newClass; res->nMasks = nMasks; res->nComponents = (int)*ccCounter + 1; res->timestamp = hdr->timestamp;
    res->detectError = hdr->detectError;
}
__global__ void k_seg_tables(SegTables t, uint8_t* __restrict__ idToIndex, uint8_t* __restrict__ indexToId, uint8_t* __restrict__ isModel)
{
    const int i = threadIdx.x;
    idToIndex[i] = t.idToIndex[i]; indexToId[i] = t.indexToId[i]; isModel[i] = t.isModel[i];
}
__global__ void k_frame_header(FrameHdr h, FrameHdr* __restrict__ d)
{
    const int i = threadIdx.x;
    if (i == 0) { d->timestamp = h.timestamp; d->nMasks = h.nMasks; d->detectError = 0; d->maskGiven = h.maskGiven; }
    d->classIDs[i] = h.classIDs[i];
}
__global__ void k_person_table(const FrameHdr* __restrict__ hdr, int personClassID, uint8_t* __restrict__ isPerson)
{
    const int i = threadIdx.x;
    isPerson[i] = (i < hdr->nMasks && hdr->classIDs[i] == personClassID) ? 1 : 0;
}
__global__ void k_seg_assign(const int* __restrict__ lab, const int* __restrict__ mapToMask, const uint8_t* __restrict__ ignore, int P,
                             uint8_t* __restrict__ seg)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    seg[i] = ignore[i] ? 255 : (uint8_t)mapToMask[lab[i]];
}
__global__ void k_mask_overlap(const uint8_t* __restrict__ seg, const uint8_t* __restrict__ projID, const uint8_t* __restrict__ idToIndex,
                               const uint8_t* __restrict__ isModelId, int P, unsigned* __restrict__ maskOverlap)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int key = -1;
    if (i < P) { uint8_t id = projID[i]; if (isModelId[id]) key = (int)idToIndex[id] * 256 + seg[i]; }
    warpAggAdd(reinterpret_cast<int*>(maskOverlap), key);
}
// maskToID lookup + "unused components are absorbed by the model they overlap" (MfSegmentation.cpp:495-522).  The reference relabels a
// component inside the rectangle [left, left + width] x [top, top + height] of its connected-components statistics, i.e. of the component
// BEFORE the edge-removal sweeps grew it: pixels the sweeps attached outside that rectangle keep their mask value.
__global__ void k_seg_final(const uint8_t* __restrict__ seg, const int* __restrict__ lab, const int* __restrict__ mapToMask,
                            const int* __restrict__ absorb, const uint8_t* __restrict__ maskToID, const int* __restrict__ box, int P, int W,
                            uint8_t* __restrict__ out)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    uint8_t s = maskToID[seg[i]];
    int c = lab[i];
    if (c > 0 && mapToMask[c] == 0 && absorb[c] > 0) {
        const int y = i / W, x = i - y * W;
        if (x >= box[4 * c] && x <= box[4 * c + 2] + 1 && y >= box[4 * c + 1] && y <= box[4 * c + 3] + 1) s = (uint8_t)absorb[c];
    }
    out[i] = s;
}
__global__ void k_apply_ignore(const uint8_t* __restrict__ mask, const uint8_t* __restrict__ isPerson, const FrameHdr* __restrict__ hdr, int P,
                               uint8_t* __restrict__ ignore, uint8_t* __restrict__ edges)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    if (hdr->nMasks) ignore[i] = isPerson[mask[i]] ? 255 : 0;
    if (ignore[i]) edges[i] = 0;
}
// model-ID image from the global-projection keys (GlobalProjection.cpp:43-111): low word = modelIndex << 26 | surfel id
__global__ void k_proj_resolve(unsigned long long* __restrict__ key, int P, const uint8_t* __restrict__ indexToId, uint8_t* __restrict__ out)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    unsigned long long k = key[i];
    uint8_t id = 0;
    if (k != KEY_EMPTY) { key[i] = KEY_EMPTY; id = indexToId[(uint32_t)(k & 0xffffffffull) >> 26]; }
    out[i] = id;
}

void launch_cc(const uint8_t* img, int W, int H, int* L, int* dense, int* lab, int* area, int* box, uint32_t* counter, Enq q)
{
    int P = W * H;
    dim3 gt((W + CC_TW - 1) / CC_TW, (H + CC_TH - 1) / CC_TH);
    launch(q, "k_cc_tile", k_cc_tile, gt, CC_TW * CC_TH, 0, img, W, H, L, area, counter);
    const int nEdge = ((W - 1) / CC_TW) * H + ((H - 1) / CC_TH) * W;
    if (nEdge > 0) launch(q, "k_cc_border", k_cc_border, (nEdge + 255) / 256, 256, 0, img, W, H, L);
    launch(q, "k_cc_number", k_cc_number, (P + 255) / 256, 256, 0, L, P, dense, counter, box);
    launch(q, "k_cc_relabel", k_cc_relabel, (P + 255) / 256, 256, 0, L, dense, P, W, lab, area, box);
}
void launch_remove_edges(int* labA, int* labB, const float* depth, const int* area, int W, int H, int iterations, Enq q)
{
    dim3 b(32, 8), g((W + 31) / 32, (H + 7) / 8);
    for (int i = 0; i < iterations; ++i) {          // caller guarantees an even ping-pong ends in labA when iterations is odd -> see host
        launch(q, "k_remove_edges", k_remove_edges, g, b, 0, i % 2 == 0 ? labA : labB, i % 2 == 0 ? labB : labA, depth, area, W, H);
    }
}
void launch_seg_hist(const int* lab, const uint8_t* projID, const uint8_t* mask, int P, const uint8_t* idToIndex, int nModels, const FrameHdr* hdr,
                     int* compModel, int* compMask, Enq q)
{
    launch(q, "k_seg_hist", k_seg_hist, (P + 255) / 256, 256, 0, lab, projID, mask, P, idToIndex, nModels, hdr, compModel, compMask);
}
void launch_clear_hist(const uint32_t* ccCounter, const FrameHdr* hdr, int nModels, int* compModel, int* compMask, Enq q)
{
    launch(q, "k_clear_hist", k_clear_hist, num_sms(), 256, 0, ccCounter, hdr, nModels, compModel, compMask);
}
void launch_component_map(const uint32_t* ccCounter, const int* area, const int* compModel, const int* compMask, int nModels, const FrameHdr* hdr,
                          const uint8_t* indexToId, int minMapped, int* mapToMask, int* absorb, int* maskPixels, Enq q)
{
    launch(q, "k_component_map", k_component_map, num_sms(), 128, 0, ccCounter, area, compModel, compMask, nModels, hdr, indexToId, minMapped, mapToMask, absorb, maskPixels);
}
void launch_vote(const FrameHdr* hdr, const VoteParams& vp, const int* maskPixels, const unsigned* maskOverlap, const uint32_t* ccCounter,
                 uint8_t* maskToID, FrameResult* res, Enq q)
{
    launch(q, "k_vote", k_vote, 1, 32, 0, hdr, vp, maskPixels, maskOverlap, ccCounter, maskToID, res);
}
void launch_seg_tables(const SegTables& t, uint8_t* idToIndex, uint8_t* indexToId, uint8_t* isModel, Enq q)
{
    launch(q, "k_seg_tables", k_seg_tables, 1, 256, 0, t, idToIndex, indexToId, isModel);
}
void launch_frame_header(const FrameHdr& h, FrameHdr* d, Enq q) { launch(q, "k_frame_header", k_frame_header, 1, 256, 0, h, d); }
void launch_person_table(const FrameHdr* hdr, int personClassID, uint8_t* isPerson, Enq q)
{
    launch(q, "k_person_table", k_person_table, 1, 256, 0, hdr, personClassID, isPerson);
}
void launch_seg_assign(const int* lab, const int* mapToMask, const uint8_t* ignore, int P, uint8_t* seg, Enq q)
{
    launch(q, "k_seg_assign", k_seg_assign, (P + 255) / 256, 256, 0, lab, mapToMask, ignore, P, seg);
}
void launch_mask_overlap(const uint8_t* seg, const uint8_t* projID, const uint8_t* idToIndex, const uint8_t* isModelId, int P, unsigned* maskOverlap, Enq q)
{
    launch(q, "k_mask_overlap", k_mask_overlap, (P + 255) / 256, 256, 0, seg, projID, idToIndex, isModelId, P, maskOverlap);
}
void launch_seg_final(const uint8_t* seg, const int* lab, const int* mapToMask, const int* absorb, const uint8_t* maskToID, const int* box, int P, int W,
                      uint8_t* out, Enq q)
{
    launch(q, "k_seg_final", k_seg_final, (P + 255) / 256, 256, 0, seg, lab, mapToMask, absorb, maskToID, box, P, W, out);
}
void launch_apply_ignore(const uint8_t* mask, const uint8_t* isPerson, const FrameHdr* hdr, int P, uint8_t* ignore, uint8_t* edges, Enq q)
{
    launch(q, "k_apply_ignore", k_apply_ignore, (P + 255) / 256, 256, 0, mask, isPerson, hdr, P, ignore, edges);
}
void launch_proj_resolve(uint64_t* key, int P, const uint8_t* indexToId, uint8_t* out, Enq q)
{
    launch(q, "k_proj_resolve", k_proj_resolve, (P + 255) / 256, 256, 0, (unsigned long long*)key, P, indexToId, out);
}

}  // namespace mfb
