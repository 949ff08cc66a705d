// mf_rpn.cu -- Mask R-CNN region-proposal stage on the backbone's P2..P6 (sm_90a): RPN head, proposal layer, pyramid ROI Align.
//
// The network is matterport mrcnn's inference graph with the COCO InferenceConfig defaults, written from upstream memory (the source is not
// vendored; DESIGN §3c, rules R-TOPK / R-NMS / R-ROILEVEL in §4):
//   rpn_graph        shared 3x3 256->512 conv + ReLU on every level, 1x1 512->6 class logits (channel a*2+c), 1x1 512->12 box deltas
//                    (channel a*4+k, k = dy dx log(dh) log(dw)), 3 anchors per feature pixel
//   ProposalLayer    softmax score, deltas * RPN_BBOX_STD_DEV, top min(6000, A) by score, apply_box_deltas_graph, clip to [0,0,1,1],
//                    greedy NMS at IoU 0.7 up to 1000 boxes, zero padding to 1000
//   PyramidROIAlign  level from the box area, tf.image.crop_and_resize (bilinear) on P2..P5 -> [n][P][P][256] bf16 (NHWC per ROI)
// The 3x3 conv runs through the backbone's conv path (cnn_conv: implicit wgmma GEMM, or im2col + GEMM where its geometry guard refuses the
// shape); the two 1x1 heads are ONE wgmma GEMM over the concatenated conv outputs of all levels, 18 weight rows zero-padded to 64, with the
// fp32 epilogue.  Everything after the GEMMs is IEEE fp32 in a fixed operation order (this file is compiled -fmad=false), so proposals
// and pooled features are reproducible bit for bit by the numpy restatement in tests/rpn_ref.py.
//
// Proposal layer: a sequence of launches on one stream, no inter-CTA waits.
//   k_rpn_keys      key = ~ord(score) << 32 | anchor index: ascending key order is R-TOPK order; resets the selection state
//   k_sel_hist/pick radix select of the k-th smallest key, 8 bits per pass: 4 passes over the score bits, then the used anchor-index bits
//   k_sel_compact   the k keys <= the k-th one (unordered: slots from an atomic counter)
//   k_sort_decode   one CTA: bitonic sort of the k keys in shared memory, then apply_box_deltas + clip in R-TOPK order
//   k_nms_mask      IoU > 0.7 bitmask: candidate i x 64-candidate words (upper triangle only)
//   k_nms_scan      one warp: the greedy scan over the bitmask, stop at 1000 kept, zero padding
#include "mf_common.cuh"
#include "mf_boxes.cuh"
#include "mf_kernels.h"
#include "../../include/maskfusion_b200.h"
#include <cuda_bf16.h>
#include <algorithm>
#include <math.h>
#include <string.h>
#include <string>
#include <vector>

namespace mfb {

constexpr int RPN_PRE_NMS = 6000, RPN_POST_NMS = 1000, RPN_POOL = 7, RPN_CH = 256, RPN_MID = 512, RPN_HEAD_N = 64;
constexpr int NMS_WORDS = (RPN_PRE_NMS + 63) / 64;          // 94 words of 64 candidates
constexpr int SORT_CAP = 8192;                              // bitonic sort size >= RPN_PRE_NMS, 64 KB of keys in shared memory
constexpr float RPN_NMS_THRESHOLD = 0.7f;

struct SelState { unsigned long long prefix, mask; unsigned krem, nsel; unsigned hist[256]; };

// softmax over the two logits (Keras: exp(x - max) / sum) -> foreground score -> R-TOPK key; block 0 resets the selection state
__global__ void k_rpn_keys(const float2* __restrict__ logits, int n, int k, unsigned long long* __restrict__ keys, SelState* st)
{
    if (blockIdx.x == 0) {
        for (int t = threadIdx.x; t < 256; t += blockDim.x) st->hist[t] = 0;
        if (threadIdx.x == 0) { st->prefix = 0; st->mask = 0; st->krem = (unsigned)k; st->nsel = 0; }
    }
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float2 l = logits[i];
        const float m = l.y > l.x ? l.y : l.x;
        const float e0 = det_expf(l.x - m), e1 = det_expf(l.y - m);
        const float score = e1 / (e0 + e1);
        keys[i] = ((unsigned long long)(~score_ord(score)) << 32) | (unsigned)i;
    }
}

// histogram of the 8-bit digit at `shift` over the keys that match the prefix selected so far
__global__ void k_sel_hist(const unsigned long long* __restrict__ keys, int n, SelState* st, int shift)
{
    __shared__ unsigned h[256];
    for (int t = threadIdx.x; t < 256; t += blockDim.x) h[t] = 0;
    __syncthreads();
    const unsigned long long mask = st->mask, prefix = st->prefix;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long key = keys[i];
        if ((key & mask) == prefix) atomicAdd(&h[(key >> shift) & 255], 1u);
    }
    __syncthreads();
    for (int t = threadIdx.x; t < 256; t += blockDim.x)
        if (h[t]) atomicAdd(&st->hist[t], h[t]);
}

// the digit bin that holds the krem-th smallest matching key joins the prefix; the histogram is cleared for the next pass
__global__ void k_sel_pick(SelState* st, int shift)
{
    __shared__ unsigned h[256];
    h[threadIdx.x] = st->hist[threadIdx.x];
    st->hist[threadIdx.x] = 0;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned cum = 0;
        for (int d = 0; d < 256; ++d) {
            if (cum + h[d] >= st->krem) {
                st->prefix |= (unsigned long long)d << shift;
                st->mask |= 0xFFull << shift;
                st->krem -= cum;
                break;
            }
            cum += h[d];
        }
    }
}

// keys are unique (the anchor index is in the low half): exactly k of them are <= the k-th smallest
__global__ void k_sel_compact(const unsigned long long* __restrict__ keys, int n, SelState* st, unsigned long long* __restrict__ sel)
{
    const unsigned long long kth = st->prefix;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long key = keys[i];
        if (key <= kth) sel[atomicAdd(&st->nsel, 1u)] = key;
    }
}

// one CTA: bitonic sort of the k selected keys (padded with ~0 to a power of two), then the boxes in R-TOPK order
__global__ void __launch_bounds__(1024) k_sort_decode(const unsigned long long* __restrict__ sel, int k, const float4* __restrict__ deltas,
                                                      const float4* __restrict__ anchors, float4* __restrict__ boxes)
{
    extern __shared__ unsigned long long sk[];
    int P = 1;
    while (P < k) P <<= 1;
    for (int i = threadIdx.x; i < P; i += blockDim.x) sk[i] = i < k ? sel[i] : ~0ull;
    __syncthreads();
    cta_bitonic_sort(sk, P);
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        const unsigned idx = (unsigned)(sk[i] & 0xFFFFFFFFull);
        boxes[i] = decode_box(anchors[idx], deltas[idx], make_float4(0.f, 0.f, 1.f, 1.f));
    }
}

// bit j of word (i, c) set <=> candidate 64c + j comes after i and IoU(i, 64c + j) > 0.7; words left of the diagonal are not written
__global__ void __launch_bounds__(64) k_nms_mask(const float4* __restrict__ boxes, int k, int words, unsigned long long* __restrict__ mask)
{
    const int row = blockIdx.y, col = blockIdx.x;
    if (col < row) return;
    const int rowSize = min(k - row * 64, 64), colSize = min(k - col * 64, 64);
    __shared__ float4 cb[64];
    if ((int)threadIdx.x < colSize) cb[threadIdx.x] = boxes[col * 64 + threadIdx.x];
    __syncthreads();
    if ((int)threadIdx.x >= rowSize) return;
    const int i = row * 64 + threadIdx.x;
    const float4 bi = boxes[i];
    unsigned long long bits = 0;
    for (int j = row == col ? threadIdx.x + 1 : 0; j < colSize; ++j)
        if (iou_tf(bi, cb[j]) > RPN_NMS_THRESHOLD) bits |= 1ull << j;
    mask[(size_t)i * words + col] = bits;
}

// one warp, greedy in R-TOPK order; lane l holds the suppression words l, l + 32, l + 64
__global__ void __launch_bounds__(32) k_nms_scan(const float4* __restrict__ boxes, const unsigned long long* __restrict__ mask, int k, int words,
                                                 float4* __restrict__ rois, int* __restrict__ count)
{
    const int lane = threadIdx.x;
    unsigned long long r0 = 0, r1 = 0, r2 = 0;
    int kept = 0;
    for (int i = 0; i < k && kept < RPN_POST_NMS; ++i) {
        const int w = i >> 6, slot = w >> 5;
        const unsigned long long mine = slot == 0 ? r0 : (slot == 1 ? r1 : r2);
        const unsigned long long v = __shfl_sync(0xFFFFFFFFu, mine, w & 31);
        if ((v >> (i & 63)) & 1ull) continue;
        if (lane == 0) rois[kept] = boxes[i];
        ++kept;
        const unsigned long long* row = mask + (size_t)i * words;
        if (lane >= w && lane < words) r0 |= row[lane];
        if (lane + 32 >= w && lane + 32 < words) r1 |= row[lane + 32];
        if (lane + 64 >= w && lane + 64 < words) r2 |= row[lane + 64];
    }
    for (int j = kept + lane; j < RPN_POST_NMS; j += 32) rois[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane == 0) *count = kept;
}

// head GEMM rows [pixel][64] (0..5 logits, 6..17 deltas) -> logits [A][2], deltas [A][4] with anchor = 3 * pixel + a
__global__ void k_rpn_split(const float* __restrict__ head, int pixels, float* __restrict__ logits, float* __restrict__ deltas)
{
    const int total = pixels * 18;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
        const int p = t / 18, c = t - p * 18;
        const float v = head[(size_t)p * RPN_HEAD_N + c];
        if (c < 6) logits[(size_t)p * 6 + c] = v;
        else deltas[(size_t)p * 12 + c - 6] = v;
    }
}

// ---- pyramid ROI Align (tf.image.crop_and_resize, bilinear, extrapolation value 0) ----
struct RoiLevels { const __nv_bfloat16* P[4]; int H[4], W[4]; };

// R-ROILEVEL: t = h*w * fp32(S^2 / 224^2) against the exact boundaries of 4 + round(log2(sqrt(h*w) * S / 224)); NaN / degenerate -> 2
MF_D int roi_level(float4 b, float areaScale)
{
    const float t = ((b.z - b.x) * (b.w - b.y)) * areaScale;
    return 2 + (t >= 0.125f) + (t >= 0.5f) + (t >= 2.0f);
}

// block (roi, output row), thread = channel pair; out [n][P][P][256] bf16, each value rounded once from the fp32 interpolation
__global__ void __launch_bounds__(128) k_roi_align(const float4* __restrict__ boxes, int pool, RoiLevels lv, float areaScale,
                                                   __nv_bfloat16* __restrict__ out)
{
    const int roi = blockIdx.x, iy = blockIdx.y, c = 2 * threadIdx.x;
    const float4 b = boxes[roi];
    const int li = roi_level(b, areaScale) - 2;                     // selects, not an indexed load: the parameter struct stays in registers
    const __nv_bfloat16* f = li == 0 ? lv.P[0] : li == 1 ? lv.P[1] : li == 2 ? lv.P[2] : lv.P[3];
    const int H = li == 0 ? lv.H[0] : li == 1 ? lv.H[1] : li == 2 ? lv.H[2] : lv.H[3];
    const int W = li == 0 ? lv.W[0] : li == 1 ? lv.W[1] : li == 2 ? lv.W[2] : lv.W[3];
    const float hs = ((b.z - b.x) * (float)(H - 1)) / (float)(pool - 1);
    const float ws = ((b.w - b.y) * (float)(W - 1)) / (float)(pool - 1);
    const float in_y = b.x * (float)(H - 1) + (float)iy * hs;
    __nv_bfloat162* o = reinterpret_cast<__nv_bfloat162*>(out + (((size_t)roi * pool + iy) * pool) * RPN_CH + c);
    const __nv_bfloat162 zero = __floats2bfloat162_rn(0.f, 0.f);
    if (!(in_y >= 0.0f && in_y <= (float)(H - 1))) {               // outside the map (or NaN): the whole row is the extrapolation value
        for (int ix = 0; ix < pool; ++ix) o[ix * (RPN_CH / 2)] = zero;
        return;
    }
    const int ty = (int)floorf(in_y), by = (int)ceilf(in_y);
    const float yl = in_y - (float)ty;
    for (int ix = 0; ix < pool; ++ix) {
        const float in_x = b.y * (float)(W - 1) + (float)ix * ws;
        if (!(in_x >= 0.0f && in_x <= (float)(W - 1))) { o[ix * (RPN_CH / 2)] = zero; continue; }
        const int lx = (int)floorf(in_x), rx = (int)ceilf(in_x);
        const float xl = in_x - (float)lx;
        const float2 tl = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(f + ((size_t)ty * W + lx) * RPN_CH + c));
        const float2 tr = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(f + ((size_t)ty * W + rx) * RPN_CH + c));
        const float2 bl = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(f + ((size_t)by * W + lx) * RPN_CH + c));
        const float2 br = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(f + ((size_t)by * W + rx) * RPN_CH + c));
        const float t0 = tl.x + (tr.x - tl.x) * xl, t1 = tl.y + (tr.y - tl.y) * xl;
        const float b0 = bl.x + (br.x - bl.x) * xl, b1 = bl.y + (br.y - bl.y) * xl;
        o[ix * (RPN_CH / 2)] = __floats2bfloat162_rn(t0 + (b0 - t0) * yl, t1 + (b1 - t1) * yl);
    }
}

static uint32_t lcg(uint32_t& s) { s = s * 1664525u + 1013904223u; return s; }
static float urand(uint32_t& s) { return (float)(lcg(s) >> 8) * (1.0f / 16777216.0f) * 2.f - 1.f; }
static float bf16_round(float f) { return __bfloat162float(__float2bfloat16(f)); }

void synth_weights(float* w, float* b, int rows, int K, float gain, uint32_t& seed)
{
    const float sc = gain * sqrtf(2.0f / (float)K);
    for (int o = 0; o < rows; ++o)
        for (int kk = 0; kk < K; ++kk) w[(size_t)o * K + kk] = bf16_round(urand(seed) * sc * 1.7320508f);
    for (int o = 0; o < rows; ++o) b[o] = urand(seed) * 0.05f;
}

static int rpn_fail(const std::string& msg) { cnn_set_error(msg.c_str()); return -1; }

static int check_launch(const char* what)
{
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return rpn_fail(std::string(what) + ": " + cudaGetErrorString(e));
    return 0;
}

}  // namespace mfb

using namespace mfb;

struct mf_rpn {
    mf_backbone* bb = nullptr;
    cudaStream_t s = nullptr;
    int S = 0, A = 0, pixels = 0;
    int lh[5] = {}, pixOff[6] = {};                          // P2..P6 side length, first pixel of each level in the concatenation
    std::vector<float> hWc, hBc, hWh, hBh;                   // conv [512 x 2304], heads [64 x 512] (rows >= 18 zero), fp32 master copies
    __nv_bfloat16 *dWc = nullptr, *dWh = nullptr, *col = nullptr, *conv = nullptr, *pooled = nullptr;
    float *dBc = nullptr, *dBh = nullptr, *head = nullptr, *logits = nullptr, *deltas = nullptr, *anchors = nullptr, *rois = nullptr;
    unsigned long long *keys = nullptr, *sel = nullptr, *mask = nullptr;
    SelState* st = nullptr;
    float4* boxes = nullptr;
    int* count = nullptr;
};

static RoiLevels roi_levels(mf_backbone* bb)
{
    RoiLevels lv;
    for (int i = 0; i < 4; ++i) {
        int d[3];
        lv.P[i] = (const __nv_bfloat16*)mf_backbone_output(bb, 4 + i, d);
        lv.H[i] = d[0]; lv.W[i] = d[1];
    }
    return lv;
}

static int roi_align(mf_backbone* bb, const float* boxes, int n, int pool, void* out, cudaStream_t s)
{
    if (n == 0) return 0;
    int d[3];
    mf_backbone_output(bb, 4, d);
    const int S = d[0] * 4;
    const float areaScale = (float)((double)S * (double)S / (224.0 * 224.0));
    prof_mark(s, "k_roi_align");
    k_roi_align<<<dim3(n, pool), RPN_CH / 2, 0, s>>>((const float4*)boxes, pool, roi_levels(bb), areaScale, (__nv_bfloat16*)out);
    return check_launch("k_roi_align");
}

// the proposal layer on logits [n][2], deltas [n][4], anchors [n][4] (device) -> h->rois [1000][4], h->count
static int propose(mf_rpn* h, const float* logits, const float* deltas, const float* anchors, int n)
{
    const cudaStream_t s = h->s;
    const int k = n < RPN_PRE_NMS ? n : RPN_PRE_NMS;
    const int grid = (n + 255) / 256, histGrid = std::min((n + 2047) / 2048, 2 * num_sms());
    prof_mark(s, "k_rpn_keys");
    k_rpn_keys<<<grid, 256, 0, s>>>((const float2*)logits, n, k, h->keys, h->st);
    int shifts[8], np = 0;
    for (int sh = 56; sh >= 32; sh -= 8) shifts[np++] = sh;
    int idxBits = 0;
    while (idxBits < 32 && ((n - 1) >> idxBits)) ++idxBits;                  // anchor-index bits that vary
    for (int sh = 24; sh >= 0; sh -= 8)
        if (sh < idxBits) shifts[np++] = sh;
    for (int p = 0; p < np; ++p) {
        prof_mark(s, "k_sel_hist");
        k_sel_hist<<<histGrid, 256, 0, s>>>(h->keys, n, h->st, shifts[p]);
        prof_mark(s, "k_sel_pick");
        k_sel_pick<<<1, 256, 0, s>>>(h->st, shifts[p]);
    }
    prof_mark(s, "k_sel_compact");
    k_sel_compact<<<grid, 256, 0, s>>>(h->keys, n, h->st, h->sel);
    prof_mark(s, "k_sort_decode");
    k_sort_decode<<<1, 1024, SORT_CAP * sizeof(unsigned long long), s>>>(h->sel, k, (const float4*)deltas, (const float4*)anchors, h->boxes);
    const int words = (k + 63) / 64;
    prof_mark(s, "k_nms_mask");
    k_nms_mask<<<dim3(words, words), 64, 0, s>>>(h->boxes, k, words, h->mask);
    prof_mark(s, "k_nms_scan");
    k_nms_scan<<<1, 32, 0, s>>>(h->boxes, h->mask, k, words, (float4*)h->rois, h->count);
    return check_launch("proposal layer");
}

// ==========================================================================================
// C ABI (declared in include/maskfusion_b200.h)
// ==========================================================================================
extern "C" void mf_rpn_destroy(mf_rpn* h)
{
    if (!h) return;
    void* ptrs[] = {h->dWc, h->dWh, h->col, h->conv, h->pooled, h->dBc, h->dBh, h->head, h->logits, h->deltas, h->anchors, h->rois,
                    h->keys, h->sel, h->mask, h->st, h->boxes, h->count};
    for (void* p : ptrs) if (p) cudaFree(p);
    delete h;
}

extern "C" mf_rpn* mf_rpn_create(mf_backbone* bb, unsigned seed)
{
    if (!bb) { rpn_fail("rpn: no backbone"); return nullptr; }
    mf_rpn* h = new mf_rpn;
    h->bb = bb;
    h->s = (cudaStream_t)mf_backbone_stream(bb);
    int d[3];
    mf_backbone_output(bb, 4, d);
    h->S = d[0] * 4;
    for (int l = 0; l < 5; ++l) {
        h->lh[l] = h->S >> (l + 2);
        h->pixOff[l + 1] = h->pixOff[l] + h->lh[l] * h->lh[l];
    }
    h->pixels = h->pixOff[5];
    h->A = 3 * h->pixels;
    // weights: shared conv (gain 1).  The synthetic P levels are O(100) (the moulded input is in pixel units), and so is the conv output:
    // the class-logit layer is damped to logits of a few units (scores spread over (0, 1) instead of saturating at 0 / 1) and the delta
    // layer to |delta| ~ 0.1 (decoded boxes stay near their anchors)
    uint32_t sd = seed ? seed : 1u;
    const int Kc = 9 * RPN_CH;
    h->hWc.assign((size_t)RPN_MID * Kc, 0.f); h->hBc.assign(RPN_MID, 0.f);
    h->hWh.assign((size_t)RPN_HEAD_N * RPN_MID, 0.f); h->hBh.assign(RPN_HEAD_N, 0.f);
    synth_weights(h->hWc.data(), h->hBc.data(), RPN_MID, Kc, 1.0f, sd);
    synth_weights(h->hWh.data(), h->hBh.data(), 6, RPN_MID, 2e-4f, sd);
    synth_weights(h->hWh.data() + 6 * RPN_MID, h->hBh.data() + 6, 12, RPN_MID, 2e-5f, sd);
    // anchors: generate_pyramid_anchors + norm_boxes in double, rounded once to float; order (level, y, x, ratio)
    std::vector<float> anc((size_t)h->A * 4);
    const double ratios[3] = {0.5, 1.0, 2.0}, S1 = (double)(h->S - 1);
    size_t a = 0;
    for (int l = 0; l < 5; ++l) {
        const double scale = 32.0 * (1 << l), stride = 4.0 * (1 << l);
        for (int y = 0; y < h->lh[l]; ++y)
            for (int x = 0; x < h->lh[l]; ++x)
                for (int r = 0; r < 3; ++r, ++a) {
                    const double bh = scale / sqrt(ratios[r]), bw = scale * sqrt(ratios[r]), cy = y * stride, cx = x * stride;
                    anc[a * 4 + 0] = (float)((cy - 0.5 * bh) / S1);
                    anc[a * 4 + 1] = (float)((cx - 0.5 * bw) / S1);
                    anc[a * 4 + 2] = (float)((cy + 0.5 * bh - 1.0) / S1);
                    anc[a * 4 + 3] = (float)((cx + 0.5 * bw - 1.0) / S1);
                }
    }
    // im2col scratch only for the levels whose shape the implicit 3x3 path refuses
    size_t colElems = 0;
    for (int l = 0; l < 5; ++l)
        if (!cnn_conv_implicit(3, 1, 1, RPN_CH, h->lh[l], h->lh[l])) colElems = std::max(colElems, (size_t)h->lh[l] * h->lh[l] * Kc);
    const size_t A = h->A;
    bool ok = cudaMalloc(&h->dWc, h->hWc.size() * 2) == cudaSuccess && cudaMalloc(&h->dWh, h->hWh.size() * 2) == cudaSuccess &&
              cudaMalloc(&h->dBc, RPN_MID * 4) == cudaSuccess && cudaMalloc(&h->dBh, RPN_HEAD_N * 4) == cudaSuccess &&
              (colElems == 0 || cudaMalloc(&h->col, colElems * 2) == cudaSuccess) &&
              cudaMalloc(&h->conv, (size_t)h->pixels * RPN_MID * 2) == cudaSuccess && cudaMalloc(&h->head, (size_t)h->pixels * RPN_HEAD_N * 4) == cudaSuccess &&
              cudaMalloc(&h->logits, A * 2 * 4) == cudaSuccess && cudaMalloc(&h->deltas, A * 4 * 4) == cudaSuccess &&
              cudaMalloc(&h->anchors, A * 4 * 4) == cudaSuccess && cudaMalloc(&h->keys, A * 8) == cudaSuccess &&
              cudaMalloc(&h->sel, RPN_PRE_NMS * 8) == cudaSuccess && cudaMalloc(&h->mask, (size_t)RPN_PRE_NMS * NMS_WORDS * 8) == cudaSuccess &&
              cudaMalloc(&h->st, sizeof(SelState)) == cudaSuccess && cudaMalloc(&h->boxes, RPN_PRE_NMS * 16) == cudaSuccess &&
              cudaMalloc(&h->rois, RPN_POST_NMS * 16) == cudaSuccess && cudaMalloc(&h->count, 4) == cudaSuccess &&
              cudaMalloc(&h->pooled, (size_t)RPN_POST_NMS * RPN_POOL * RPN_POOL * RPN_CH * 2) == cudaSuccess;
    if (!ok) { rpn_fail("rpn: cudaMalloc failed"); mf_rpn_destroy(h); return nullptr; }
    std::vector<__nv_bfloat16> wc(h->hWc.size()), wh(h->hWh.size());
    for (size_t i = 0; i < wc.size(); ++i) wc[i] = __float2bfloat16(h->hWc[i]);
    for (size_t i = 0; i < wh.size(); ++i) wh[i] = __float2bfloat16(h->hWh[i]);
    ok = cudaMemcpy(h->dWc, wc.data(), wc.size() * 2, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(h->dWh, wh.data(), wh.size() * 2, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(h->dBc, h->hBc.data(), RPN_MID * 4, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(h->dBh, h->hBh.data(), RPN_HEAD_N * 4, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(h->anchors, anc.data(), anc.size() * 4, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemset(h->rois, 0, RPN_POST_NMS * 16) == cudaSuccess && cudaMemset(h->count, 0, 4) == cudaSuccess &&
         cudaFuncSetAttribute(k_sort_decode, cudaFuncAttributeMaxDynamicSharedMemorySize, SORT_CAP * (int)sizeof(unsigned long long)) == cudaSuccess;
    if (!ok) { rpn_fail("rpn: upload failed"); mf_rpn_destroy(h); return nullptr; }
    return h;
}

extern "C" int mf_rpn_run(mf_rpn* h, int stages)
{
    if (!h) return rpn_fail("rpn: null handle");
    const cudaStream_t s = h->s;
    if (stages & MF_RPN_CONV)
        for (int l = 0; l < 5; ++l) {
            int d[3];
            const void* in = mf_backbone_output(h->bb, 4 + l, d);
            if (cnn_conv(in, d[0], d[1], RPN_CH, RPN_MID, 3, 1, 1, h->dWc, h->dBc, h->col, h->conv + (size_t)h->pixOff[l] * RPN_MID, 1, s)) return -2;
        }
    if (stages & MF_RPN_HEADS) {
        if (launch_gemm_bf16(h->conv, h->dWh, h->dBh, nullptr, h->head, h->pixels, RPN_HEAD_N, RPN_MID, 0, s, nullptr, true)) return -2;
        prof_mark(s, "k_rpn_split");
        k_rpn_split<<<std::min((h->pixels * 18 + 255) / 256, 8 * num_sms()), 256, 0, s>>>(h->head, h->pixels, h->logits, h->deltas);
        if (check_launch("k_rpn_split")) return -3;
    }
    if ((stages & MF_RPN_PROPOSALS) && propose(h, h->logits, h->deltas, h->anchors, h->A)) return -3;
    if ((stages & MF_RPN_ROI_ALIGN) && roi_align(h->bb, h->rois, RPN_POST_NMS, RPN_POOL, h->pooled, s)) return -3;
    return 0;
}

extern "C" int mf_rpn_forward(mf_rpn* h) { return mf_rpn_run(h, MF_RPN_CONV | MF_RPN_HEADS | MF_RPN_PROPOSALS | MF_RPN_ROI_ALIGN); }

extern "C" int mf_rpn_propose(mf_rpn* h, const float* d_logits, const float* d_deltas, const float* d_anchors, int n_anchors)
{
    if (!h) return rpn_fail("rpn: null handle");
    if (n_anchors < 1 || n_anchors > h->A)
        return rpn_fail("rpn_propose: n_anchors = " + std::to_string(n_anchors) + " outside [1, " + std::to_string(h->A) + "]");
    if (!d_logits || !d_deltas || !d_anchors || ((uintptr_t)d_logits & 7) || ((uintptr_t)d_deltas & 15) || ((uintptr_t)d_anchors & 15))
        return rpn_fail("rpn_propose: logits need 8-byte, deltas and anchors 16-byte aligned device pointers");
    return propose(h, d_logits, d_deltas, d_anchors, n_anchors) ? -3 : 0;
}

extern "C" int mf_roi_align_bf16(mf_backbone* bb, const float* d_boxes, int n, int pool, void* d_out)
{
    if (!bb) return rpn_fail("roi_align: no backbone");
    if (n < 0 || pool < 2 || pool > 64) return rpn_fail("roi_align: need n >= 0 and 2 <= pool <= 64");
    if (n > 0 && (!d_boxes || !d_out || ((uintptr_t)d_boxes & 15) || ((uintptr_t)d_out & 3)))
        return rpn_fail("roi_align: boxes need a 16-byte, out a 4-byte aligned device pointer");
    return roi_align(bb, d_boxes, n, pool, d_out, (cudaStream_t)mf_backbone_stream(bb)) ? -3 : 0;
}

extern "C" int mf_rpn_num_anchors(mf_rpn* h) { return h ? h->A : -1; }

extern "C" int mf_rpn_get_weights(mf_rpn* h, float* conv_w, float* conv_b, float* head_w, float* head_b)
{
    if (!h) return rpn_fail("rpn: null handle");
    if (conv_w) memcpy(conv_w, h->hWc.data(), h->hWc.size() * 4);
    if (conv_b) memcpy(conv_b, h->hBc.data(), h->hBc.size() * 4);
    if (head_w) memcpy(head_w, h->hWh.data(), (size_t)18 * RPN_MID * 4);
    if (head_b) memcpy(head_b, h->hBh.data(), 18 * 4);
    return 0;
}

// pretrained weights (mf_weights.cu): read, checked and folded on the host first; the copy is ordered on the stream and complete on return
extern "C" int mf_rpn_load_weights(mf_rpn* h, const char* path)
{
    if (!h) return rpn_fail("rpn: null handle");
    std::vector<float> wc(h->hWc.size()), bc(h->hBc.size()), wh(h->hWh.size()), bh(h->hBh.size());
    float* w[2] = {wc.data(), wh.data()};
    float* b[2] = {bc.data(), bh.data()};
    int rows[2], K[2];
    for (int i = 0; i < 2; ++i) mrcnn_layer_dims(MRCNN_RPN, i, &rows[i], &K[i]);
    if (mrcnn_layer_count(MRCNN_RPN) != 2 || (size_t)rows[0] * K[0] != wc.size() || (size_t)rows[1] * K[1] != wh.size())
        return rpn_fail("rpn: the weight-name table does not match the handle's tables");
    if (mrcnn_fold(path, MRCNN_RPN, w, b)) return -1;
    std::vector<__nv_bfloat16> wcb(wc.size()), whb(wh.size());
    for (size_t i = 0; i < wc.size(); ++i) wcb[i] = __float2bfloat16(wc[i]);
    for (size_t i = 0; i < wh.size(); ++i) whb[i] = __float2bfloat16(wh[i]);
    cudaError_t e = cudaMemcpyAsync(h->dWc, wcb.data(), wcb.size() * 2, cudaMemcpyHostToDevice, h->s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(h->dWh, whb.data(), whb.size() * 2, cudaMemcpyHostToDevice, h->s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(h->dBc, bc.data(), bc.size() * 4, cudaMemcpyHostToDevice, h->s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(h->dBh, bh.data(), bh.size() * 4, cudaMemcpyHostToDevice, h->s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->s);
    if (e != cudaSuccess) return rpn_fail(std::string("rpn: weight upload: ") + cudaGetErrorString(e));
    h->hWc.swap(wc); h->hBc.swap(bc); h->hWh.swap(wh); h->hBh.swap(bh);
    return 0;
}

static int download(mf_rpn* h, void* dst, const void* src, size_t bytes)
{
    if (!h) return rpn_fail("rpn: null handle");
    if (cudaStreamSynchronize(h->s) != cudaSuccess || cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost) != cudaSuccess)
        return rpn_fail(std::string("rpn download: ") + cudaGetErrorString(cudaGetLastError()));
    return 0;
}

extern "C" int mf_rpn_get_anchors(mf_rpn* h, float* anchors)
{
    return h ? download(h, anchors, h->anchors, (size_t)h->A * 16) : rpn_fail("rpn: null handle");
}

extern "C" int mf_rpn_get_head_outputs(mf_rpn* h, float* logits, float* deltas)
{
    if (!h) return rpn_fail("rpn: null handle");
    return download(h, logits, h->logits, (size_t)h->A * 8) || download(h, deltas, h->deltas, (size_t)h->A * 16) ? -1 : 0;
}

extern "C" int mf_rpn_download_conv(mf_rpn* h, int level, void* host_bf16)
{
    if (!h) return rpn_fail("rpn: null handle");
    if (level < 0 || level > 4) return rpn_fail("rpn: level must be 0..4 (P2..P6)");
    return download(h, host_bf16, h->conv + (size_t)h->pixOff[level] * RPN_MID, (size_t)h->lh[level] * h->lh[level] * RPN_MID * 2);
}

extern "C" int mf_rpn_get_proposals(mf_rpn* h, float* rois)
{
    int n = 0;
    if (!h) return rpn_fail("rpn: null handle");
    if (download(h, rois, h->rois, RPN_POST_NMS * 16) || download(h, &n, h->count, 4)) return -1;
    return n;
}

extern "C" int mf_rpn_get_pooled(mf_rpn* h, void* host_bf16)
{
    return h ? download(h, host_bf16, h->pooled, (size_t)RPN_POST_NMS * RPN_POOL * RPN_POOL * RPN_CH * 2) : rpn_fail("rpn: null handle");
}

// ---- what the detection heads (mf_heads.cu) read of the handle ----
mf_backbone* mfb::rpn_backbone(mf_rpn* h) { return h->bb; }
const float* mfb::rpn_rois(mf_rpn* h) { return h->rois; }
const void* mfb::rpn_pooled(mf_rpn* h) { return h->pooled; }
