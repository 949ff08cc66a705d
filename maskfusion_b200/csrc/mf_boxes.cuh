// mf_boxes.cuh -- box arithmetic shared by the proposal layer (mf_rpn.cu) and the detection heads (mf_heads.cu), and the export rule of
// generate_id_image shared by the host function (mf_loader.cu) and the device id-image pass (mf_heads.cu).
// Files that use the device functions are compiled -fmad=false: the numpy restatements (tests/rpn_ref.py, tests/heads_ref.py) repeat
// every operation in this order.
#pragma once
#include <stdint.h>
#include "mf_common.cuh"

namespace mfb {

// order-preserving map of a float to uint32 (ascending); -0 is +0, NaN -> 0 (below -inf, so ~ord puts it last)
MF_D uint32_t score_ord(float s)
{
    if (s != s) return 0u;
    if (s == 0.0f) s = 0.0f;
    const uint32_t u = __float_as_uint(s);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// apply_box_deltas_graph (upstream operation order, deltas scaled by BBOX_STD_DEV = RPN_BBOX_STD_DEV = 0.1 0.1 0.2 0.2) + clip_boxes_graph
// to the window w = (y1, x1, y2, x2); box = y1 x1 y2 x2.  The RPN clips to (0, 0, 1, 1), the detection layer to the letter-box window.
MF_D float4 decode_box(float4 a, float4 d, float4 win)
{
    d.x = d.x * 0.1f; d.y = d.y * 0.1f; d.z = d.z * 0.2f; d.w = d.w * 0.2f;
    float h = a.z - a.x, w = a.w - a.y;
    float cy = a.x + 0.5f * h, cx = a.y + 0.5f * w;
    cy = cy + d.x * h;
    cx = cx + d.y * w;
    h = h * det_expf(d.z);
    w = w * det_expf(d.w);
    const float y1 = cy - 0.5f * h, x1 = cx - 0.5f * w;
    const float y2 = y1 + h, x2 = x1 + w;
    return make_float4(fmaxf(fminf(y1, win.z), win.x), fmaxf(fminf(x1, win.w), win.y), fmaxf(fminf(y2, win.z), win.x), fmaxf(fminf(x2, win.w), win.y));
}

// ascending bitonic sort of P (a power of two) keys in shared memory by the whole CTA; ends with a barrier
MF_D void cta_bitonic_sort(unsigned long long* sk, int P)
{
    for (int size = 2; size <= P; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = threadIdx.x; i < P / 2; i += blockDim.x) {
                const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const bool asc = (lo & size) == 0;
                const unsigned long long a = sk[lo], b = sk[hi];
                if ((a > b) == asc) { sk[lo] = b; sk[hi] = a; }
            }
            __syncthreads();
        }
}

// TensorFlow's NMS IoU: corners min/max-normalised, an empty box overlaps nothing
MF_D float lesser(float a, float b) { return b < a ? b : a; }       // std::min
MF_D float greater(float a, float b) { return a < b ? b : a; }      // std::max
MF_D float iou_tf(float4 i, float4 j)
{
    const float ymin_i = lesser(i.x, i.z), xmin_i = lesser(i.y, i.w), ymax_i = greater(i.x, i.z), xmax_i = greater(i.y, i.w);
    const float ymin_j = lesser(j.x, j.z), xmin_j = lesser(j.y, j.w), ymax_j = greater(j.x, j.z), xmax_j = greater(j.y, j.w);
    const float area_i = (ymax_i - ymin_i) * (xmax_i - xmin_i);
    const float area_j = (ymax_j - ymin_j) * (xmax_j - xmin_j);
    if (area_i <= 0.0f || area_j <= 0.0f) return 0.0f;
    const float iymin = greater(ymin_i, ymin_j), ixmin = greater(xmin_i, xmin_j);
    const float iymax = lesser(ymax_i, ymax_j), ixmax = lesser(xmax_i, xmax_j);
    const float inter = greater(iymax - iymin, 0.0f) * greater(ixmax - ixmin, 0.0f);
    return inter / ((area_i + area_j) - inter);
}

// generate_id_image's per-detection decision (Core/Segmentation/MaskRCNN/helpers.py:70-98): a detection is exported when its class passes
// the filter (empty filter: every class) and score >= min_score (the float32 score against a double, as NumPy 1.x compares them).  Its id is
// `ordinal` + 1 (ordinal = detections exported before it) unless the class id occurs IN `special` (a list indexed BY class id,
// helpers.py:91-92); a numpy assignment into the uint8 image wraps.  Returns 1 (exported, *id set), 0 (skipped) or -1 (special[class id] is
// out of range: IndexError in Python).
MF_HD int id_export(int cid, float score, double min_score, const int32_t* filter, int n_filter, const int32_t* special, int n_special,
                    int ordinal, uint8_t* id)
{
    bool pass = n_filter == 0;
    for (int k = 0; k < n_filter && !pass; ++k) pass = filter[k] == cid;
    if (!pass || !((double)score >= min_score)) return 0;
    int val = ordinal + 1;
    bool sp = false;
    for (int k = 0; k < n_special && !sp; ++k) sp = special[k] == cid;
    if (sp) {
        if (cid < 0 || cid >= n_special) return -1;
        val = special[cid];
    }
    *id = (uint8_t)val;
    return 1;
}

}  // namespace mfb
