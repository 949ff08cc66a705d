// mf_weights.cu -- the layer table of the Mask R-CNN backbone, RPN and detector handles and their weight store: seeded tables, or
// pretrained weights from a safetensors file (host code only).  DESIGN §3c has the name table and the folding rule R-FOLD.
//
// File: an 8-byte little-endian header length N, N bytes of JSON {name: {"dtype", "shape", "data_offsets"}, "__metadata__": {str: str}},
// then the data section; data_offsets are [begin, end) byte offsets into that section.  The JSON is parsed by a reader of exactly this
// grammar; everything is bounds-checked before any tensor is read, and every message names the file and, where there is one, the tensor.
// Names are matterport's Keras names "<layer>/<param>" (nested-model prefixes and the ":0" suffix removed, scripts/convert_mrcnn_h5.py),
// arrays in the Keras layouts, F32 only.  Tensors no layer asks for are ignored (Keras load_weights(by_name=True)).
//
// R-FOLD (BatchNorm in inference mode, Keras epsilon 1e-3), in double per output channel o:
//   s = gamma / sqrt(moving_variance + 1e-3);  w' = bf16_rn((float)(w * s));  b' = (float)((bias - moving_mean) * s + beta)
// and s = 1, b' = (float)bias for a layer without BatchNorm.  Compiled with -ffp-contract=off: no fused multiply-add changes a rounding.
#include "mf_kernels.h"
#include <cuda_bf16.h>
#include <assert.h>
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <map>
#include <string>
#include <vector>

namespace {

struct Tensor { std::string dtype; std::vector<long long> shape; long long begin = 0, end = 0; };

// one source array of a handle layer: its Keras name, its Keras shape, the first GEMM row it fills, the gain of its seeded rows
struct Part { std::string layer; std::vector<long long> shape; int row0; float gain; };
struct LayerSpec {
    std::string name;                 // the handle layer's name: the Keras layer, or "a+b" for two layers stacked in one GEMM
    std::vector<Part> parts;
    std::string bn;                   // BatchNorm layer folded into it ("" = none)
    int stride, pad;
    bool deconv;                      // Conv2DTranspose (kh, kw, out, in): row (dy*kw + dx)*out + o, column c; bias repeated per (dy, dx)
    int rows, K;                      // the handle's table: [rows x K], zero padded to the GEMM's multiples of 64
};

int kpad(long long n) { return (int)((n + 63) / 64 * 64); }

long long part_cout(const LayerSpec& s, const Part& pt) { return s.deconv ? pt.shape[2] : pt.shape.back(); }
long long part_rows(const LayerSpec& s, const Part& pt) { return s.deconv ? pt.shape[0] * pt.shape[1] * pt.shape[2] : pt.shape.back(); }
long long part_cols(const LayerSpec& s, const Part& pt)      // K used: kh * kw * cin, the input width of a dense layer, cin of the deconv
{
    if (s.deconv) return pt.shape[3];
    long long cols = 1;
    for (size_t d = 0; d + 1 < pt.shape.size(); ++d) cols *= pt.shape[d];
    return cols;
}

LayerSpec layer(const std::string& name, std::vector<Part> parts, const std::string& bn, int stride, int pad, bool deconv = false)
{
    LayerSpec s{name, std::move(parts), bn, stride, pad, deconv, 0, 0};
    const Part& last = s.parts.back();
    s.rows = kpad(last.row0 + part_rows(s, last));
    s.K = kpad(part_cols(s, last));
    return s;
}

LayerSpec conv(const std::string& name, int k, int cin, int cout, const std::string& bn, int stride, int pad, float gain)
{
    return layer(name, {{name, {k, k, cin, cout}, 0, gain}}, bn, stride, pad);
}

// ResNet-101 (stages 3, 4, 23, 3; the stride in the first 1x1 of a stage, as in Keras/matterport) + FPN(256).  Seeded at gain 1 (He-style:
// activations stay O(1) through 101 layers) except branch2c at 0.5 (the residual sums keep O(1) variance) and the shortcut and lateral 1x1
// convs at 0.7.  Order: conv1, per block branch2a, 2b, 2c (+ branch1 in block a), fpn_c2p2..c5p5, fpn_p2..p5
std::vector<LayerSpec> backbone_specs()
{
    std::vector<LayerSpec> v;
    v.push_back(conv("conv1", 7, 3, 64, "bn_conv1", 2, 3, 1.0f));
    const int nblocks[4] = {3, 4, 23, 3}, mid[4] = {64, 128, 256, 512};
    int cin = 64;
    for (int st = 0; st < 4; ++st)
        for (int blk = 0; blk < nblocks[st]; ++blk) {
            const int f = mid[st], cout = 4 * f, stride = (blk == 0 && st > 0) ? 2 : 1;
            const std::string id = std::to_string(st + 2) + (char)('a' + blk) + "_branch";
            v.push_back(conv("res" + id + "2a", 1, cin, f, "bn" + id + "2a", stride, 0, 1.0f));
            v.push_back(conv("res" + id + "2b", 3, f, f, "bn" + id + "2b", 1, 1, 1.0f));
            v.push_back(conv("res" + id + "2c", 1, f, cout, "bn" + id + "2c", 1, 0, 0.5f));
            if (blk == 0) v.push_back(conv("res" + id + "1", 1, cin, cout, "bn" + id + "1", stride, 0, 0.7f));
            cin = cout;
        }
    const int cdim[4] = {256, 512, 1024, 2048};
    for (int i = 0; i < 4; ++i) v.push_back(conv("fpn_c" + std::to_string(i + 2) + "p" + std::to_string(i + 2), 1, cdim[i], 256, "", 1, 0, 0.7f));
    for (int i = 0; i < 4; ++i) v.push_back(conv("fpn_p" + std::to_string(i + 2), 3, 256, 256, "", 1, 1, 1.0f));
    return v;
}

// the RPN handle: shared 3x3 conv [512 x 2304]; class logits (6) and box deltas (12) as one GEMM of 64 rows.  The synthetic P levels are
// O(100) (the moulded input is in pixel units), and so is the conv output: the seeded class-logit rows are damped to logits of a few units
// (scores spread over (0, 1) instead of saturating at 0 / 1), the delta rows to |delta| ~ 0.1 (decoded boxes stay near their anchors)
std::vector<LayerSpec> rpn_specs()
{
    return {conv("rpn_conv_shared", 3, 256, 512, "", 1, 1, 1.0f),
            layer("rpn_class_raw+rpn_bbox_pred", {{"rpn_class_raw", {1, 1, 512, 6}, 0, 2e-4f}, {"rpn_bbox_pred", {1, 1, 512, 12}, 6, 2e-5f}}, "", 1, 0)};
}

// the detector handle: FC1, FC2, class logits + box deltas, 4 mask convs, transposed conv, mask logits.  Seeded at gain 1 except the output
// layers: the synthetic FC and mask-conv outputs are O(1000) (the pooled features carry the pixel-unit scale of the moulded input), so the
// class logits are damped to a few units (at gain 1 every softmax saturates; far below, the 81-way softmax stays near uniform and no ROI
// reaches the 0.7 confidence), the deltas to |delta| ~ 0.15 (refined boxes stay near their proposals), the mask logits to a few units
// (mask pixels on both sides of 0.5)
std::vector<LayerSpec> detector_specs()
{
    std::vector<LayerSpec> v;
    v.push_back(conv("mrcnn_class_conv1", 7, 256, 1024, "mrcnn_class_bn1", 1, 0, 1.0f));
    v.push_back(conv("mrcnn_class_conv2", 1, 1024, 1024, "mrcnn_class_bn2", 1, 0, 1.0f));
    v.push_back(layer("mrcnn_class_logits+mrcnn_bbox_fc", {{"mrcnn_class_logits", {1024, 81}, 0, 1e-3f}, {"mrcnn_bbox_fc", {1024, 324}, 81, 2e-5f}}, "", 1, 0));
    for (int i = 1; i <= 4; ++i)
        v.push_back(conv("mrcnn_mask_conv" + std::to_string(i), 3, 256, 256, "mrcnn_mask_bn" + std::to_string(i), 1, 1, 1.0f));
    v.push_back(layer("mrcnn_mask_deconv", {{"mrcnn_mask_deconv", {2, 2, 256, 256}, 0, 1.0f}}, "", 2, 0, true));
    v.push_back(conv("mrcnn_mask", 1, 256, 81, "", 1, 0, 1e-3f));
    return v;
}

const std::vector<LayerSpec>& specs(int part)
{
    static const std::vector<LayerSpec> t[3] = {backbone_specs(), rpn_specs(), detector_specs()};
    return t[part];
}

float bf16_rn(float f) { return __bfloat162float(__float2bfloat16(f)); }

// the relayout of one part into its layer's table, shared by the file (fold) and the seeded generator: row r < part_rows of the part is
// table row row0 + r and takes bf16_rn(wv(r, j)) in its first part_cols columns j, in that order; then its biases bv(r), in row order
template <typename WV, typename BV>
void relayout(const LayerSpec& s, const Part& pt, float* w, float* b, WV wv, BV bv)
{
    const long long rows = part_rows(s, pt), cols = part_cols(s, pt);
    for (long long r = 0; r < rows; ++r) {
        float* row = w + (size_t)(pt.row0 + r) * s.K;
        for (long long j = 0; j < cols; ++j) row[j] = bf16_rn(wv(r, j));
    }
    for (long long r = 0; r < rows; ++r) b[pt.row0 + r] = bv(r);
}

struct Lcg {
    uint32_t s;
    float urand() { s = s * 1664525u + 1013904223u; return (float)(s >> 8) * (1.0f / 16777216.0f) * 2.f - 1.f; }
};

// the seeded layer (tables zeroed by the caller): per part, He-style uniform weights of gain * sqrt(2 / K used), then biases of +-0.05
void seed_layer(const LayerSpec& s, Lcg& g, float* w, float* b)
{
    for (const Part& pt : s.parts) {
        const float sc = pt.gain * sqrtf(2.0f / (float)part_cols(s, pt));
        relayout(s, pt, w, b, [&](long long, long long) { return g.urand() * sc * 1.7320508f; }, [&](long long) { return g.urand() * 0.05f; });
        const long long cout = part_cout(s, pt);
        if (s.deconv)                    // all rows' biases are drawn, then every (dy, dx) takes the first one's
            for (long long r = cout; r < part_rows(s, pt); ++r) b[pt.row0 + r] = b[pt.row0 + r % cout];
    }
}

std::string shape_str(const std::vector<long long>& s)
{
    std::string r = "(";
    for (size_t i = 0; i < s.size(); ++i) r += (i ? ", " : "") + std::to_string(s[i]);
    return r + (s.size() == 1 ? ",)" : ")");
}

std::string printable(const std::string& s)      // a name from a damaged header: bytes outside printable ASCII as \xNN
{
    std::string r;
    for (unsigned char c : s) {
        char buf[8];
        if (c >= 0x20 && c < 0x7f) r += (char)c;
        else { snprintf(buf, sizeof buf, "\\x%02x", c); r += buf; }
    }
    return r;
}

// ---- the header: a JSON reader of exactly the safetensors grammar ----
struct Json {
    const char* p; const char* e;
    std::string err;
    void ws() { while (p < e && (*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r')) ++p; }
    bool lit(char c) { ws(); if (p < e && *p == c) { ++p; return true; } return false; }
    bool fail(const std::string& m) { if (err.empty()) err = m; return false; }
    bool expect(char c) { return lit(c) || fail(std::string("expected '") + c + "'"); }
    bool str(std::string& out)
    {
        out.clear();
        if (!lit('"')) return fail("expected a string");
        while (p < e && *p != '"') {
            unsigned char c = (unsigned char)*p++;
            if (c < 0x20) return fail("control character in a string");
            if (c != '\\') { out += (char)c; continue; }
            if (p >= e) break;
            c = (unsigned char)*p++;
            switch (c) {
            case '"': case '\\': case '/': out += (char)c; break;
            case 'b': out += '\b'; break;
            case 'f': out += '\f'; break;
            case 'n': out += '\n'; break;
            case 'r': out += '\r'; break;
            case 't': out += '\t'; break;
            case 'u': {
                if (e - p < 4) return fail("truncated \\u escape");
                unsigned v = 0;
                for (int i = 0; i < 4; ++i) {
                    const char h = *p++;
                    const int d = h >= '0' && h <= '9' ? h - '0' : h >= 'a' && h <= 'f' ? h - 'a' + 10 : h >= 'A' && h <= 'F' ? h - 'A' + 10 : -1;
                    if (d < 0) return fail("bad \\u escape");
                    v = v * 16 + d;
                }
                if (v >= 0xD800 && v < 0xE000) return fail("surrogate \\u escape");
                if (v < 0x80) out += (char)v;
                else if (v < 0x800) { out += (char)(0xC0 | (v >> 6)); out += (char)(0x80 | (v & 63)); }
                else { out += (char)(0xE0 | (v >> 12)); out += (char)(0x80 | ((v >> 6) & 63)); out += (char)(0x80 | (v & 63)); }
                break;
            }
            default: return fail("bad escape in a string");
            }
        }
        if (p >= e) return fail("unterminated string");
        ++p;
        return true;
    }
    bool uint(long long& v)                      // a non-negative integer below 2^53
    {
        ws();
        if (p >= e || *p < '0' || *p > '9') return fail("expected a non-negative integer");
        if (*p == '0' && p + 1 < e && p[1] >= '0' && p[1] <= '9') return fail("leading zero in an integer");
        v = 0;
        while (p < e && *p >= '0' && *p <= '9') {
            v = v * 10 + (*p++ - '0');
            if (v > (1ll << 53)) return fail("integer out of range");
        }
        if (p < e && (*p == '.' || *p == 'e' || *p == 'E')) return fail("expected an integer");
        return true;
    }
    bool uints(std::vector<long long>& v)
    {
        v.clear();
        if (!expect('[')) return false;
        if (lit(']')) return true;
        do {
            long long x;
            if (!uint(x)) return false;
            v.push_back(x);
            if (v.size() > 8) return fail("more than 8 dimensions");
        } while (lit(','));
        return expect(']');
    }
    bool tensor(Tensor& t)
    {
        if (!expect('{')) return false;
        bool dt = false, sh = false, off = false;
        do {
            std::string k;
            if (!str(k) || !expect(':')) return false;
            if (k == "dtype" && !dt) { dt = true; if (!str(t.dtype)) return false; }
            else if (k == "shape" && !sh) { sh = true; if (!uints(t.shape)) return false; }
            else if (k == "data_offsets" && !off) {
                off = true;
                std::vector<long long> o;
                if (!uints(o)) return false;
                if (o.size() != 2) return fail("data_offsets must be [begin, end]");
                t.begin = o[0]; t.end = o[1];
            } else return fail("unexpected or repeated field \"" + printable(k) + "\"");
        } while (lit(','));
        if (!expect('}')) return false;
        return (dt && sh && off) || fail("needs dtype, shape and data_offsets");
    }
    bool metadata()
    {
        if (!expect('{')) return false;
        if (lit('}')) return true;
        do {
            std::string k, v;
            if (!str(k) || !expect(':') || !str(v)) return false;
        } while (lit(','));
        return expect('}');
    }
};

struct WeightFile {
    std::string path;
    FILE* fp = nullptr;
    long long dataStart = 0, dataSize = 0;
    std::map<std::string, Tensor> tensors;
    std::string err;
    ~WeightFile() { if (fp) fclose(fp); }

    bool fail(const std::string& m) { err = path + ": " + m; return false; }
    bool failT(const std::string& name, const std::string& m) { return fail("tensor '" + printable(name) + "': " + m); }

    bool open(const char* p)
    {
        path = p ? p : "(null)";
        if (!p || !(fp = fopen(p, "rb"))) return fail("cannot open");
        if (fseeko(fp, 0, SEEK_END) != 0) return fail("cannot seek");
        const long long size = ftello(fp);
        uint8_t n8[8];
        if (size < 8 || fseeko(fp, 0, SEEK_SET) != 0 || fread(n8, 1, 8, fp) != 8) return fail("truncated: no 8-byte header length");
        unsigned long long n = 0;
        for (int i = 7; i >= 0; --i) n = (n << 8) | n8[i];
        if (n < 2 || n > 100000000ull) return fail("header length " + std::to_string(n) + " outside [2, 1e8]");
        if ((long long)n > size - 8) return fail("header length " + std::to_string(n) + " larger than the file (" + std::to_string(size) + " bytes)");
        std::vector<char> hdr(n);
        if (fread(hdr.data(), 1, n, fp) != n) return fail("cannot read the header");
        dataStart = 8 + (long long)n; dataSize = size - dataStart;
        Json j{hdr.data(), hdr.data() + n, ""};
        std::string entry, prev;                  // the entry being parsed, the last one parsed
        bool ok = j.expect('{');
        if (ok && !j.lit('}')) {
            do {
                prev.swap(entry);
                ok = j.str(entry) && j.expect(':');
                if (!ok) break;
                if (entry == "__metadata__") { ok = j.metadata(); if (!ok) break; continue; }
                Tensor t;
                ok = j.tensor(t);
                if (!ok) break;
                if (!tensors.emplace(entry, t).second) { j.fail("repeated name"); ok = false; break; }
            } while (j.lit(','));
            ok = ok && j.expect('}');
        }
        if (ok) { j.ws(); if (j.p != j.e) { j.fail("trailing bytes after the header object"); ok = false; } }
        if (!ok) {
            const std::string where = "header byte " + std::to_string(j.p - hdr.data()) + ": " + j.err;
            if (!entry.empty()) return failT(entry, "bad header JSON at " + where);
            return fail("bad header JSON" + (prev.empty() ? std::string() : " after tensor '" + printable(prev) + "'") + " at " + where);
        }
        for (const auto& kv : tensors) {
            const Tensor& t = kv.second;
            if (t.begin > t.end || t.end > dataSize)
                return failT(kv.first, "data_offsets [" + std::to_string(t.begin) + ", " + std::to_string(t.end) + "] outside the " +
                                           std::to_string(dataSize) + "-byte data section (truncated file?)");
        }
        return true;
    }

    // the F32 array `name` of exactly `shape`, as float
    bool read(const std::string& name, const std::vector<long long>& shape, std::vector<float>& out)
    {
        const auto it = tensors.find(name);
        if (it == tensors.end()) return failT(name, "missing");
        const Tensor& t = it->second;
        if (t.dtype != "F32") return failT(name, "dtype " + printable(t.dtype) + ", only F32 is read");
        if (t.shape != shape) return failT(name, "shape " + shape_str(t.shape) + ", the layer needs " + shape_str(shape));
        long long n = 1;
        for (long long d : shape) n *= d;
        if (t.end - t.begin != 4 * n)
            return failT(name, "data_offsets [" + std::to_string(t.begin) + ", " + std::to_string(t.end) + "] hold " + std::to_string(t.end - t.begin) +
                                   " bytes, shape " + shape_str(shape) + " of F32 needs " + std::to_string(4 * n));
        out.resize((size_t)n);
        if (fseeko(fp, dataStart + t.begin, SEEK_SET) != 0 || fread(out.data(), 4, (size_t)n, fp) != (size_t)n) return failT(name, "read failed");
        return true;                             // little-endian file, little-endian host
    }

    // R-FOLD + relayout of one handle layer into w [rows x K] and b [rows] (zero padded)
    bool fold(const LayerSpec& s, float* w, float* b)
    {
        std::vector<double> scale, shift;
        std::vector<float> kern, bias;
        memset(w, 0, (size_t)s.rows * s.K * sizeof(float));
        memset(b, 0, (size_t)s.rows * sizeof(float));
        for (const Part& pt : s.parts) {
            const long long cout = part_cout(s, pt), rows = part_rows(s, pt), cols = part_cols(s, pt);
            if (!read(pt.layer + "/kernel", pt.shape, kern) || !read(pt.layer + "/bias", {cout}, bias)) return false;
            scale.assign((size_t)cout, 1.0); shift.assign((size_t)cout, 0.0);
            if (!s.bn.empty()) {
                std::vector<float> g, be, m, v;
                if (!read(s.bn + "/gamma", {cout}, g) || !read(s.bn + "/beta", {cout}, be) || !read(s.bn + "/moving_mean", {cout}, m) ||
                    !read(s.bn + "/moving_variance", {cout}, v)) return false;
                for (long long o = 0; o < cout; ++o) {
                    scale[o] = (double)g[o] / sqrt((double)v[o] + 1e-3);
                    shift[o] = ((double)bias[o] - (double)m[o]) * scale[o] + (double)be[o];
                }
            } else
                for (long long o = 0; o < cout; ++o) shift[o] = bias[o];
            // (kh, kw, cin, cout) or (in, out): column j of output o is kern[j * cout + o]; the deconv's (kh, kw, out, in) is already
            // [row = (dy*kw + dx)*out + o][c]
            relayout(s, pt, w, b, [&](long long r, long long j) { return (float)((double)kern[s.deconv ? r * cols + j : j * rows + r] * scale[r % cout]); },
                     [&](long long r) { return (float)shift[r % cout]; });
        }
        return true;
    }
};

}  // namespace

namespace mfb {

static const char* const HANDLE_NAME[3] = {"backbone", "rpn", "detector"};

int mrcnn_num_layers(int part) { return (int)specs(part).size(); }

LayerGeom mrcnn_layer(int part, int i)
{
    const LayerSpec& s = specs(part)[i];
    const std::vector<long long>& sh = s.parts[0].shape;
    const int cin = (int)(s.deconv ? sh[3] : sh.size() == 4 ? sh[2] : sh[0]), k = sh.size() == 4 ? (int)sh[0] : 1;
    return {cin, s.rows, k, s.stride, s.pad, s.K};
}

// bf16 weights and fp32 biases onto the device, complete on return
static cudaError_t upload(const WeightStore& st, const std::vector<float>& w, const std::vector<float>& b, cudaStream_t s)
{
    std::vector<__nv_bfloat16> wbf(w.size());
    for (size_t i = 0; i < wbf.size(); ++i) wbf[i] = __float2bfloat16(w[i]);
    cudaError_t e = cudaMemcpyAsync(st.dW.p, wbf.data(), wbf.size() * sizeof(__nv_bfloat16), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(st.dB.p, b.data(), b.size() * sizeof(float), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    return e;
}

WeightStore::WeightStore(int part_, unsigned seed, cudaStream_t s) : part(part_)
{
    const std::vector<LayerSpec>& t = specs(part);
    size_t nw = 0, nb = 0;
    for (const LayerSpec& l : t) {
        assert(l.rows % 64 == 0 && l.K % 64 == 0);      // every table and bias starts 128-byte aligned (TMA maps of the GEMM's B operand)
        wOff.push_back(nw); bOff.push_back(nb);
        nw += (size_t)l.rows * l.K; nb += (size_t)l.rows;
    }
    hW.assign(nw, 0.f); hB.assign(nb, 0.f);
    Lcg g{seed ? seed : 1u};
    for (size_t i = 0; i < t.size(); ++i) seed_layer(t[i], g, &hW[wOff[i]], &hB[bOff[i]]);
    dW.alloc(nw); dB.alloc(nb);
    cudaCheck(upload(*this, hW, hB, s), "weight upload");
}

void WeightStore::load(const char* path, cudaStream_t s)
{
    const std::vector<LayerSpec>& t = specs(part);
    std::vector<float> w(hW.size()), b(hB.size());
    WeightFile f;
    bool ok = f.open(path);
    for (size_t i = 0; ok && i < t.size(); ++i) ok = f.fold(t[i], &w[wOff[i]], &b[bOff[i]]);
    if (!ok) throw CudaError{f.err};
    const cudaError_t e = upload(*this, w, b, s);
    if (e != cudaSuccess) throw CudaError{std::string(HANDLE_NAME[part]) + ": weight upload: " + cudaGetErrorString(e)};
    hW.swap(w); hB.swap(b);
}

void WeightStore::get(int i, float* w, float* b, int rows) const
{
    if (i < 0 || i >= (int)wOff.size()) throw CudaError{std::string(HANDLE_NAME[part]) + ": bad layer index"};
    const LayerSpec& l = specs(part)[i];
    if (rows < 0) rows = l.rows;
    if (w) memcpy(w, &hW[wOff[i]], (size_t)rows * l.K * sizeof(float));
    if (b) memcpy(b, &hB[bOff[i]], (size_t)rows * sizeof(float));
}

}  // namespace mfb

// one handle layer as the loaders fold it, without a CUDA device: dims = {rows, K}; w / bias NULL: only the dims
extern "C" int mf_mrcnn_read_layer(const char* path, const char* layer, float* w_rows_K, float* bias_rows, int* dims)
{
    MF_TRY
    for (int part = 0; part < 3; ++part)
        for (const LayerSpec& s : specs(part)) {
            if (!layer || s.name != layer) continue;
            if (dims) { dims[0] = s.rows; dims[1] = s.K; }
            if (!w_rows_K || !bias_rows) return 0;
            WeightFile f;
            if (!f.open(path) || !f.fold(s, w_rows_K, bias_rows)) throw mfb::CudaError{f.err};
            return 0;
        }
    throw mfb::CudaError{std::string("mrcnn_read_layer: no layer named '") + (layer ? layer : "(null)") + "'"};
    MF_CATCH(-1)
}
