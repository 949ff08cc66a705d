// mf_weights.cu -- pretrained Mask R-CNN weights from a safetensors file into the layer tables of the backbone, RPN and detector handles
// (host code only).  DESIGN §3c has the name table and the folding rule R-FOLD.
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
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <map>
#include <string>
#include <vector>

namespace {

struct Tensor { std::string dtype; std::vector<long long> shape; long long begin = 0, end = 0; };

// one source array of a handle layer: its Keras name, its Keras shape, the first GEMM row it fills
struct Part { std::string layer; std::vector<long long> shape; int row0; };
struct LayerSpec {
    std::string name;                 // the handle layer's name: the Keras layer, or "a+b" for two layers stacked in one GEMM
    std::vector<Part> parts;
    std::string bn;                   // BatchNorm layer folded into it ("" = none)
    int rows, K;                      // the handle's table: [rows x K], zero padded
    bool deconv;                      // Conv2DTranspose (kh, kw, out, in): row (dy*kw + dx)*out + o, column c; bias repeated per (dy, dx)
};

LayerSpec conv(const std::string& name, int kh, int kw, int cin, int cout, const std::string& bn, int rows, int K)
{
    LayerSpec s;
    s.name = name; s.parts = {{name, {kh, kw, cin, cout}, 0}}; s.bn = bn; s.rows = rows; s.K = K; s.deconv = false;
    return s;
}

int kpad(int K) { return (K + 63) / 64 * 64; }

// the backbone's layer table order (mf_backbone_create): conv1, per block branch2a, 2b, 2c (+ branch1 in block a), fpn_c2p2..c5p5, fpn_p2..p5
std::vector<LayerSpec> backbone_specs()
{
    std::vector<LayerSpec> v;
    v.push_back(conv("conv1", 7, 7, 3, 64, "bn_conv1", 64, kpad(7 * 7 * 3)));
    const int nblocks[4] = {3, 4, 23, 3}, mid[4] = {64, 128, 256, 512};
    int cin = 64;
    for (int st = 0; st < 4; ++st)
        for (int blk = 0; blk < nblocks[st]; ++blk) {
            const int f = mid[st], cout = 4 * f;
            const std::string id = std::to_string(st + 2) + (char)('a' + blk) + "_branch";
            v.push_back(conv("res" + id + "2a", 1, 1, cin, f, "bn" + id + "2a", f, kpad(cin)));
            v.push_back(conv("res" + id + "2b", 3, 3, f, f, "bn" + id + "2b", f, kpad(9 * f)));
            v.push_back(conv("res" + id + "2c", 1, 1, f, cout, "bn" + id + "2c", cout, kpad(f)));
            if (blk == 0) v.push_back(conv("res" + id + "1", 1, 1, cin, cout, "bn" + id + "1", cout, kpad(cin)));
            cin = cout;
        }
    const int cdim[4] = {256, 512, 1024, 2048};
    for (int i = 0; i < 4; ++i) v.push_back(conv("fpn_c" + std::to_string(i + 2) + "p" + std::to_string(i + 2), 1, 1, cdim[i], 256, "", 256, cdim[i]));
    for (int i = 0; i < 4; ++i) v.push_back(conv("fpn_p" + std::to_string(i + 2), 3, 3, 256, 256, "", 256, 9 * 256));
    return v;
}

// the RPN handle: shared 3x3 conv [512 x 2304]; class logits (6) and box deltas (12) as one GEMM of 64 rows
std::vector<LayerSpec> rpn_specs()
{
    LayerSpec head;
    head.name = "rpn_class_raw+rpn_bbox_pred";
    head.parts = {{"rpn_class_raw", {1, 1, 512, 6}, 0}, {"rpn_bbox_pred", {1, 1, 512, 12}, 6}};
    head.rows = 64; head.K = 512; head.deconv = false;
    return {conv("rpn_conv_shared", 3, 3, 256, 512, "", 512, 9 * 256), head};
}

// the detector handle, mf_heads.cu LAYERS order: FC1, FC2, class logits + box deltas, 4 mask convs, transposed conv, mask logits
std::vector<LayerSpec> detector_specs()
{
    std::vector<LayerSpec> v;
    v.push_back(conv("mrcnn_class_conv1", 7, 7, 256, 1024, "mrcnn_class_bn1", 1024, 7 * 7 * 256));
    v.push_back(conv("mrcnn_class_conv2", 1, 1, 1024, 1024, "mrcnn_class_bn2", 1024, 1024));
    LayerSpec head;
    head.name = "mrcnn_class_logits+mrcnn_bbox_fc";
    head.parts = {{"mrcnn_class_logits", {1024, 81}, 0}, {"mrcnn_bbox_fc", {1024, 324}, 81}};
    head.rows = 448; head.K = 1024; head.deconv = false;
    v.push_back(head);
    for (int i = 1; i <= 4; ++i)
        v.push_back(conv("mrcnn_mask_conv" + std::to_string(i), 3, 3, 256, 256, "mrcnn_mask_bn" + std::to_string(i), 256, 9 * 256));
    LayerSpec dec;
    dec.name = "mrcnn_mask_deconv"; dec.parts = {{"mrcnn_mask_deconv", {2, 2, 256, 256}, 0}}; dec.rows = 4 * 256; dec.K = 256; dec.deconv = true;
    v.push_back(dec);
    v.push_back(conv("mrcnn_mask", 1, 1, 256, 81, "", 128, 256));
    return v;
}

const std::vector<LayerSpec>& specs(int part)
{
    static const std::vector<LayerSpec> t[3] = {backbone_specs(), rpn_specs(), detector_specs()};
    return t[part];
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
            const long long cout = s.deconv ? pt.shape[2] : pt.shape.back();
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
            if (s.deconv) {                  // (kh, kw, out, in): already [row = (dy*kw + dx)*out + o][c]
                const long long cin = pt.shape[3], taps = pt.shape[0] * pt.shape[1];
                for (long long r = 0; r < taps * cout; ++r) {
                    for (long long c = 0; c < cin; ++c) w[r * s.K + c] = __bfloat162float(__float2bfloat16(kern[r * cin + c]));
                    b[r] = (float)shift[r % cout];
                }
                continue;
            }
            long long cols = 1;                  // (kh, kw, cin, cout) or (in, out): column j of output o is kern[j * cout + o]
            for (size_t d = 0; d + 1 < pt.shape.size(); ++d) cols *= pt.shape[d];
            for (long long o = 0; o < cout; ++o) {
                float* row = w + (size_t)(pt.row0 + o) * s.K;
                for (long long j = 0; j < cols; ++j) row[j] = __bfloat162float(__float2bfloat16((float)((double)kern[j * cout + o] * scale[o])));
                b[pt.row0 + o] = (float)shift[o];
            }
        }
        return true;
    }
};

}  // namespace

namespace mfb {

int mrcnn_layer_count(int part) { return (int)specs(part).size(); }

void mrcnn_layer_dims(int part, int i, int* rows, int* K)
{
    const LayerSpec& s = specs(part)[i];
    *rows = s.rows; *K = s.K;
}

int mrcnn_fold(const char* path, int part, float* const* w, float* const* b)
{
    WeightFile f;
    bool ok = f.open(path);
    for (size_t i = 0; ok && i < specs(part).size(); ++i) ok = f.fold(specs(part)[i], w[i], b[i]);
    if (!ok) { cnn_set_error(f.err.c_str()); return -1; }
    return 0;
}

}  // namespace mfb

// one handle layer as the loaders fold it, without a CUDA device: dims = {rows, K}; w / bias NULL: only the dims
extern "C" int mf_mrcnn_read_layer(const char* path, const char* layer, float* w_rows_K, float* bias_rows, int* dims)
{
    for (int part = 0; part < 3; ++part)
        for (const LayerSpec& s : specs(part)) {
            if (!layer || s.name != layer) continue;
            if (dims) { dims[0] = s.rows; dims[1] = s.K; }
            if (!w_rows_K || !bias_rows) return 0;
            WeightFile f;
            if (!f.open(path) || !f.fold(s, w_rows_K, bias_rows)) { mfb::cnn_set_error(f.err.c_str()); return -1; }
            return 0;
        }
    mfb::cnn_set_error((std::string("mrcnn_read_layer: no layer named '") + (layer ? layer : "(null)") + "'").c_str());
    return -1;
}
