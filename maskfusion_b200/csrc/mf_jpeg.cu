// mf_jpeg.cu -- baseline JPEG decoder for the loaders (host code only).
//
// The reference decodes JPEG colour with libjpeg (.klg: GUI/Tools/JPEGLoader.h:33-86, jpeg_read_scanlines with the library
// defaults; image directories: cv::imread, GUI/Tools/ImageLogReader.cpp:245).  libjpeg is not in this build, and a loader whose
// pixels differ from the reference's by decoder rounding would break the bit-exact association contract before the first kernel
// runs.  This is therefore a restatement of what libjpeg computes with its DEFAULT settings, not "a" JPEG decoder:
//   entropy decoding    ITU T.81 baseline / extended sequential, 8-bit, Huffman, restart intervals
//   inverse DCT         jidctint.c `jpeg_idct_islow` (JDCT_ISLOW): 13-bit constants, PASS1_BITS = 2, DESCALE rounding
//   chroma upsampling   jdsample.c fancy ("triangle") h2v1 / h2v2 (do_fancy_upsampling = TRUE), replicated image edges
//   colour conversion   jdcolor.c YCbCr -> RGB, 16-bit fixed-point tables with ONE_HALF rounding
// Pinned against OpenCV's decoder (libjpeg-turbo, bit-compatible with libjpeg for these methods) in tests/test_cpu_loader.py.
// Progressive, arithmetic-coded, 12-bit and CMYK files are refused.
#include "mf_kernels.h"
#include <stdint.h>
#include <string.h>
#include <string>
#include <vector>

namespace mfb {

namespace {

struct Huff { uint8_t bits[17]; uint8_t vals[256]; int mincode[17], maxcode[18], valptr[17]; bool present = false; };

struct Comp { int id = 0, h = 0, v = 0, tq = 0, td = 0, ta = 0; int inScan = 0; int wBlocks = 0, hBlocks = 0; std::vector<int16_t> coef; int dcPred = 0; int dsW = 0, dsH = 0; std::vector<uint8_t> plane; int planeW = 0, planeH = 0; };

struct BitReader {
    const uint8_t* p; const uint8_t* end; uint32_t buf = 0; int cnt = 0; bool hitMarker = false;
    int nextByte()
    {
        if (p >= end) return 0;
        int b = *p++;
        if (b == 0xFF) {
            if (p < end && *p == 0x00) { ++p; return 0xFF; }
            --p; hitMarker = true; return 0;                 // a marker: feed zeros (libjpeg does the same until the restart logic runs)
        }
        return b;
    }
    int bit()
    {
        if (cnt == 0) { buf = (uint32_t)(hitMarker ? 0 : nextByte()); cnt = 8; }
        --cnt;
        return (buf >> cnt) & 1;
    }
    int bitsN(int n) { int v = 0; while (n--) v = (v << 1) | bit(); return v; }
    void reset() { cnt = 0; buf = 0; hitMarker = false; }
};

void buildHuff(Huff& h)
{
    int code = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
        h.valptr[l] = k; h.mincode[l] = code;
        code += h.bits[l]; k += h.bits[l];
        h.maxcode[l] = h.bits[l] ? code - 1 : -1;
        code <<= 1;
    }
    h.maxcode[17] = 0x7fffffff;
    h.present = true;
}

int decodeSym(BitReader& br, const Huff& h)
{
    int code = 0;
    for (int l = 1; l <= 16; ++l) {
        code = (code << 1) | br.bit();
        if (h.maxcode[l] >= 0 && code <= h.maxcode[l] && code >= h.mincode[l]) return h.vals[h.valptr[l] + code - h.mincode[l]];
    }
    return -1;
}

inline int extend(int v, int t) { return v < (1 << (t - 1)) ? v - (1 << t) + 1 : v; }

const int zigzag[64] = {0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
                        35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// jidctint.c: jpeg_idct_islow
#define CONST_BITS 13
#define PASS1_BITS 2
#define DESCALE(x, n) (((x) + (1 << ((n)-1))) >> (n))
inline uint8_t rangeLimit(int v) { v += 128; return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

void idctIslow(const int16_t* coef, const uint16_t* q, uint8_t* out, int stride)
{
    const int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299, F1847 = 15137, F1961 = 16069,
              F2053 = 16819, F2562 = 20995, F3072 = 25172;
    int ws[64];
    for (int c = 0; c < 8; ++c) {
        const int16_t* in = coef + c; const uint16_t* qq = q + c; int* w = ws + c;
        int z2 = in[16] * qq[16], z3 = in[48] * qq[48];
        int z1 = (z2 + z3) * F0541;
        int tmp2 = z1 + z3 * (-F1847), tmp3 = z1 + z2 * F0765;
        z2 = in[0] * qq[0]; z3 = in[32] * qq[32];
        int tmp0 = (z2 + z3) << CONST_BITS, tmp1 = (z2 - z3) << CONST_BITS;
        int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
        tmp0 = in[56] * qq[56]; tmp1 = in[40] * qq[40]; tmp2 = in[24] * qq[24]; tmp3 = in[8] * qq[8];
        z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2; int z4 = tmp1 + tmp3;
        int z5 = (z3 + z4) * F1175;
        tmp0 *= F0298; tmp1 *= F2053; tmp2 *= F3072; tmp3 *= F1501;
        z1 *= -F0899; z2 *= -F2562; z3 *= -F1961; z4 *= -F0390;
        z3 += z5; z4 += z5;
        tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
        w[0] = DESCALE(tmp10 + tmp3, CONST_BITS - PASS1_BITS); w[56] = DESCALE(tmp10 - tmp3, CONST_BITS - PASS1_BITS);
        w[8] = DESCALE(tmp11 + tmp2, CONST_BITS - PASS1_BITS); w[48] = DESCALE(tmp11 - tmp2, CONST_BITS - PASS1_BITS);
        w[16] = DESCALE(tmp12 + tmp1, CONST_BITS - PASS1_BITS); w[40] = DESCALE(tmp12 - tmp1, CONST_BITS - PASS1_BITS);
        w[24] = DESCALE(tmp13 + tmp0, CONST_BITS - PASS1_BITS); w[32] = DESCALE(tmp13 - tmp0, CONST_BITS - PASS1_BITS);
    }
    for (int r = 0; r < 8; ++r) {
        const int* w = ws + r * 8; uint8_t* o = out + r * stride;
        int z2 = w[2], z3 = w[6];
        int z1 = (z2 + z3) * F0541;
        int tmp2 = z1 + z3 * (-F1847), tmp3 = z1 + z2 * F0765;
        int tmp0 = (w[0] + w[4]) << CONST_BITS, tmp1 = (w[0] - w[4]) << CONST_BITS;
        int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
        tmp0 = w[7]; tmp1 = w[5]; tmp2 = w[3]; tmp3 = w[1];
        z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2; int z4 = tmp1 + tmp3;
        int z5 = (z3 + z4) * F1175;
        tmp0 *= F0298; tmp1 *= F2053; tmp2 *= F3072; tmp3 *= F1501;
        z1 *= -F0899; z2 *= -F2562; z3 *= -F1961; z4 *= -F0390;
        z3 += z5; z4 += z5;
        tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
        const int S = CONST_BITS + PASS1_BITS + 3;
        o[0] = rangeLimit(DESCALE(tmp10 + tmp3, S)); o[7] = rangeLimit(DESCALE(tmp10 - tmp3, S));
        o[1] = rangeLimit(DESCALE(tmp11 + tmp2, S)); o[6] = rangeLimit(DESCALE(tmp11 - tmp2, S));
        o[2] = rangeLimit(DESCALE(tmp12 + tmp1, S)); o[5] = rangeLimit(DESCALE(tmp12 - tmp1, S));
        o[3] = rangeLimit(DESCALE(tmp13 + tmp0, S)); o[4] = rangeLimit(DESCALE(tmp13 - tmp0, S));
    }
}

inline uint16_t be16(const uint8_t* p) { return (uint16_t)((p[0] << 8) | p[1]); }

}  // namespace

// -> interleaved 8-bit RGB (3 channels, libjpeg's JCS_RGB order) or gray replicated to 3 channels
bool decodeJPEG(const uint8_t* data, size_t size, int& W, int& H, std::vector<uint8_t>& rgb, std::string& err)
{
    if (size < 4 || data[0] != 0xFF || data[1] != 0xD8) { err = "not a JPEG stream"; return false; }
    uint16_t qt[4][64]; bool qtPresent[4] = {false, false, false, false};
    Huff dc[4], ac[4];
    std::vector<Comp> comps;
    int restartInterval = 0, hmax = 1, vmax = 1;
    W = H = 0;
    size_t pos = 2;
    bool gotSOF = false;
    while (pos + 4 <= size) {
        if (data[pos] != 0xFF) { ++pos; continue; }
        const int m = data[pos + 1];
        if (m == 0xFF) { ++pos; continue; }
        pos += 2;
        if (m == 0xD8 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) continue;
        if (m == 0xD9) break;
        if (pos + 2 > size) break;
        const int len = be16(data + pos);
        if (len < 2 || pos + len > size) { err = "JPEG: truncated marker segment"; return false; }
        const uint8_t* seg = data + pos + 2; const int n = len - 2;
        if (m == 0xDB) {                                                            // DQT
            int i = 0;
            while (i < n) {
                const int pq = seg[i] >> 4, tq = seg[i] & 15; ++i;
                if (tq > 3 || i + (pq ? 128 : 64) > n) { err = "JPEG: bad DQT"; return false; }
                for (int k = 0; k < 64; ++k) { qt[tq][zigzag[k]] = pq ? be16(seg + i + 2 * k) : seg[i + k]; }
                i += pq ? 128 : 64; qtPresent[tq] = true;
            }
        } else if (m == 0xC0 || m == 0xC1) {                                        // SOF0 / SOF1 (Huffman, sequential)
            if (n < 6 || seg[0] != 8) { err = "JPEG: only 8-bit samples are supported"; return false; }
            H = be16(seg + 1); W = be16(seg + 3);
            const int nc = seg[5];
            if (!(nc == 1 || nc == 3) || n < 6 + 3 * nc || W <= 0 || H <= 0) { err = "JPEG: unsupported number of components"; return false; }
            if (W > 16384 || H > 16384) { err = "JPEG: image side above 16384"; return false; }
            comps.resize(nc);
            for (int c = 0; c < nc; ++c) {
                comps[c].id = seg[6 + 3 * c]; comps[c].h = seg[7 + 3 * c] >> 4; comps[c].v = seg[7 + 3 * c] & 15; comps[c].tq = seg[8 + 3 * c];
                if (comps[c].h < 1 || comps[c].v < 1 || comps[c].tq > 3) { err = "JPEG: bad component"; return false; }
                hmax = comps[c].h > hmax ? comps[c].h : hmax; vmax = comps[c].v > vmax ? comps[c].v : vmax;
            }
            gotSOF = true;
        } else if (m == 0xC2 || (m >= 0xC3 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC)) {
            err = "JPEG: progressive / lossless / arithmetic-coded streams are not supported"; return false;
        } else if (m == 0xC4) {                                                     // DHT
            int i = 0;
            while (i + 17 <= n) {
                const int tc = seg[i] >> 4, th = seg[i] & 15; ++i;
                if (tc > 1 || th > 3) { err = "JPEG: bad DHT"; return false; }
                Huff& h = tc ? ac[th] : dc[th];
                int total = 0; h.bits[0] = 0;
                for (int l = 1; l <= 16; ++l) { h.bits[l] = seg[i + l - 1]; total += h.bits[l]; }
                i += 16;
                if (total > 256 || i + total > n) { err = "JPEG: bad DHT"; return false; }
                memcpy(h.vals, seg + i, total); i += total;
                buildHuff(h);
            }
        } else if (m == 0xDD) { if (n >= 2) restartInterval = be16(seg); }          // DRI
        else if (m == 0xDA) {                                                        // SOS: the (single) scan follows
            if (!gotSOF) { err = "JPEG: scan before frame header"; return false; }
            if (n < 1) { err = "JPEG: empty scan header"; return false; }
            const int ns = seg[0];
            if (ns != (int)comps.size() || n < 1 + 2 * ns + 3) { err = "JPEG: non-interleaved multi-scan files are not supported"; return false; }
            for (int k = 0; k < ns; ++k) {
                const int cid = seg[1 + 2 * k];
                const int td = seg[2 + 2 * k] >> 4, ta = seg[2 + 2 * k] & 15;
                if (td > 3 || ta > 3) { err = "JPEG: scan selects a Huffman table outside 0..3"; return false; }
                // the first frame component with this id that no earlier scan entry took (duplicate ids in the SOF stay distinct)
                bool found = false;
                for (auto& c : comps) if (c.id == cid && !c.inScan) { c.td = td; c.ta = ta; c.inScan = 1; found = true; break; }
                if (!found) { err = "JPEG: scan references an unknown component"; return false; }
            }
            for (auto& c : comps) if (!c.inScan) { err = "JPEG: a frame component is missing from the scan"; return false; }
            pos += len;
            break;
        }
        pos += len;
    }
    if (!gotSOF || pos >= size) { err = "JPEG: no image data"; return false; }
    if (comps.size() == 3 && !(comps[1].h == 1 && comps[1].v == 1 && comps[2].h == 1 && comps[2].v == 1 &&
                               ((hmax == 1 && vmax == 1) || (hmax == 2 && vmax == 1) || (hmax == 2 && vmax == 2)))) {
        err = "JPEG: only 4:4:4, 4:2:2 and 4:2:0 chroma sampling are supported"; return false;
    }
    if (comps.size() == 1) { comps[0].h = comps[0].v = 1; hmax = vmax = 1; }        // a single-component scan is never interleaved
    const int mcuW = 8 * hmax, mcuH = 8 * vmax;
    const int mcusX = (W + mcuW - 1) / mcuW, mcusY = (H + mcuH - 1) / mcuH;
    for (auto& c : comps) {
        if (!qtPresent[c.tq] || !dc[c.td].present || !ac[c.ta].present) { err = "JPEG: missing quantisation / Huffman table"; return false; }
        c.wBlocks = mcusX * c.h; c.hBlocks = mcusY * c.v;
        c.planeW = c.wBlocks * 8; c.planeH = c.hBlocks * 8;
        c.plane.assign((size_t)c.planeW * c.planeH, 0);
        c.dsW = (W * c.h + hmax - 1) / hmax; c.dsH = (H * c.v + vmax - 1) / vmax;   // downsampled_width / _height (jdmaster.c)
        c.dcPred = 0;
    }
    // ---- entropy decoding + IDCT, MCU by MCU ----
    BitReader br; br.p = data + pos; br.end = data + size;
    int16_t block[64];
    int restartsLeft = restartInterval;
    for (int my = 0; my < mcusY; ++my)
        for (int mx = 0; mx < mcusX; ++mx) {
            if (restartInterval && restartsLeft == 0) {
                // byte-align, expect RSTn
                br.reset();
                while (br.p + 1 < br.end && !(br.p[0] == 0xFF && br.p[1] >= 0xD0 && br.p[1] <= 0xD7)) ++br.p;
                if (br.p + 1 < br.end) br.p += 2;
                for (auto& c : comps) c.dcPred = 0;
                restartsLeft = restartInterval;
            }
            for (auto& c : comps)
                for (int by = 0; by < c.v; ++by)
                    for (int bx = 0; bx < c.h; ++bx) {
                        memset(block, 0, sizeof block);
                        int t = decodeSym(br, dc[c.td]);
                        if (t < 0 || t > 11) { err = "JPEG: corrupt DC coefficient"; return false; }
                        int diff = t ? extend(br.bitsN(t), t) : 0;
                        c.dcPred += diff; block[0] = (int16_t)c.dcPred;
                        for (int k = 1; k < 64;) {
                            int rs = decodeSym(br, ac[c.ta]);
                            if (rs < 0) { err = "JPEG: corrupt AC coefficient"; return false; }
                            int r = rs >> 4, s = rs & 15;
                            if (s == 0) { if (r == 15) { k += 16; continue; } break; }
                            k += r;
                            if (k > 63) { err = "JPEG: corrupt AC run"; return false; }
                            block[zigzag[k]] = (int16_t)extend(br.bitsN(s), s);
                            ++k;
                        }
                        const int px = (mx * c.h + bx) * 8, py = (my * c.v + by) * 8;
                        idctIslow(block, qt[c.tq], &c.plane[(size_t)py * c.planeW + px], c.planeW);
                    }
            if (restartInterval) --restartsLeft;
        }
    // ---- upsampling (jdsample.c, fancy) + colour conversion (jdcolor.c) ----
    rgb.assign((size_t)W * H * 3, 0);
    if (comps.size() == 1) {
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x) { uint8_t v = comps[0].plane[(size_t)y * comps[0].planeW + x]; uint8_t* o = &rgb[((size_t)y * W + x) * 3]; o[0] = o[1] = o[2] = v; }
        return true;
    }
    const bool h2 = hmax == 2, v2 = vmax == 2;
    std::vector<uint8_t> up[2];
    for (int ci = 1; ci <= 2; ++ci) {
        const Comp& c = comps[ci];
        std::vector<uint8_t>& u = up[ci - 1];
        if (!h2) { u.clear(); continue; }
        const int dw = c.dsW, dh = c.dsH, outW = dw * 2;
        u.assign((size_t)outW * H + outW, 0);
        auto rowPtr = [&](int r) { r = r < 0 ? 0 : (r >= dh ? dh - 1 : r); return &c.plane[(size_t)r * c.planeW]; };   // replicated top / bottom rows (jdmainct.c)
        if (!v2) {                                                                     // h2v1_fancy_upsample
            for (int y = 0; y < H; ++y) {
                const uint8_t* in = rowPtr(y); uint8_t* o = &u[(size_t)y * outW];
                if (dw == 1) { o[0] = o[1] = in[0]; continue; }
                int inv = in[0];
                o[0] = (uint8_t)inv; o[1] = (uint8_t)((inv * 3 + in[1] + 2) >> 2);
                for (int i = 1; i < dw - 1; ++i) { inv = in[i] * 3; o[2 * i] = (uint8_t)((inv + in[i - 1] + 1) >> 2); o[2 * i + 1] = (uint8_t)((inv + in[i + 1] + 2) >> 2); }
                inv = in[dw - 1];
                o[2 * (dw - 1)] = (uint8_t)((inv * 3 + in[dw - 2] + 1) >> 2); o[2 * (dw - 1) + 1] = (uint8_t)inv;
            }
        } else {                                                                       // h2v2_fancy_upsample
            for (int y = 0; y < H; ++y) {
                const int r0 = y >> 1, r1 = (y & 1) ? r0 + 1 : r0 - 1;               // nearest input row, next nearest (above for even output rows)
                const uint8_t* in0 = rowPtr(r0); const uint8_t* in1 = rowPtr(r1); uint8_t* o = &u[(size_t)y * outW];
                if (dw == 1) { int t = in0[0] * 3 + in1[0]; o[0] = (uint8_t)((t * 4 + 8) >> 4); o[1] = (uint8_t)((t * 4 + 7) >> 4); continue; }
                int thiscol = in0[0] * 3 + in1[0], nextcol = in0[1] * 3 + in1[1], lastcol;
                o[0] = (uint8_t)((thiscol * 4 + 8) >> 4); o[1] = (uint8_t)((thiscol * 3 + nextcol + 7) >> 4);
                lastcol = thiscol; thiscol = nextcol;
                for (int i = 1; i < dw - 1; ++i) {
                    nextcol = in0[i + 1] * 3 + in1[i + 1];
                    o[2 * i] = (uint8_t)((thiscol * 3 + lastcol + 8) >> 4); o[2 * i + 1] = (uint8_t)((thiscol * 3 + nextcol + 7) >> 4);
                    lastcol = thiscol; thiscol = nextcol;
                }
                o[2 * (dw - 1)] = (uint8_t)((thiscol * 3 + lastcol + 8) >> 4); o[2 * (dw - 1) + 1] = (uint8_t)((thiscol * 4 + 7) >> 4);
            }
        }
    }
    // jdcolor.c build_ycc_rgb_table
    struct YccTables { int crR[256], cbB[256], crG[256], cbG[256]; };
    static const YccTables tab = [] {
        YccTables t;
        for (int i = 0; i < 256; ++i) {
            const int x = i - 128;
            t.crR[i] = (int)((91881LL * x + 32768) >> 16);        // FIX(1.40200)
            t.cbB[i] = (int)((116130LL * x + 32768) >> 16);       // FIX(1.77200)
            t.crG[i] = -46802 * x;                                // FIX(0.71414)
            t.cbG[i] = -22554 * x + 32768;                        // FIX(0.34414) + ONE_HALF
        }
        return t;
    }();
    const Comp& Y = comps[0];
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            const int yy = Y.plane[(size_t)y * Y.planeW + x];
            int cb, cr;
            if (h2) { const int outW = comps[1].dsW * 2; cb = up[0][(size_t)y * outW + x]; cr = up[1][(size_t)y * (comps[2].dsW * 2) + x]; }
            else { cb = comps[1].plane[(size_t)y * comps[1].planeW + x]; cr = comps[2].plane[(size_t)y * comps[2].planeW + x]; }
            int r = yy + tab.crR[cr], g = yy + ((tab.cbG[cb] + tab.crG[cr]) >> 16), b = yy + tab.cbB[cb];
            uint8_t* o = &rgb[((size_t)y * W + x) * 3];
            o[0] = (uint8_t)(r < 0 ? 0 : (r > 255 ? 255 : r)); o[1] = (uint8_t)(g < 0 ? 0 : (g > 255 ? 255 : g)); o[2] = (uint8_t)(b < 0 ? 0 : (b > 255 ? 255 : b));
        }
    return true;
}

}  // namespace mfb

// test hook behind the C ABI: decode a JPEG byte stream to RGB (out must hold width*height*3 bytes; call with out == NULL for the size)
extern "C" int mf_decode_jpeg(const uint8_t* data, int size, uint8_t* out, int capacity, int* width, int* height)
{
    MF_TRY
    if (!data || size <= 0) { mf_set_error("decode_jpeg: empty input"); return -1; }
    int W = 0, H = 0; std::vector<uint8_t> rgb; std::string err;
    if (!mfb::decodeJPEG(data, (size_t)size, W, H, rgb, err)) { mf_set_error(err); return -2; }
    if (width) *width = W;
    if (height) *height = H;
    if (out) {
        if ((size_t)capacity < rgb.size()) { mf_set_error("decode_jpeg: output buffer too small"); return -3; }
        memcpy(out, rgb.data(), rgb.size());
    }
    return 0;
    MF_CATCH(-4)
}
