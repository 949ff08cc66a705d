// mf_loader.cu -- image-directory loader behind the C ABI (host code only).
//   mf_dir_*  <-  ImageLogReader  (GUI/Tools/ImageLogReader.{h,cpp}; constructed at GUI/MainController.cpp:150-176 for "-dir")
// File discovery (prefix + one extension per stream, start index 0 or 1, zero-padded index of width indexW), the default
// "Color"/"Depth"/"Mask" prefixes when directories overlap, the mask description file (class ids + boxes), the depth
// conversions and the timestamps (index * 1000 / 24 Hz, :283) follow the reference.  The reference decodes with OpenCV
// (cv::imread); OpenCV, libpng, libjpeg and OpenEXR do not exist in this build, so PNG (zlib is here), binary PNM, baseline JPEG and
// scan-line OpenEXR are decoded in-tree and the rest is refused with a message:
//   colour  .png .ppm .jpg (-> 8-bit RGB in file order: cv::imread gives BGR and the reader swaps unconditionally, :247-248; JPEG: mf_jpeg.cu)
//   depth   .png 16-bit gray (-> 0.001f * v, :262-268); .exr scan-line HALF/FLOAT, NONE/RLE/ZIPS/ZIP (-> the gray channel, or B of R,G,B: :253-258)
//   mask    .png / .pgm 8-bit gray (cv::IMREAD_GRAYSCALE of a gray file is the identity)
// Unlike KlgLogReader, hasMore() lets the LAST frame through (currentFrame starts at -1, :145,:326).
// The reference's background buffering thread (:203-220) is an I/O detail and is not reproduced: frames are decoded on demand.
#include "../../include/maskfusion_b200.h"
#include "mf_boxes.cuh"
#include "mf_kernels.h"
#include <dirent.h>
#include <stdio.h>
#include <stdint.h>
#include <string.h>
#include <sys/stat.h>
#include <zlib.h>
#include <algorithm>
#include <cmath>
#include <memory>
#include <string>
#include <vector>

#define MF_MAX_IMAGE_SIDE 16384          // decoders refuse larger headers before allocating (a crafted IHDR must not throw across the C ABI)
namespace mfb { bool decodeJPEG(const uint8_t* data, size_t size, int& W, int& H, std::vector<uint8_t>& rgb, std::string& err); }   // mf_jpeg.cu

namespace {

struct Image { int w = 0, h = 0, channels = 0, bits = 0; std::vector<uint8_t> data; };   // 16-bit samples in host byte order

bool readFile(const std::string& path, std::vector<uint8_t>& out)
{
    FILE* fp = fopen(path.c_str(), "rb");
    if (!fp) return false;
    fseek(fp, 0, SEEK_END); long n = ftell(fp); fseek(fp, 0, SEEK_SET);
    out.resize(n > 0 ? (size_t)n : 0);
    bool ok = n <= 0 || fread(out.data(), 1, (size_t)n, fp) == (size_t)n;
    fclose(fp);
    return ok;
}

uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }

// PNG (ISO/IEC 15948): non-interlaced, colour types 0/2/3/4/6, bit depths 8/16 (1/2/4 for gray and palette)
bool decodePNG(const std::vector<uint8_t>& f, Image& im, std::string& err)
{
    static const uint8_t sig[8] = {137, 80, 78, 71, 13, 10, 26, 10};
    if (f.size() < 33 || memcmp(f.data(), sig, 8) != 0) { err = "not a PNG file"; return false; }
    size_t pos = 8;
    int W = 0, H = 0, bits = 0, ctype = 0, interlace = 0;
    std::vector<uint8_t> idat, plte;
    bool gotHdr = false;
    while (pos + 12 <= f.size()) {
        uint32_t len = be32(&f[pos]);
        const uint8_t* type = &f[pos + 4];
        if (pos + 12 + (size_t)len > f.size()) { err = "truncated PNG chunk"; return false; }
        const uint8_t* d = &f[pos + 8];
        if (!memcmp(type, "IHDR", 4)) {
            if (len < 13) { err = "bad IHDR"; return false; }
            W = (int)be32(d); H = (int)be32(d + 4); bits = d[8]; ctype = d[9]; interlace = d[12]; gotHdr = true;
        } else if (!memcmp(type, "PLTE", 4)) plte.assign(d, d + len);
        else if (!memcmp(type, "IDAT", 4)) idat.insert(idat.end(), d, d + len);
        else if (!memcmp(type, "IEND", 4)) break;
        pos += 12 + (size_t)len;
    }
    if (!gotHdr || W <= 0 || H <= 0) { err = "PNG without a valid IHDR"; return false; }
    if (W > MF_MAX_IMAGE_SIDE || H > MF_MAX_IMAGE_SIDE) { err = "PNG: image side above 16384"; return false; }
    if (interlace) { err = "interlaced PNG is not supported"; return false; }
    int ch = ctype == 0 ? 1 : ctype == 2 ? 3 : ctype == 3 ? 1 : ctype == 4 ? 2 : ctype == 6 ? 4 : 0;
    if (!ch || !(bits == 8 || bits == 16 || ((ctype == 0 || ctype == 3) && (bits == 1 || bits == 2 || bits == 4)))) { err = "unsupported PNG colour type / bit depth"; return false; }
    const size_t bpp = std::max<size_t>(1, (size_t)ch * bits / 8);            // filter distance in bytes
    const size_t rowBytes = ((size_t)W * ch * bits + 7) / 8;
    std::vector<uint8_t> raw((rowBytes + 1) * (size_t)H);
    unsigned long rawLen = (unsigned long)raw.size();
    if (uncompress(raw.data(), &rawLen, idat.data(), (unsigned long)idat.size()) != Z_OK || rawLen != raw.size()) { err = "PNG: zlib stream does not decode to the image size"; return false; }
    std::vector<uint8_t> pix(rowBytes * (size_t)H);
    for (int y = 0; y < H; ++y) {
        const uint8_t ft = raw[(rowBytes + 1) * y];
        const uint8_t* src = &raw[(rowBytes + 1) * y + 1];
        uint8_t* cur = &pix[rowBytes * y];
        const uint8_t* up = y ? &pix[rowBytes * (y - 1)] : nullptr;
        for (size_t i = 0; i < rowBytes; ++i) {
            const int a = i >= bpp ? cur[i - bpp] : 0, b = up ? up[i] : 0, c = (up && i >= bpp) ? up[i - bpp] : 0;
            int v = src[i];
            switch (ft) {
                case 0: break;
                case 1: v += a; break;
                case 2: v += b; break;
                case 3: v += (a + b) >> 1; break;
                case 4: { int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c); v += (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c); break; }
                default: err = "PNG: bad filter type"; return false;
            }
            cur[i] = (uint8_t)v;
        }
    }
    // unpack to 8- or 16-bit samples, expand palette / low bit depths
    im.w = W; im.h = H;
    if (ctype == 3) {
        im.channels = 3; im.bits = 8; im.data.resize((size_t)W * H * 3);
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x) {
                int idx;
                if (bits == 8) idx = pix[rowBytes * y + x];
                else { int per = 8 / bits, sh = (per - 1 - x % per) * bits; idx = (pix[rowBytes * y + x / per] >> sh) & ((1 << bits) - 1); }
                for (int c = 0; c < 3; ++c) im.data[((size_t)y * W + x) * 3 + c] = (size_t)idx * 3 + c < plte.size() ? plte[idx * 3 + c] : 0;
            }
        return true;
    }
    im.channels = ch;
    if (bits < 8) {          // gray 1/2/4 -> 8 bit, scaled to the full range like libpng's expand
        im.bits = 8; im.data.resize((size_t)W * H);
        const int per = 8 / bits, maxv = (1 << bits) - 1;
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x) { int sh = (per - 1 - x % per) * bits; int v = (pix[rowBytes * y + x / per] >> sh) & maxv; im.data[(size_t)y * W + x] = (uint8_t)(v * 255 / maxv); }
        return true;
    }
    im.bits = bits;
    if (bits == 8) { im.data.swap(pix); return true; }
    im.data.resize(pix.size());
    for (size_t i = 0; i + 1 < pix.size(); i += 2) { uint16_t v = (uint16_t)((pix[i] << 8) | pix[i + 1]); memcpy(&im.data[i], &v, 2); }   // big endian -> host
    return true;
}

// binary PNM: P5 (gray) / P6 (rgb), maxval < 65536
bool decodePNM(const std::vector<uint8_t>& f, Image& im, std::string& err)
{
    if (f.size() < 7 || f[0] != 'P' || (f[1] != '5' && f[1] != '6')) { err = "not a binary PGM/PPM file"; return false; }
    size_t pos = 2; long vals[3]; int got = 0;
    while (got < 3 && pos < f.size()) {
        if (f[pos] == '#') { while (pos < f.size() && f[pos] != '\n') ++pos; continue; }
        if (isspace(f[pos])) { ++pos; continue; }
        long v = 0; bool any = false;
        while (pos < f.size() && isdigit(f[pos])) { v = v * 10 + (f[pos] - '0'); if (v > 65535) v = 65536; ++pos; any = true; }
        if (!any) { err = "bad PNM header"; return false; }
        vals[got++] = v;
    }
    if (got < 3 || pos >= f.size()) { err = "bad PNM header"; return false; }
    ++pos;   // single whitespace after maxval
    if (vals[0] > MF_MAX_IMAGE_SIDE || vals[1] > MF_MAX_IMAGE_SIDE || vals[2] < 1 || vals[2] > 65535) { err = "PNM: image side above 16384 or bad maxval"; return false; }
    im.w = (int)vals[0]; im.h = (int)vals[1]; im.channels = f[1] == '6' ? 3 : 1; im.bits = vals[2] > 255 ? 16 : 8;
    const size_t n = (size_t)im.w * im.h * im.channels * (im.bits / 8);
    if (im.w <= 0 || im.h <= 0 || pos + n > f.size()) { err = "truncated PNM data"; return false; }
    im.data.assign(f.begin() + pos, f.begin() + pos + n);
    if (im.bits == 16) for (size_t i = 0; i + 1 < n; i += 2) { uint16_t v = (uint16_t)((im.data[i] << 8) | im.data[i + 1]); memcpy(&im.data[i], &v, 2); }
    return true;
}

// OpenEXR scan-line images (depth of the synthetic datasets; the reference reads them with cv::imread(IMREAD_UNCHANGED), ImageLogReader.cpp:251).
// In-tree decoder of the subset a depth image uses: single-part scan-line files, compression NONE / RLE / ZIPS / ZIP, HALF or FLOAT
// channels, no sub-sampling.  The depth is what the reference takes from OpenCV's result (:253-258): the only channel of a gray file
// (CV_32FC1) or element [0] of a CV_32FC3 pixel, which in OpenCV's BGR order is the file's B channel.  Tiled, multi-part, deep and
// PIZ / PXR24 / B44 / DWA files are refused with a message naming the feature.
float halfToFloat(uint16_t h)
{
    const uint32_t sign = (uint32_t)(h >> 15) << 31, exp = (h >> 10) & 0x1fu, man = h & 0x3ffu;
    uint32_t bits;
    if (exp == 0) {
        if (man == 0) bits = sign;
        else { int e = -1; uint32_t m = man; do { ++e; m <<= 1; } while (!(m & 0x400u)); bits = sign | ((uint32_t)(127 - 15 - e) << 23) | ((m & 0x3ffu) << 13); }
    } else if (exp == 31) bits = sign | 0x7f800000u | (man << 13);
    else bits = sign | ((exp + 112u) << 23) | (man << 13);
    float f; memcpy(&f, &bits, 4); return f;
}

bool decodeEXRDepth(const std::vector<uint8_t>& f, int& W, int& H, std::vector<float>& depth, std::string& err)
{
    size_t pos = 0;
    auto need = [&](size_t n) { return pos + n <= f.size(); };
    auto rd32 = [&](size_t at) { uint32_t v; memcpy(&v, &f[at], 4); return v; };
    if (f.size() < 8 || rd32(0) != 20000630u) { err = "not an OpenEXR file"; return false; }
    const uint32_t ver = rd32(4);
    if ((ver & 0xffu) != 2) { err = "EXR: unsupported file version"; return false; }
    if (ver & 0x200u) { err = "EXR: tiled files are not supported"; return false; }
    if (ver & 0x1800u) { err = "EXR: deep / multi-part files are not supported"; return false; }
    pos = 8;
    struct Chan { std::string name; int type; int xs, ys; };
    std::vector<Chan> chans;
    int compression = -1, lineOrder = 0; int dw[4] = {0, 0, -1, -1}; bool haveDW = false;
    for (;;) {
        size_t e = pos; while (e < f.size() && f[e]) ++e;
        if (e >= f.size()) { err = "EXR: truncated header"; return false; }
        if (e == pos) { ++pos; break; }                                   // empty name: end of header
        std::string name((const char*)&f[pos], e - pos); pos = e + 1;
        e = pos; while (e < f.size() && f[e]) ++e;
        if (e >= f.size()) { err = "EXR: truncated header"; return false; }
        std::string type((const char*)&f[pos], e - pos); pos = e + 1;
        if (!need(4)) { err = "EXR: truncated header"; return false; }
        const uint32_t sz = rd32(pos); pos += 4;
        if (sz > f.size() || !need(sz)) { err = "EXR: truncated attribute"; return false; }
        if (name == "channels" && type == "chlist") {
            size_t q = pos; const size_t end = pos + sz;
            while (q < end && f[q]) {
                size_t z = q; while (z < end && f[z]) ++z;
                if (z + 17 > end) { err = "EXR: bad channel list"; return false; }
                Chan c; c.name.assign((const char*)&f[q], z - q); c.type = (int)rd32(z + 1); c.xs = (int)rd32(z + 9); c.ys = (int)rd32(z + 13);
                chans.push_back(c); q = z + 17;
            }
        } else if (name == "compression" && sz >= 1) compression = f[pos];
        else if (name == "dataWindow" && sz >= 16) { for (int k = 0; k < 4; ++k) dw[k] = (int)rd32(pos + 4 * k); haveDW = true; }
        else if (name == "lineOrder" && sz >= 1) lineOrder = f[pos];
        pos += sz;
    }
    (void)lineOrder;                                                      // chunks carry their y coordinate: any order decodes
    if (chans.empty() || !haveDW || compression < 0) { err = "EXR: header lacks channels / dataWindow / compression"; return false; }
    const long long w = (long long)dw[2] - dw[0] + 1, h = (long long)dw[3] - dw[1] + 1;
    if (w <= 0 || h <= 0 || w > MF_MAX_IMAGE_SIDE || h > MF_MAX_IMAGE_SIDE) { err = "EXR: empty data window or image side above 16384"; return false; }
    if (compression > 3) {
        const char* nm[] = {"NONE", "RLE", "ZIPS", "ZIP", "PIZ", "PXR24", "B44", "B44A", "DWAA", "DWAB"};
        err = std::string("EXR: compression ") + (compression < 10 ? nm[compression] : "?") + " is not supported (NONE, RLE, ZIPS, ZIP are)"; return false;
    }
    // which channel is the depth: "B" of an R,G,B file (OpenCV returns BGR; the reference reads element 0), else "Y", else the only channel
    int pick = -1; bool hasR = false, hasG = false, hasB = false;
    for (size_t i = 0; i < chans.size(); ++i) { hasR |= chans[i].name == "R"; hasG |= chans[i].name == "G"; hasB |= chans[i].name == "B"; }
    for (size_t i = 0; i < chans.size(); ++i) {
        if (hasR && hasG && hasB) { if (chans[i].name == "B") pick = (int)i; }
        else if (chans[i].name == "Y") pick = (int)i;
    }
    if (pick < 0 && chans.size() == 1) pick = 0;
    if (pick < 0) { err = "EXR: no R,G,B / Y / single channel to take the depth from"; return false; }
    size_t lineBytes = 0, pickOff = 0;
    for (size_t i = 0; i < chans.size(); ++i) {
        if (chans[i].xs != 1 || chans[i].ys != 1) { err = "EXR: sub-sampled channels are not supported"; return false; }
        if (chans[i].type < 0 || chans[i].type > 2) { err = "EXR: bad pixel type"; return false; }
        if ((int)i == pick) pickOff = lineBytes;
        lineBytes += (size_t)w * (chans[i].type == 1 ? 2 : 4);
    }
    if (chans[pick].type == 0) { err = "Unsupported depth-files: 32SC1"; return false; }      // UINT channel: the reference rejects the type (:269-271)
    const int linesPerBlock = compression == 3 ? 16 : 1;
    const size_t nChunks = ((size_t)h + linesPerBlock - 1) / linesPerBlock;
    if (!need(nChunks * 8)) { err = "EXR: truncated offset table"; return false; }
    W = (int)w; H = (int)h;
    depth.assign((size_t)W * H, 0.f);
    std::vector<uint8_t> raw, tmp;
    for (size_t c = 0; c < nChunks; ++c) {
        uint64_t off; memcpy(&off, &f[pos + c * 8], 8);
        if (off > f.size() || off + 8 > f.size()) { err = "EXR: chunk offset beyond the file"; return false; }
        const int y = (int)rd32((size_t)off); const uint32_t csz = rd32((size_t)off + 4);
        const size_t data = (size_t)off + 8;
        if (csz > f.size() || data + csz > f.size()) { err = "EXR: truncated chunk"; return false; }
        const long long y0 = (long long)y - dw[1];
        if (y0 < 0 || y0 >= h) { err = "EXR: chunk outside the data window"; return false; }
        const int nl = (int)std::min<long long>(linesPerBlock, h - y0);
        const size_t rawLen = lineBytes * (size_t)nl;
        raw.resize(rawLen);
        if (compression == 0 || csz == rawLen) {                           // stored uncompressed (also the escape of the compressors)
            if (csz != rawLen) { err = "EXR: chunk size does not match the scan-line size"; return false; }
            memcpy(raw.data(), &f[data], rawLen);
        } else {
            tmp.resize(rawLen);
            if (compression == 1) {                                        // RLE (ImfRle.cpp): n < 0: -n literal bytes; n >= 0: next byte n + 1 times
                size_t ip = data, op = 0; const size_t iend = data + csz;
                while (ip < iend) {
                    const int n = (int8_t)f[ip++];
                    if (n < 0) { const size_t cnt = (size_t)(-n); if (ip + cnt > iend || op + cnt > rawLen) { err = "EXR: bad RLE stream"; return false; } memcpy(&tmp[op], &f[ip], cnt); ip += cnt; op += cnt; }
                    else { const size_t cnt = (size_t)n + 1; if (ip >= iend || op + cnt > rawLen) { err = "EXR: bad RLE stream"; return false; } memset(&tmp[op], f[ip++], cnt); op += cnt; }
                }
                if (op != rawLen) { err = "EXR: RLE stream does not decode to the scan-line size"; return false; }
            } else {
                unsigned long outLen = (unsigned long)rawLen;
                if (uncompress(tmp.data(), &outLen, &f[data], csz) != Z_OK || outLen != rawLen) { err = "EXR: zlib stream does not decode to the scan-line size"; return false; }
            }
            // undo the byte predictor, then the even/odd byte split (ImfZip.cpp / ImfRleCompressor.cpp)
            for (size_t i = 1; i < rawLen; ++i) tmp[i] = (uint8_t)(tmp[i - 1] + tmp[i] - 128);
            const size_t half = (rawLen + 1) / 2;
            for (size_t i = 0; i < rawLen; ++i) raw[i] = (i & 1) ? tmp[half + i / 2] : tmp[i / 2];
        }
        for (int l = 0; l < nl; ++l) {
            const uint8_t* src = raw.data() + (size_t)l * lineBytes + pickOff;
            float* dst = &depth[(size_t)(y0 + l) * W];
            if (chans[pick].type == 2) memcpy(dst, src, (size_t)W * 4);
            else for (int x = 0; x < W; ++x) { uint16_t hv; memcpy(&hv, src + 2 * x, 2); dst[x] = halfToFloat(hv); }
        }
    }
    return true;
}

bool loadImage(const std::string& path, const std::string& ext, Image& im, std::string& err)
{
    std::vector<uint8_t> f;
    if (!readFile(path, f)) { err = "cannot read " + path; return false; }
    if (ext == ".png") return decodePNG(f, im, err);
    if (ext == ".ppm" || ext == ".pgm") return decodePNM(f, im, err);
    if (ext == ".jpg") {
        std::vector<uint8_t> rgb;
        if (!mfb::decodeJPEG(f.data(), f.size(), im.w, im.h, rgb, err)) return false;
        im.channels = 3; im.bits = 8; im.data.swap(rgb);
        return true;
    }
    err = "no decoder for " + ext + " files (supported: .png, .jpg, .ppm, .pgm; .exr depth through decodeEXRDepth)";
    return false;
}

bool exists(const std::string& p) { struct stat st; return stat(p.c_str(), &st) == 0 && S_ISREG(st.st_mode); }

std::string withSlash(const char* d) { std::string s = d ? d : ""; if (!s.empty() && s.back() != '/') s += '/'; return s; }

std::string indexString(unsigned width, size_t index)
{
    char buf[64];
    snprintf(buf, sizeof buf, "%0*zu", (int)width, index);
    return buf;
}

}  // namespace

struct mf_dir {
    std::string colorDir, depthDir, maskDir, colorPre, depthPre, maskPre, colorExt, depthExt, maskExt;
    unsigned indexW = 4, startIndex = 0;
    int numFrames = 0, currentFrame = -1, W = 0, H = 0;
    bool hasMasks = false; size_t maxMasks = 0;
    float rateHz = 24;                                   // ImageLogReader.h:92
};

// countFilesInDir of the reference constructor (:86-114): files whose stem starts with `prefix` and whose (lower-cased) extension is in
// the list; all of them must share one extension.  Returns -1 on a mixed set.
static int countFiles(const std::string& dir, const std::string& prefix, const std::vector<std::string>& exts, std::string& outExt, std::string& err)
{
    outExt.clear();
    DIR* d = opendir(dir.c_str());
    if (!d) { err = "cannot open directory " + dir; return -1; }
    int n = 0;
    while (struct dirent* e = readdir(d)) {
        std::string name = e->d_name;
        if (!exists(dir + name)) continue;
        size_t dot = name.find_last_of('.');
        if (dot == std::string::npos || dot == 0) continue;
        std::string stem = name.substr(0, dot), ext = name.substr(dot);
        std::transform(ext.begin(), ext.end(), ext.begin(), [](unsigned char c) { return (char)tolower(c); });
        if (stem.compare(0, prefix.size(), prefix) != 0) continue;
        if (std::find(exts.begin(), exts.end(), ext) == exts.end()) continue;
        if (outExt.empty()) outExt = ext;
        else if (outExt != ext) { closedir(d); err = "Error: Files in the dataset ( " + dir + ", " + prefix + ") are required to have the same extension."; return -1; }
        ++n;
    }
    closedir(d);
    return n;
}

extern "C" mf_dir* mf_dir_open(const char* color_dir, const char* depth_dir, const char* mask_dir, int index_width, const char* color_prefix,
                               const char* depth_prefix, const char* mask_prefix)
{
    MF_TRY
    if (!color_dir) { mf_set_error("mf_dir_open: null colour directory"); return nullptr; }
    std::unique_ptr<mf_dir> r(new mf_dir);
    r->colorDir = withSlash(color_dir); r->depthDir = withSlash(depth_dir && *depth_dir ? depth_dir : color_dir);
    r->maskDir = withSlash(mask_dir && *mask_dir ? mask_dir : "");
    r->colorPre = color_prefix ? color_prefix : ""; r->depthPre = depth_prefix ? depth_prefix : ""; r->maskPre = mask_prefix ? mask_prefix : "";
    r->indexW = index_width > 0 ? (unsigned)index_width : 4;
    const bool noMaskDir = r->maskDir.empty();
    // overlapping directories but no distinct prefixes: default prefixes (:79-84)
    if (((r->depthDir == r->colorDir) || (r->maskDir == r->colorDir) || (r->maskDir == r->depthDir)) &&
        (r->depthPre == r->colorPre && r->maskPre == r->colorPre)) { r->colorPre = "Color"; r->depthPre = "Depth"; r->maskPre = "Mask"; }
    std::string err;
    int nc = countFiles(r->colorDir, r->colorPre, {".jpg", ".png", ".ppm"}, r->colorExt, err);
    int nd = nc < 0 ? -1 : countFiles(r->depthDir, r->depthPre, {".exr", ".png"}, r->depthExt, err);
    int nm = (nd < 0 || noMaskDir) ? 0 : countFiles(r->maskDir, r->maskPre, {".png", ".pgm"}, r->maskExt, err);
    if (nc < 0 || nd < 0 || nm < 0) { mf_set_error(err); return nullptr; }
    if (nm > 0) { r->hasMasks = true; r->maxMasks = (size_t)nm; }
    if (nc != nd) { mf_set_error("Error: Number of RGB-frames != Depth-frames!"); return nullptr; }
    if (r->hasMasks && nc != nm) { mf_set_error("Error: Number of RGB-frames != Mask-frames!"); return nullptr; }
    r->numFrames = nc;
    int index = 0;
    for (; index < 2; ++index)
        if (exists(r->colorDir + r->colorPre + indexString(r->indexW, (size_t)index) + r->colorExt)) { r->startIndex = (unsigned)index; break; }
    if (index == 2) { mf_set_error("Error: Could not find start index."); return nullptr; }
    // image size from the first colour frame (the reference takes it from Resolution::getInstance())
    Image im;
    if (!loadImage(r->colorDir + r->colorPre + indexString(r->indexW, r->startIndex) + r->colorExt, r->colorExt, im, err)) { mf_set_error(err); return nullptr; }
    r->W = im.w; r->H = im.h;
    return r.release();
    MF_CATCH(nullptr)
}
extern "C" void mf_dir_close(mf_dir* r) { delete r; }
extern "C" int mf_dir_num_frames(mf_dir* r) { return r ? r->numFrames : -1; }
extern "C" int mf_dir_has_more(mf_dir* r) { return r ? (r->currentFrame + 1 < r->numFrames) : 0; }      // :326
extern "C" int mf_dir_has_masks(mf_dir* r) { return r && r->hasMasks ? 1 : 0; }
extern "C" int mf_dir_set_max_masks(mf_dir* r, int n) { if (!r) return -1; r->maxMasks = n < 0 ? 0 : (size_t)n; return 0; }   // "-nm", MainController.cpp:168-173
extern "C" int mf_dir_size(mf_dir* r, int* w, int* h) { if (!r) return -1; if (w) *w = r->W; if (h) *h = r->H; return 0; }

// test hook behind the C ABI: an OpenEXR byte stream -> the float depth image the reader delivers (out == NULL: only the size)
extern "C" int mf_decode_exr_depth(const uint8_t* data, int size, float* out, int capacity, int* width, int* height)
{
    MF_TRY
    if (!data || size <= 0) { mf_set_error("decode_exr_depth: empty input"); return -1; }
    std::vector<uint8_t> f(data, data + size); std::vector<float> d; int W = 0, H = 0; std::string err;
    if (!decodeEXRDepth(f, W, H, d, err)) { mf_set_error(err); return -2; }
    if (width) *width = W;
    if (height) *height = H;
    if (out) {
        if ((size_t)capacity < d.size()) { mf_set_error("decode_exr_depth: output buffer too small"); return -3; }
        memcpy(out, d.data(), d.size() * sizeof(float));
    }
    return 0;
    MF_CATCH(-4)
}

// ImageLogReader::getNext + loadFrameFromDrive (:222-288).  mask / class_ids / boxes may be NULL.  *n_class_ids: in = capacity of
// class_ids (and of boxes / 4), out = number of ids read (0 when the frame has no description file).  Returns 1 when a mask was
// delivered, 0 when not, < 0 on error.
extern "C" int mf_dir_get_next(mf_dir* r, uint8_t* rgb, float* depth, uint8_t* mask, int32_t* class_ids, int32_t* boxes, int* n_class_ids,
                               int64_t* timestamp)
{
    MF_TRY
    if (!r) { mf_set_error("null reader"); return -1; }
    if (!rgb || !depth) { mf_set_error("mf_dir_get_next: null output buffer"); return -1; }
    if (r->currentFrame + 1 >= r->numFrames) { mf_set_error("no more frames"); return -2; }
    const size_t index = (size_t)(r->currentFrame + 1);
    const std::string idx = indexString(r->indexW, index + r->startIndex);
    const std::string depthPath = r->depthDir + r->depthPre + idx + r->depthExt, rgbPath = r->colorDir + r->colorPre + idx + r->colorExt;
    if (!exists(depthPath)) { mf_set_error("Could not find depth-image file: " + depthPath); return -3; }
    if (!exists(rgbPath)) { mf_set_error("Could not find rgb-image file: " + rgbPath); return -3; }
    const std::string maskBase = r->maskDir + r->maskPre + idx, maskPath = maskBase + r->maskExt, descr = maskBase + ".txt";
    const int cap = n_class_ids ? *n_class_ids : 0;
    if (n_class_ids) *n_class_ids = 0;
    if (r->hasMasks) {
        if (!exists(maskPath)) { mf_set_error("Could not find mask-image file: " + maskPath); return -3; }
        if (exists(descr) && class_ids) {              // loadMaskIDs (:302-322)
            FILE* fp = fopen(descr.c_str(), "r");
            std::string first; int ch;
            while (fp && (ch = fgetc(fp)) != EOF && ch != '\n') first += (char)ch;
            std::vector<int> ids{0};                   // mask 0 is always background
            size_t p = 0;
            while (p < first.size()) {
                while (p < first.size() && first[p] == ' ') ++p;
                size_t q = p; while (q < first.size() && first[q] != ' ') ++q;
                if (q > p) ids.push_back(atoi(first.substr(p, q - p).c_str()));
                p = q;
            }
            std::vector<int> bx; int a, b, c, d;
            while (fp && fscanf(fp, "%d %d %d %d", &a, &b, &c, &d) == 4) { bx.push_back(b); bx.push_back(a); bx.push_back(d - b); bx.push_back(c - a); }   // cv::Rect(b, a, d-b, c-a)
            if (fp) fclose(fp);
            if (!bx.empty() && bx.size() / 4 != ids.size() - 1) { mf_set_error("Bounding-boxes provided, but number does not match class ids."); return -4; }
            if ((int)ids.size() > cap) { mf_set_error("class id buffer too small"); return -5; }
            for (size_t i = 0; i < ids.size(); ++i) class_ids[i] = ids[i];
            if (boxes) for (size_t i = 0; i < bx.size(); ++i) boxes[i] = bx[i];
            *n_class_ids = (int)ids.size();
        }
    }
    std::string err; Image im;
    // colour: cv::imread(path) == 8-bit, 3 channels; gray is replicated, alpha dropped, 16-bit scaled by >> 8
    if (!loadImage(rgbPath, r->colorExt, im, err)) { mf_set_error("Could not read rgb-image file. (" + err + ")"); return -6; }
    if (im.w != r->W || im.h != r->H) { mf_set_error("rgb-image size differs from the first frame"); return -6; }
    const size_t P = (size_t)r->W * r->H;
    for (size_t i = 0; i < P; ++i)
        for (int c = 0; c < 3; ++c) {
            const int sc = im.channels >= 3 ? c : 0;
            const size_t e = i * im.channels + sc;
            uint8_t v;
            if (im.bits == 16) { uint16_t t; memcpy(&t, &im.data[e * 2], 2); v = (uint8_t)(t >> 8); } else v = im.data[e];
            rgb[i * 3 + c] = v;
        }
    // depth: cv::imread(path, IMREAD_UNCHANGED); only CV_16UC1 is decodable here (:262-268)
    if (r->depthExt == ".exr") {
        // cv::imread(IMREAD_UNCHANGED) of an EXR file: CV_32FC1, or CV_32FC3 of which the reference keeps element 0 (:253-258)
        std::vector<uint8_t> fb; std::vector<float> dz; int dwid = 0, dhei = 0;
        if (!readFile(depthPath, fb)) { mf_set_error("Could not read depth-image file. (cannot read " + depthPath + ")"); return -7; }
        if (!decodeEXRDepth(fb, dwid, dhei, dz, err)) { mf_set_error("Could not read depth-image file. (" + err + ")"); return -7; }
        if (dwid != r->W || dhei != r->H) { mf_set_error("depth-image size differs from the colour image"); return -7; }
        memcpy(depth, dz.data(), P * sizeof(float));
    } else {
    if (!loadImage(depthPath, r->depthExt, im, err)) { mf_set_error("Could not read depth-image file. (" + err + ")"); return -7; }
    if (im.w != r->W || im.h != r->H) { mf_set_error("depth-image size differs from the colour image"); return -7; }
    if (!(im.bits == 16 && im.channels == 1)) { mf_set_error(std::string("Unsupported depth-files: ") + (im.bits == 16 ? "16U" : "8U") + "C" + std::to_string(im.channels)); return -7; }
    for (size_t i = 0; i < P; ++i) { uint16_t t; memcpy(&t, &im.data[i * 2], 2); depth[i] = 0.001f * (float)t; }
    }
    int gotMask = 0;
    if (r->hasMasks && index < r->maxMasks && mask) {
        if (!loadImage(maskPath, r->maskExt, im, err) || (size_t)im.w * im.h != P) { mf_set_error("Could not read mask-image file."); return -8; }
        if (im.channels != 1 || im.bits != 8) { mf_set_error("Incompatible mask image."); return -8; }
        memcpy(mask, im.data.data(), P);
        gotMask = 1;
    }
    if (timestamp) *timestamp = (int64_t)((float)index * 1000.0f / r->rateHz);        // :283 (float product truncated into the int64 field)
    r->currentFrame++;
    return gotMask;
    MF_CATCH(-9)
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Mask R-CNN post-processing: detections -> id image   <- generate_id_image, Core/Segmentation/MaskRCNN/helpers.py:70-98
// (called by MaskRCNN.py.in:105-111 after model.detect; the id image, class list and boxes are what MaskRCNN.cpp:83-151 reads back).
// masks: H x W x N uint8 (the network's layout, N fastest), scores / class_ids / rois (N x 4, y1 x1 y2 x2) per detection.
// Detections are written in order: a later detection overwrites an earlier one where they overlap; ids are 1..n in export order
// unless `special_assignments` maps the class (a list indexed BY CLASS ID, used when the class id occurs IN the list, helpers.py:91-92).
// Returns the number of exported detections, < 0 on error.  Pinned against the reference's own Python function (tests/test_cpu_loader.py).
// PreSegmentation::performSegmentation (Core/Segmentation/PreSegmentation.cpp:28-90): the "-segMethod precomputed" performer -- host code in the
// reference as well.  The input mask's values are mapped to model ids through a table that persists over the frames (`mapping`, the function's
// static vector in the reference): a value seen before keeps its model; the FIRST unseen value met in raster order takes `next_model_id` when
// new models are allowed (and every later pixel of that value follows it); other unseen values stay background for this frame.  Per model (in
// list order, the new one last): superPixelCount = pixels / 256 (integer; the new model: at least 1), then the mean depth and the mean absolute
// deviation of the depth over the pixels assigned to it, accumulated in float in raster order exactly as the reference does (these feed
// Model::setMaxDepth, MaskFusion.cpp:291,337-341).  Returns the number of model entries written (n_models, + 1 with a new label), < 0 on error.
extern "C" int mf_pre_segmentation(const uint8_t* mask, const float* depth, int W, int H, const uint8_t* model_ids, int n_models, int next_model_id,
                                   int allow_new, uint8_t* mapping, uint8_t* full_segmentation, int* has_new_label, uint32_t* super_pixel_count,
                                   float* depth_mean, float* depth_std)
{
    MF_TRY
    if (!mask || !depth || !model_ids || !mapping || !full_segmentation || !super_pixel_count || !depth_mean || !depth_std || W <= 0 || H <= 0 ||
        n_models < 1 || n_models > 255 || next_model_id < 0 || next_model_id > 255) { mf_set_error("mf_pre_segmentation: bad arguments"); return -1; }
    const size_t P = (size_t)W * H;
    unsigned char modelIdToIndex[256];
    memset(modelIdToIndex, 0, sizeof modelIdToIndex);                 // (uninitialised in the reference; ids outside the list never occur in its output)
    for (int i = 0; i < n_models; ++i) modelIdToIndex[model_ids[i]] = (unsigned char)i;
    modelIdToIndex[next_model_id] = (unsigned char)n_models;
    std::vector<unsigned> outIds(256, 0);
    bool hasNew = false;
    for (size_t i = 0; i < P; ++i) {
        const unsigned char vIn = mask[i];
        unsigned char vOut = 0;
        if (vIn) {
            if (mapping[vIn] != 0) { vOut = mapping[vIn]; outIds[vOut]++; }
            else if (allow_new && !hasNew) { vOut = (unsigned char)next_model_id; mapping[vIn] = vOut; hasNew = true; outIds[vOut]++; }
        } else outIds[0]++;
        full_segmentation[i] = vOut;
    }
    const int n = n_models + (hasNew ? 1 : 0);
    for (int i = 0; i < n_models; ++i) super_pixel_count[i] = outIds[model_ids[i]] / (16 * 16);
    if (hasNew) { const float c = (float)(outIds[next_model_id] / (16 * 16)); super_pixel_count[n_models] = (unsigned)(c > 1.0f ? c : 1.0f); }
    std::vector<unsigned> cnts(n, 0);
    for (int i = 0; i < n; ++i) { depth_mean[i] = 0.f; depth_std[i] = 0.f; }
    for (size_t i = 0; i < P; ++i) { const size_t k = modelIdToIndex[full_segmentation[i]]; if ((int)k < n) { depth_mean[k] += depth[i]; cnts[k]++; } }
    for (int i = 0; i < n; ++i) depth_mean[i] /= cnts[i] ? cnts[i] : 1;
    for (size_t i = 0; i < P; ++i) { const size_t k = modelIdToIndex[full_segmentation[i]]; if ((int)k < n) depth_std[k] += std::abs(depth_mean[k] - depth[i]); }
    for (int i = 0; i < n; ++i) depth_std[i] /= cnts[i] ? cnts[i] : 1;
    if (has_new_label) *has_new_label = hasNew ? 1 : 0;
    return n;
    MF_CATCH(-2)
}

extern "C" int mf_generate_id_image(const uint8_t* masks, int H, int W, int N, const float* scores, const int32_t* class_ids, const int32_t* rois,
                                    double min_score, const int32_t* class_filter, int n_filter, const int32_t* special_assignments, int n_special,
                                    uint8_t* id_image, int32_t* exported_class_ids, int32_t* exported_rois)
{
    MF_TRY
    if (N > 256) { mf_set_error("Too many masks in image."); return -1; }                 // helpers.py:78-79
    if (!id_image || (N > 0 && (!masks || !scores || !class_ids || !rois))) { mf_set_error("generate_id_image: null argument"); return -2; }
    const size_t P = (size_t)H * W;
    memset(id_image, 0, P);
    int n = 0;
    for (int m = 0; m < N; ++m) {
        const int cid = class_ids[m];
        uint8_t v = 0;
        const int e = mfb::id_export(cid, scores[m], min_score, class_filter, n_filter, special_assignments, n_special, n, &v);
        if (e < 0) { mf_set_error("generate_id_image: special_assignments[class_id] out of range"); return -3; }   // Python: IndexError
        if (e == 0) continue;
        for (size_t p = 0; p < P; ++p) if (masks[p * N + m] == 1) id_image[p] = v;
        if (exported_class_ids) exported_class_ids[n] = cid;
        if (exported_rois) for (int k = 0; k < 4; ++k) exported_rois[n * 4 + k] = rois[m * 4 + k];
        ++n;
    }
    return n;
    MF_CATCH(-1)
}

// ---------------------------------------------------------------------------------------------------------------------------------
// PLY export of one model   <- the lambda in MaskFusion::savePly, Core/MaskFusion.cpp:733-848
// surfels: n x 12 floats in the reference's layout (Model.h:190-192: position|conf, colour|-|initTime|lastTime, normal|radius), as
// mf_download_surfels returns them.  Vertices with conf > threshold are written as x y z (float) r g b (uchar, from the packed colour)
// nx ny nz (float, NEGATED as the reference does) radius (float), binary little endian.  Returns the number of vertices written.
extern "C" int mf_write_ply(const char* path, const float* surfels, int n, float conf_threshold)
{
    MF_TRY
    if (!path || (n > 0 && !surfels) || n < 0) { mf_set_error("write_ply: bad arguments"); return -1; }
    int valid = 0;
    for (int i = 0; i < n; ++i) if (surfels[(size_t)i * 12 + 3] > conf_threshold) ++valid;      // SurfelMap::countValid
    FILE* fp = fopen(path, "wb");
    if (!fp) { mf_set_error(std::string("cannot write ") + path); return -2; }
    fprintf(fp, "ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z"
                "\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nproperty float nx\nproperty float ny\nproperty float nz"
                "\nproperty float radius\nend_header\n", valid);
    for (int i = 0; i < n; ++i) {
        const float* s = surfels + (size_t)i * 12;
        if (!(s[3] > conf_threshold)) continue;
        fwrite(s, sizeof(float), 3, fp);
        const int c = (int)s[4];
        const unsigned char rgb[3] = {(unsigned char)(c >> 16 & 0xFF), (unsigned char)(c >> 8 & 0xFF), (unsigned char)(c & 0xFF)};
        fwrite(rgb, 1, 3, fp);
        const float nr[4] = {s[8] * -1, s[9] * -1, s[10] * -1, s[11]};
        fwrite(nr, sizeof(float), 4, fp);
    }
    fclose(fp);
    return valid;
    MF_CATCH(-1)
}
