// Host half of the streaming JPEG pipeline: a header scan that classifies every file of a split, and a
// baseline / extended Huffman entropy decoder for the files the GPU decode kernels (csrc/jpeg.cu) take.
// The decoder stops at the quantised coefficients; dequantisation, IDCT, upsampling and colour conversion
// run on the device.  It handles one interleaved scan holding every component (what JPEG encoders write for
// sequential files), with or without restart intervals, with standard or optimised tables.  Anything it
// cannot decode exactly -- or any data it would have to guess at -- raises an error naming the file.
#include "jpeg.h"

#include <atomic>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <thread>

namespace b200 {

namespace {

// zig-zag index -> natural (row-major) index
const int kNatural[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

uint32_t be16(const uint8_t* p) { return (uint32_t(p[0]) << 8) | p[1]; }
uint32_t be32(const uint8_t* p) { return (be16(p) << 16) | be16(p + 2); }

bool read_file(const std::string& path, std::vector<uint8_t>& buf) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  fseek(f, 0, SEEK_END);
  const long size = ftell(f);
  fseek(f, 0, SEEK_SET);
  buf.resize(size > 0 ? size : 0);
  const bool ok = size > 0 && fread(buf.data(), 1, size, f) == static_cast<size_t>(size);
  fclose(f);
  return ok;
}

bool is_sof(int m) { return m >= 0xC0 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC; }

// Frame / colour checks shared by the scan and the decoder: is this a file the stream decoder reproduces?
bool stream_decodable(const ImageHeader& h, bool adobe_rgb, const int* ids, int ns) {
  if (h.sof != 0 && h.sof != 1) return false;          // progressive, lossless, arithmetic: PIL
  if (h.H < 1 || h.W < 1 || ns != h.ncomp) return false;
  if (h.ncomp == 1) return h.h[0] >= 1 && h.h[0] <= 4 && h.v[0] >= 1 && h.v[0] <= 4;
  if (h.ncomp != 3) return false;                      // CMYK / YCCK / anything else
  if (adobe_rgb || (ids[0] == 'R' && ids[1] == 'G' && ids[2] == 'B')) return false;   // RGB-coded
  const bool luma = (h.h[0] == 1 && h.v[0] == 1) || (h.h[0] == 2 && h.v[0] == 1) || (h.h[0] == 2 && h.v[0] == 2);
  return luma && h.h[1] == 1 && h.v[1] == 1 && h.h[2] == 1 && h.v[2] == 1;
}

int64_t count_blocks(const ImageHeader& h) {
  int64_t n = 0;
  for (int c = 0; c < h.ncomp; ++c) {
    int bw, bh;
    jpeg_block_grid(h, c, bw, bh);
    n += (int64_t)bw * bh;
  }
  return n;
}

// JPEG marker walk up to the first SOS over a file read in pieces: only the headers are read.
ImageHeader scan_jpeg(FILE* f) {
  ImageHeader h;
  bool adobe_rgb = false;
  int ids[4] = {0, 0, 0, 0};
  std::vector<uint8_t> seg;
  for (;;) {
    int c = fgetc(f);
    if (c != 0xFF) return h;
    do c = fgetc(f); while (c == 0xFF);
    if (c == EOF || c == 0xD9) return h;
    if (c == 0x01 || (c >= 0xD0 && c <= 0xD7)) continue;   // no payload
    uint8_t lb[2];
    if (fread(lb, 1, 2, f) != 2) return h;
    const int len = (int)be16(lb) - 2;
    if (len < 0) return h;
    const bool want = is_sof(c) || c == 0xDA || c == 0xEE;
    if (!want) {
      if (fseek(f, len, SEEK_CUR) != 0) return h;
      continue;
    }
    seg.resize(len);
    if (len && fread(seg.data(), 1, len, f) != (size_t)len) return h;
    if (c == 0xEE) {                 // Adobe APP14: transform 0 means the components are RGB
      if (len >= 12 && !memcmp(seg.data(), "Adobe", 5) && seg[11] == 0) adobe_rgb = true;
    } else if (is_sof(c)) {
      if (len < 6) return h;
      h.sof = c - 0xC0;
      h.H = (int)be16(&seg[1]);
      h.W = (int)be16(&seg[3]);
      h.ncomp = seg[5];
      if (seg[0] != 8 || len < 6 + 3 * h.ncomp || h.ncomp > 4) { h.ncomp = h.ncomp > 4 ? 0 : h.ncomp; return h; }
      for (int i = 0; i < h.ncomp; ++i) {
        ids[i] = seg[6 + 3 * i];
        h.h[i] = seg[7 + 3 * i] >> 4;
        h.v[i] = seg[7 + 3 * i] & 15;
      }
    } else {                         // SOS
      if (h.sof < 0 || len < 1) return h;
      if (stream_decodable(h, adobe_rgb, ids, seg[0])) {
        h.kind = kFileJpeg;
        h.blocks = count_blocks(h);
      }
      return h;
    }
  }
}

// ------------------------------------------------------------------------------------------ entropy decoder
inline int extend(int v, int s) { return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }

struct Huff {
  bool defined = false;
  uint8_t look_len[512];      // 9-bit lookahead: code length (0: longer code)
  uint8_t look_val[512];
  // AC tables: a code and its value bits within the 9-bit lookahead, decoded at once:
  // (value << 16) | (run << 8) | bits consumed; 0 when they do not fit
  int32_t fast_ac[512];
  int32_t maxcode[18];        // largest code of each length, -1 if none
  int32_t valptr[17], mincode[17];
  uint8_t vals[256];
};

void build_huff(Huff& t, const uint8_t* bits, const uint8_t* vals, int nvals, const std::string& path) {
  memset(t.look_len, 0, sizeof(t.look_len));
  memcpy(t.vals, vals, nvals);
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    // the codes of length l must fit in l bits, and none may be all ones (libjpeg's jdhuff.c check): refused
    // before any of them goes into the lookahead tables
    if (code + bits[l - 1] >= (1 << l)) throw std::runtime_error(path + ": bad Huffman table");
    t.valptr[l] = k;
    t.mincode[l] = code;
    for (int i = 0; i < bits[l - 1]; ++i, ++k, ++code) {
      if (l <= 9) {
        const int shift = 9 - l;
        for (int j = 0; j < (1 << shift); ++j) {
          t.look_len[(code << shift) | j] = (uint8_t)l;
          t.look_val[(code << shift) | j] = vals[k];
        }
      }
    }
    t.maxcode[l] = bits[l - 1] ? code - 1 : -1;
    code <<= 1;
  }
  t.maxcode[17] = 0x7fffffff;
  for (int i = 0; i < 512; ++i) {
    t.fast_ac[i] = 0;
    const int len = t.look_len[i], rs = t.look_val[i], r = rs >> 4, sz = rs & 15;
    if (len && sz && len + sz <= 9) {
      const int v = extend((i >> (9 - len - sz)) & ((1 << sz) - 1), sz);
      t.fast_ac[i] = (int32_t)((uint32_t)v << 16) | (r << 8) | (len + sz);
    }
  }
  t.defined = true;
}

class BitReader {
 public:
  BitReader(const uint8_t* p, const uint8_t* end, const std::string& path) : p_(p), end_(end), path_(path) {}

  // Value of the next `n` (<= 16) bits without consuming them.
  uint32_t peek(int n) {
    if (nbits_ < n) fill();
    return (uint32_t)(acc_ >> (nbits_ - n)) & ((1u << n) - 1);
  }
  void skip(int n) {
    nbits_ -= n;
    if (nbits_ < pad_) throw std::runtime_error(path_ + ": truncated JPEG data (the entropy-coded segment ends early)");
  }
  int get(int n) {
    if (n == 0) return 0;
    const uint32_t v = peek(n);
    skip(n);
    return (int)v;
  }
  int decode(const Huff& t) {
    const uint32_t look = peek(9);
    if (t.look_len[look]) {
      const int v = t.look_val[look];
      skip(t.look_len[look]);
      return v;
    }
    const uint32_t code16 = peek(16);
    for (int l = 10; l <= 16; ++l) {
      const int32_t code = (int32_t)(code16 >> (16 - l));
      if (t.maxcode[l] >= 0 && code <= t.maxcode[l]) {
        skip(l);
        return t.vals[t.valptr[l] + code - t.mincode[l]];
      }
    }
    throw std::runtime_error(path_ + ": bad Huffman code in the JPEG data");
  }
  // At a restart boundary: drop the byte's padding bits and read RSTn.
  void restart(int n) {
    // bytes between the interval's last bits and the marker are skipped, as libjpeg does
    while (p_ < end_ && !(p_[0] == 0xFF && p_ + 1 < end_ && p_[1] != 0x00)) p_ += p_[0] == 0xFF && p_ + 1 < end_ ? 2 : 1;
    while (end_ - p_ >= 2 && p_[1] == 0xFF) ++p_;       // fill bytes
    nbits_ = pad_ = 0;
    acc_ = 0;
    if (end_ - p_ < 2 || p_[0] != 0xFF || p_[1] != 0xD0 + n)
      throw std::runtime_error(path_ + ": missing or out-of-order restart marker in the JPEG data");
    p_ += 2;
  }
 private:
  void fill() {
    while (nbits_ <= 56) {
      uint32_t byte = 0;
      if (p_ < end_ && !(p_[0] == 0xFF && (p_ + 1 >= end_ || p_[1] != 0x00))) {
        byte = *p_;
        p_ += byte == 0xFF ? 2 : 1;           // stuffed FF 00
      } else {
        pad_ += 8;                            // marker or end of file: zeros that must not be consumed
      }
      acc_ = (acc_ << 8) | byte;
      nbits_ += 8;
    }
  }
  uint64_t acc_ = 0;
  int nbits_ = 0, pad_ = 0;
  const uint8_t* p_;
  const uint8_t* end_;
  const std::string& path_;
};

}  // namespace

ImageHeader scan_image_header(const std::string& path) {
  ImageHeader h;
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return h;
  uint8_t sig[8];
  const size_t n = fread(sig, 1, 8, f);
  static const uint8_t png[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
  if (n >= 2 && sig[0] == 0xFF && sig[1] == 0xD8) {
    fseek(f, 2, SEEK_SET);
    h = scan_jpeg(f);
  } else if (n == 8 && !memcmp(sig, png, 8)) {
    uint8_t ihdr[25];                        // length, "IHDR", 13 bytes, CRC
    if (fread(ihdr, 1, 25, f) == 25 && !memcmp(ihdr + 4, "IHDR", 4)) {
      h.W = (int)be32(ihdr + 8);
      h.H = (int)be32(ihdr + 12);
      const int depth = ihdr[16], ctype = ihdr[17], interlace = ihdr[20];
      // what csrc/png_decode.cpp decodes
      if (depth == 8 && interlace == 0 && (ctype == 0 || ctype == 2 || ctype == 3 || ctype == 4 || ctype == 6) &&
          h.W >= 1 && h.H >= 1 && h.W <= 16384 && h.H <= 16384)
        h.kind = kFilePng;
    }
  }
  fclose(f);
  return h;
}

void scan_image_headers(const std::vector<std::string>& paths, int threads, std::vector<ImageHeader>& out) {
  out.assign(paths.size(), ImageHeader());
  std::atomic<size_t> next{0};
  auto work = [&]() {
    for (size_t i; (i = next.fetch_add(1)) < paths.size();) out[i] = scan_image_header(paths[i]);
  };
  std::vector<std::thread> pool;
  for (int t = 0; t < std::max(threads, 1); ++t) pool.emplace_back(work);
  for (auto& t : pool) t.join();
}

void jpeg_entropy_decode(const std::string& path, const ImageHeader& want, int16_t* coef, int32_t* quant) {
  std::vector<uint8_t> buf;
  if (!read_file(path, buf)) throw std::runtime_error(path + ": cannot read the file");
  auto bad = [&](const char* what) { return std::runtime_error(path + ": " + what); };
  const uint8_t* p = buf.data();
  const uint8_t* end = p + buf.size();
  if (buf.size() < 4 || p[0] != 0xFF || p[1] != 0xD8) throw bad("not a JPEG file");
  p += 2;
  int32_t qt[4][64];
  bool qdef[4] = {false, false, false, false};
  Huff dc[4], ac[4];
  ImageHeader h;
  int ids[4] = {0, 0, 0, 0}, tq[4] = {0, 0, 0, 0};
  bool adobe_rgb = false;
  int restart = 0;
  for (;;) {
    if (end - p < 2 || p[0] != 0xFF) throw bad("truncated or malformed JPEG header");
    while (p < end && *p == 0xFF) ++p;
    if (p >= end) throw bad("truncated JPEG header");
    const int m = *p++;
    if (m == 0xD9) throw bad("JPEG file ends before its scan");
    if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) continue;
    if (end - p < 2) throw bad("truncated JPEG header");
    const int len = (int)be16(p) - 2;
    if (len < 0 || end - p - 2 < len) throw bad("truncated JPEG header");
    const uint8_t* s = p + 2;
    p = s + len;
    if (m == 0xDB) {                                   // DQT
      for (const uint8_t* q = s; q < s + len;) {
        const int pq = *q >> 4, id = *q & 15;
        ++q;
        if (id > 3 || pq > 1 || s + len - q < 64 * (pq + 1)) throw bad("bad quantisation table");
        for (int k = 0; k < 64; ++k) qt[id][kNatural[k]] = pq ? (int32_t)be16(q + 2 * k) : q[k];
        q += 64 * (pq + 1);
        qdef[id] = true;
      }
    } else if (m == 0xC4) {                            // DHT
      for (const uint8_t* q = s; q < s + len;) {
        if (s + len - q < 17) throw bad("bad Huffman table");
        const int tc = *q >> 4, id = *q & 15;
        int n = 0;
        for (int i = 0; i < 16; ++i) n += q[1 + i];
        if (tc > 1 || id > 3 || n > 256 || s + len - q < 17 + n) throw bad("bad Huffman table");
        build_huff(tc ? ac[id] : dc[id], q + 1, q + 17, n, path);
        q += 17 + n;
      }
    } else if (m == 0xDD) {                            // DRI
      if (len < 2) throw bad("bad restart interval");
      restart = (int)be16(s);
    } else if (m == 0xEE) {
      if (len >= 12 && !memcmp(s, "Adobe", 5) && s[11] == 0) adobe_rgb = true;
    } else if (is_sof(m)) {
      if (len < 6) throw bad("bad frame header");
      h.sof = m - 0xC0;
      h.H = (int)be16(s + 1);
      h.W = (int)be16(s + 3);
      h.ncomp = s[5];
      if (s[0] != 8 || h.ncomp < 1 || h.ncomp > 4 || len < 6 + 3 * h.ncomp) throw bad("unsupported frame header");
      for (int i = 0; i < h.ncomp; ++i) {
        ids[i] = s[6 + 3 * i];
        h.h[i] = s[7 + 3 * i] >> 4;
        h.v[i] = s[7 + 3 * i] & 15;
        tq[i] = s[8 + 3 * i];
      }
    } else if (m == 0xDA) {                            // SOS: the one scan
      if (h.sof < 0 || len < 1) throw bad("scan before the frame header");
      const int ns = s[0];
      if (!stream_decodable(h, adobe_rgb, ids, ns) || len < 4 + 2 * ns)
        throw bad("not a baseline JPEG the stream decoder handles");
      if (h.H != want.H || h.W != want.W || h.ncomp != want.ncomp || count_blocks(h) != want.blocks)
        throw bad("the file changed since its header was scanned");
      for (int c = 0; c < 3; ++c)
        if (c < h.ncomp && (h.h[c] != want.h[c] || h.v[c] != want.v[c]))
          throw bad("the file changed since its header was scanned");
      int td[4], ta[4];
      for (int i = 0; i < ns; ++i) {
        if (s[1 + 2 * i] != ids[i]) throw bad("scan components out of frame order");
        td[i] = s[2 + 2 * i] >> 4;
        ta[i] = s[2 + 2 * i] & 15;
        if (td[i] > 3 || ta[i] > 3 || !dc[td[i]].defined || !ac[ta[i]].defined) throw bad("undefined Huffman table");
        if (tq[i] > 3 || !qdef[tq[i]]) throw bad("undefined quantisation table");
        memcpy(quant + 64 * i, qt[tq[i]], sizeof(qt[0]));
      }
      const uint8_t* ss = s + 1 + 2 * ns;
      if (ss[0] != 0 || ss[1] != 63 || ss[2] != 0) throw bad("not a sequential scan");
      // block grids and where each component's blocks start in `coef`
      int bw[3], bh[3];
      int64_t start[3], at = 0;
      for (int c = 0; c < ns; ++c) {
        jpeg_block_grid(h, c, bw[c], bh[c]);
        start[c] = at;
        at += (int64_t)bw[c] * bh[c];
      }
      memset(coef, 0, sizeof(int16_t) * 64 * at);
      int mcux, mcuy;
      if (ns == 1) { mcux = bw[0]; mcuy = bh[0]; }
      else { mcux = bw[0] / h.h[0]; mcuy = bh[0] / h.v[0]; }
      const int hs[3] = {ns == 1 ? 1 : h.h[0], 1, 1}, vs[3] = {ns == 1 ? 1 : h.v[0], 1, 1};
      const int32_t* q[3] = {quant, quant + 64, quant + 128};
      BitReader br(p, end, path);
      int pred[3] = {0, 0, 0};
      const int64_t total = (int64_t)mcux * mcuy;
      for (int64_t mcu = 0; mcu < total; ++mcu) {
        if (restart && mcu && mcu % restart == 0) {
          br.restart((int)((mcu / restart - 1) & 7));
          pred[0] = pred[1] = pred[2] = 0;
        }
        const int mx = (int)(mcu % mcux), my = (int)(mcu / mcux);
        for (int c = 0; c < ns; ++c) {
          for (int by = 0; by < vs[c]; ++by) {
            for (int bx = 0; bx < hs[c]; ++bx) {
              int16_t* blk = coef + 64 * (start[c] + (int64_t)(my * vs[c] + by) * bw[c] + mx * hs[c] + bx);
              const int t = br.decode(dc[td[c]]);
              if (t > 15) throw bad("bad DC coefficient in the JPEG data");
              if (t) pred[c] += extend(br.get(t), t);
              // dequantised values beyond 16 bits never come from an encoder, and libjpeg-turbo's SIMD IDCT
              // (which Pillow runs) computes them in 16-bit lanes: refuse rather than decode them differently
              if (pred[c] * q[c][0] > 32767 || pred[c] * q[c][0] < -32768) throw bad("coefficient out of range");
              blk[0] = (int16_t)pred[c];
              const Huff& act = ac[ta[c]];
              for (int k = 1; k < 64;) {
                const int32_t fa = act.fast_ac[br.peek(9)];
                if (fa) {
                  br.skip(fa & 255);
                  k += (fa >> 8) & 15;
                  if (k > 63) throw bad("bad AC run length in the JPEG data");
                  const int v = fa >> 16, at = kNatural[k];
                  if (v * q[c][at] > 32767 || v * q[c][at] < -32768) throw bad("coefficient out of range");
                  blk[at] = (int16_t)v;
                  ++k;
                  continue;
                }
                const int rs = br.decode(act);
                const int r = rs >> 4, sz = rs & 15;
                if (sz) {
                  k += r;
                  if (k > 63) throw bad("bad AC run length in the JPEG data");
                  const int v = extend(br.get(sz), sz), at = kNatural[k];
                  if (v * q[c][at] > 32767 || v * q[c][at] < -32768) throw bad("coefficient out of range");
                  blk[at] = (int16_t)v;
                  ++k;
                } else if (r == 15) {
                  k += 16;
                } else {
                  break;
                }
              }
            }
          }
        }
      }
      return;
    }
  }
}

}  // namespace b200
