// Native multi-threaded PNG decoder for the decoded-image cache (SURVEY N9: the reference decodes
// every image with PIL in the training process, every epoch, single-threaded).  Handles what an
// ImageFolder of 8-bit PNGs contains: colour types 0/2/3/4/6, bit depth 8, non-interlaced; anything
// else makes decode_pngs() report failure for that file and the Python side falls back to PIL.
// zlib does the inflate; filtering (None/Sub/Up/Average/Paeth) and RGB conversion are done here.
#include <zlib.h>

#include <atomic>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

namespace b200 {

struct PngImage {
  int w = 0, h = 0;
  std::vector<uint8_t> rgb;   // h * w * 3
  bool ok = false;
};

static uint32_t be32(const uint8_t* p) { return (uint32_t(p[0]) << 24) | (uint32_t(p[1]) << 16) | (uint32_t(p[2]) << 8) | p[3]; }

static inline uint8_t paeth(int a, int b, int c) {
  const int p = a + b - c;
  const int pa = p > a ? p - a : a - p, pb = p > b ? p - b : b - p, pc = p > c ? p - c : c - p;
  return static_cast<uint8_t>((pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c));
}

static bool decode_one(const std::string& path, PngImage& out) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  fseek(f, 0, SEEK_END);
  const long size = ftell(f);
  fseek(f, 0, SEEK_SET);
  std::vector<uint8_t> buf(size > 0 ? size : 0);
  const bool read_ok = size > 0 && fread(buf.data(), 1, size, f) == static_cast<size_t>(size);
  fclose(f);
  static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
  if (!read_ok || size < 33 || memcmp(buf.data(), sig, 8) != 0) return false;
  size_t pos = 8;
  int w = 0, h = 0, depth = 0, ctype = 0, interlace = 0;
  std::vector<uint8_t> idat, plte;
  while (pos + 12 <= buf.size()) {
    const uint32_t len = be32(&buf[pos]);
    const uint8_t* type = &buf[pos + 4];
    const uint8_t* data = &buf[pos + 8];
    if (pos + 12 + len > buf.size()) return false;
    if (!memcmp(type, "IHDR", 4)) {
      if (len < 13) return false;
      w = be32(data); h = be32(data + 4); depth = data[8]; ctype = data[9]; interlace = data[12];
    } else if (!memcmp(type, "PLTE", 4)) {
      plte.assign(data, data + len);
    } else if (!memcmp(type, "IDAT", 4)) {
      idat.insert(idat.end(), data, data + len);
    } else if (!memcmp(type, "IEND", 4)) {
      break;
    }
    pos += 12 + len;
  }
  if (w <= 0 || h <= 0 || w > 16384 || h > 16384 || depth != 8 || interlace != 0) return false;
  int ch;
  switch (ctype) {
    case 0: ch = 1; break;
    case 2: ch = 3; break;
    case 3: ch = 1; if (plte.size() < 3) return false; break;
    case 4: ch = 2; break;
    case 6: ch = 4; break;
    default: return false;
  }
  const size_t stride = static_cast<size_t>(w) * ch;
  std::vector<uint8_t> raw((stride + 1) * h);
  uLongf dlen = raw.size();
  if (uncompress(raw.data(), &dlen, idat.data(), idat.size()) != Z_OK || dlen != raw.size()) return false;
  std::vector<uint8_t> img(stride * h);
  for (int y = 0; y < h; ++y) {
    const uint8_t ft = raw[y * (stride + 1)];
    const uint8_t* src = &raw[y * (stride + 1) + 1];
    uint8_t* cur = &img[y * stride];
    const uint8_t* up = y ? &img[(y - 1) * stride] : nullptr;
    for (size_t x = 0; x < stride; ++x) {
      const int a = x >= static_cast<size_t>(ch) ? cur[x - ch] : 0;
      const int b = up ? up[x] : 0;
      const int c = (up && x >= static_cast<size_t>(ch)) ? up[x - ch] : 0;
      uint8_t v = src[x];
      switch (ft) {
        case 0: break;
        case 1: v = static_cast<uint8_t>(v + a); break;
        case 2: v = static_cast<uint8_t>(v + b); break;
        case 3: v = static_cast<uint8_t>(v + ((a + b) >> 1)); break;
        case 4: v = static_cast<uint8_t>(v + paeth(a, b, c)); break;
        default: return false;
      }
      cur[x] = v;
    }
  }
  out.w = w; out.h = h;
  out.rgb.resize(static_cast<size_t>(w) * h * 3);
  for (size_t i = 0; i < static_cast<size_t>(w) * h; ++i) {
    uint8_t r, g, b;
    const uint8_t* p = &img[i * ch];
    switch (ctype) {
      case 0: case 4: r = g = b = p[0]; break;
      case 3: {
        const size_t k = static_cast<size_t>(p[0]) * 3;
        if (k + 2 >= plte.size()) return false;
        r = plte[k]; g = plte[k + 1]; b = plte[k + 2];
        break;
      }
      default: r = p[0]; g = p[1]; b = p[2]; break;      // 2, 6 (alpha dropped, as PIL's convert("RGB"))
    }
    out.rgb[i * 3] = r; out.rgb[i * 3 + 1] = g; out.rgb[i * 3 + 2] = b;
  }
  out.ok = true;
  return true;
}

bool decode_png_file(const std::string& path, PngImage& out) {
  try {
    return decode_one(path, out);
  } catch (...) {            // e.g. bad_alloc on a corrupt header
    return false;
  }
}

// Decode all files with `threads` workers.  Returns false for files this decoder does not handle.
void decode_png_files(const std::vector<std::string>& paths, int threads, std::vector<PngImage>& out) {
  out.assign(paths.size(), PngImage());
  std::atomic<size_t> next{0};
  auto work = [&]() {
    for (;;) {
      const size_t i = next.fetch_add(1);
      if (i >= paths.size()) return;
      try {
        decode_one(paths[i], out[i]);
      } catch (...) {            // e.g. bad_alloc on a corrupt header: report "not handled", PIL decides
        out[i] = PngImage();
      }
    }
  };
  if (threads < 1) threads = 1;
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t) pool.emplace_back(work);
  for (auto& t : pool) t.join();
}

// Decode file i straight into dst + offsets[i] when it is a PNG this decoder handles and its size is
// hw[i] = (H, W); ok[i] says which files were written.  Only one decoded image per thread is alive.
void decode_png_files_into(const std::vector<std::string>& paths, int threads, uint8_t* dst, const int64_t* offsets,
                           const int64_t* hw, uint8_t* ok) {
  std::atomic<size_t> next{0};
  auto work = [&]() {
    for (;;) {
      const size_t i = next.fetch_add(1);
      if (i >= paths.size()) return;
      ok[i] = 0;
      try {
        PngImage img;
        if (decode_one(paths[i], img) && img.h == hw[i * 2] && img.w == hw[i * 2 + 1]) {
          memcpy(dst + offsets[i], img.rgb.data(), img.rgb.size());
          ok[i] = 1;
        }
      } catch (...) {            // not handled here: PIL decodes this file
      }
    }
  };
  if (threads < 1) threads = 1;
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t) pool.emplace_back(work);
  for (auto& t : pool) t.join();
}

// ok[i]: file i is a PNG this decoder takes, of size hw[i] = (H, W).  Each file is decoded and dropped.
void check_png_files(const std::vector<std::string>& paths, int threads, const int64_t* hw, uint8_t* ok) {
  std::atomic<size_t> next{0};
  auto work = [&]() {
    for (;;) {
      const size_t i = next.fetch_add(1);
      if (i >= paths.size()) return;
      PngImage img;
      ok[i] = decode_png_file(paths[i], img) && img.h == hw[i * 2] && img.w == hw[i * 2 + 1];
    }
  };
  if (threads < 1) threads = 1;
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t) pool.emplace_back(work);
  for (auto& t : pool) t.join();
}

}  // namespace b200
