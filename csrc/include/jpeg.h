// Streaming JPEG input (csrc/jpeg_decode.cpp, csrc/prefetch.cpp, csrc/jpeg.cu): what the header scan reports
// for a file, and the per-image descriptor the decode kernels read.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace b200 {

// What the stream pipeline does with a file: entropy-decode it here (kFileJpeg), decode it with the native PNG
// decoder (kFilePng), or leave it to PIL at start-up (kFileOther).
enum : int { kFileOther = 0, kFileJpeg = 1, kFilePng = 2 };

struct ImageHeader {
  int kind = kFileOther;
  int H = 0, W = 0;          // 0 when the scan could not read them (PIL decides)
  int sof = -1;              // JPEG: the frame marker's low nibble (0 baseline, 1 extended, 2 progressive, ...)
  int ncomp = 0;
  int h[4] = {0, 0, 0, 0}, v[4] = {0, 0, 0, 0};   // JPEG sampling factors per component
  int64_t blocks = 0;        // stream-JPEG: 8x8 coefficient blocks over all components, MCU padding included
};

// Reads a file only up to the frame header / first scan header.  Never throws: unreadable files are kFileOther.
ImageHeader scan_image_header(const std::string& path);
void scan_image_headers(const std::vector<std::string>& paths, int threads, std::vector<ImageHeader>& out);

// Descriptor of one image of a decode batch, int32[kJpegDesc]:
//   [0] components: 0 raw RGB, 1 grey JPEG, 3 YCbCr JPEG
//   [1] [2] luma sampling (hmax, vmax): (1,1), (2,1) or (2,2); chroma is 1x1.  Grey: (1,1)
//   [3] first 8x8 block of the image in the batch's coefficient array (running total over the batch)
//   [4] raw RGB: byte offset in the batch's raw array
//   [5..7] blocks per row of component c, [8..10] block rows of component c (MCU padding included)
//   [11..13] row of component c's quantisation table in the batch's [rows][64] table array (natural order)
// Component c's blocks follow component c-1's, each component's row by row.
constexpr int kJpegDesc = 16;

// Block grid of component c of a stream-JPEG frame (interleaved when ncomp == 3).
inline void jpeg_block_grid(const ImageHeader& h, int c, int& bw, int& bh) {
  if (h.ncomp == 1) {
    bw = (h.W + 7) / 8;
    bh = (h.H + 7) / 8;
    return;
  }
  const int hmax = h.h[0], vmax = h.v[0];
  bw = (h.W + 8 * hmax - 1) / (8 * hmax) * h.h[c];
  bh = (h.H + 8 * vmax - 1) / (8 * vmax) * h.v[c];
}

// Entropy-decodes the stream-JPEG `path`, whose scan gave `hdr`: quantised coefficients in natural order,
// hdr.blocks x 64 int16 at `coef` in the descriptor's block order, and each component's quantisation table
// (64 values, natural order) at quant + 64 c.  Throws std::runtime_error naming the path for a malformed or
// truncated file, or one that no longer matches `hdr`.
void jpeg_entropy_decode(const std::string& path, const ImageHeader& hdr, int16_t* coef, int32_t* quant);

}  // namespace b200
