// Native batch prefetcher (SURVEY N9): a C++ worker thread that, per mini-batch, gathers the
// sampled uint8 images from the decoded cache into a pinned staging ring, draws the
// RandomResizedCrop / RandomRotation / RandomHorizontalFlip parameters (torchvision's
// distributions) and publishes the slot.  It never takes the Python GIL, so it cannot stall the
// thread that launches the training step (a Python producer thread does: with the GIL's 5 ms switch
// interval the launch loop of a training step is held up).
//
// Stream splits (PrefetchConfig::stream): nothing is cached.  The worker lays each batch out in the slot (every
// JPEG's coefficient blocks, every other image's raw RGB, one descriptor row each, csrc/include/jpeg.h) and a pool
// of decode threads fills those fixed positions, so a slot's content does not depend on the thread count or on
// timing.  A failed decode ends the epoch: next() raises the error once the batches before it are consumed.
//
// Slot life cycle:  free -> (worker fills) -> ready -> (consumer: next()) -> in use ->
// (consumer: release(slot, cuda_event)) -> free; the worker cudaEventSynchronize()s the event the
// consumer recorded after its host->device copy before it overwrites the slot.
#include <cuda_runtime.h>

#include <cmath>
#include <condition_variable>
#include <cstdint>
#include <cstring>
#include <algorithm>
#include <deque>
#include <memory>
#include <functional>
#include <mutex>
#include <random>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "jpeg.h"

namespace b200 {

struct PngImage {
  int w = 0, h = 0;
  std::vector<uint8_t> rgb;
  bool ok = false;
};
bool decode_png_file(const std::string& path, PngImage& out);

// The files of a stream split and the slot arrays their batches are decoded into.
struct StreamConfig {
  std::vector<std::string> paths;
  std::vector<ImageHeader> headers;
  const uint8_t* other = nullptr;        // files PIL decoded at start-up: RGB at other + other_off[i]
  const int64_t* other_off = nullptr;    // -1: not such a file
  int16_t* ring_coef = nullptr;          // [slots][coef_cap]
  int64_t coef_cap = 0;
  int32_t* ring_quant = nullptr;         // [slots][mb * 3][64]
  uint8_t* ring_raw = nullptr;           // [slots][raw_cap]
  int64_t raw_cap = 0;
  int32_t* ring_desc = nullptr;          // [slots][mb][kJpegDesc]
  int threads = 8;
};

// fn(i) for i in [0, n) on a fixed set of threads; run() returns the first error's message ("" if none).
class DecodePool {
 public:
  explicit DecodePool(int n) {
    for (int t = 0; t < std::max(n, 1); ++t) threads_.emplace_back([this] { loop(); });
  }
  ~DecodePool() {
    {
      std::lock_guard<std::mutex> lk(mu_);
      quit_ = true;
    }
    cv_work_.notify_all();
    for (auto& t : threads_) t.join();
  }
  std::string run(int n, const std::function<void(int)>& fn) {
    std::unique_lock<std::mutex> lk(mu_);
    fn_ = &fn;
    n_ = n;
    next_ = done_ = 0;
    err_.clear();
    ++gen_;
    cv_work_.notify_all();
    cv_done_.wait(lk, [this] { return done_ == n_; });
    return err_;
  }

 private:
  void loop() {
    uint64_t seen = 0;
    std::unique_lock<std::mutex> lk(mu_);
    for (;;) {
      cv_work_.wait(lk, [&] { return quit_ || gen_ != seen; });
      if (quit_) return;
      seen = gen_;
      while (next_ < n_) {
        const int i = next_++;
        lk.unlock();
        std::string e;
        try {
          (*fn_)(i);
        } catch (const std::exception& x) {
          e = x.what();
        }
        lk.lock();
        if (!e.empty() && err_.empty()) err_ = e;
        if (++done_ == n_) cv_done_.notify_all();
      }
    }
  }
  std::vector<std::thread> threads_;
  std::mutex mu_;
  std::condition_variable cv_work_, cv_done_;
  const std::function<void(int)>* fn_ = nullptr;
  int n_ = 0, next_ = 0, done_ = 0;
  uint64_t gen_ = 0;
  bool quit_ = false;
  std::string err_;
};

struct PrefetchConfig {
  const uint8_t* cache;      // [N][H][W][3]
  const int64_t* labels;     // [N]
  int H, W, mb, slots;
  uint8_t* ring_img;         // [slots][mb][H][W][3]   (pinned)
  float* ring_par;           // [slots][mb][8]
  int64_t* ring_lab;         // [slots][mb]
  bool train;
  float scale_lo, scale_hi, ratio_lo, ratio_hi, degrees;
  // ragged splits (offsets != nullptr): the cache is one flat buffer, image i at offsets[i] with size
  // hw[i] = (H, W); a slot holds the batch's images back to back in slot_bytes, and ring_geom
  // [slots][mb][5] gets each sample's (offset in the slot, H, W, RH, RW)
  const int64_t* offsets = nullptr;
  const int64_t* hw = nullptr;
  int64_t* ring_geom = nullptr;
  int64_t slot_bytes = 0;
  int resize = 256;
  // stream splits: hw and ring_geom as above, no cache or offsets
  const StreamConfig* stream = nullptr;
};

class BatchPrefetcher {
 public:
  explicit BatchPrefetcher(const PrefetchConfig& c) : cfg_(c), events_(c.slots, nullptr) {
    for (int s = 0; s < c.slots; ++s) free_.push_back(s);
  }
  ~BatchPrefetcher() { stop(); }

  void start_epoch(std::vector<int64_t> indices, uint64_t seed) {
    stop();
    {
      std::lock_guard<std::mutex> lk(mu_);
      indices_ = std::move(indices);
      ready_.clear();
      error_.clear();
      done_ = false;
      quit_ = false;
      free_.clear();
      for (int s = 0; s < cfg_.slots; ++s) free_.push_back(s);
    }
    rng_.seed(seed);
    worker_ = std::thread([this] { run(); });
  }

  // Blocks until a batch is ready.  Returns false at the end of the epoch.
  bool next(int& slot, int& count) {
    std::unique_lock<std::mutex> lk(mu_);
    cv_ready_.wait(lk, [this] { return !ready_.empty() || done_; });
    if (ready_.empty()) {
      if (!error_.empty()) throw std::runtime_error(error_);
      return false;
    }
    slot = ready_.front().first;
    count = ready_.front().second;
    ready_.pop_front();
    return true;
  }

  void release(int slot, cudaEvent_t ev) {
    {
      std::lock_guard<std::mutex> lk(mu_);
      events_[slot] = ev;
      free_.push_back(slot);
    }
    cv_free_.notify_one();
  }

  void stop() {
    {
      std::lock_guard<std::mutex> lk(mu_);
      quit_ = true;
    }
    cv_free_.notify_all();
    if (worker_.joinable()) worker_.join();
  }

 private:
  double uni() { return std::generate_canonical<double, 53>(rng_); }

  // Parameters of one sample of an H x W source: the same draws, in the same order, for every size.
  void sample_params(float* p, int H, int W) {
    const PrefetchConfig& c = cfg_;
    if (!c.train) {
      p[0] = 0; p[1] = 0; p[2] = (float)H; p[3] = (float)W; p[4] = 1.f; p[5] = 0.f; p[6] = 0.f; p[7] = 0.f;
      return;
    }
    const double area = (double)H * W, llo = std::log(c.ratio_lo), lhi = std::log(c.ratio_hi);
    double cw = 0, ch = 0;
    bool ok = false;
    for (int t = 0; t < 10; ++t) {                      // every draw consumed: fixed RNG stride
      const double ta = area * (c.scale_lo + (c.scale_hi - c.scale_lo) * uni());
      const double ar = std::exp(llo + (lhi - llo) * uni());
      const double w = std::nearbyint(std::sqrt(ta * ar)), h = std::nearbyint(std::sqrt(ta / ar));
      if (!ok && w > 0 && w <= W && h > 0 && h <= H) { cw = w; ch = h; ok = true; }
    }
    const double u0 = uni(), u1 = uni(), ua = uni(), uf = uni();
    double top, left;
    if (ok) {
      top = std::fmin(std::floor(u0 * (H - ch + 1)), H - ch);
      left = std::fmin(std::floor(u1 * (W - cw + 1)), W - cw);
    } else {                                            // torchvision's centre-crop fallback
      const double in_ratio = (double)W / H;
      if (in_ratio < c.ratio_lo) { cw = W; ch = std::nearbyint(cw / c.ratio_lo); }
      else if (in_ratio > c.ratio_hi) { ch = H; cw = std::nearbyint(ch * c.ratio_hi); }
      else { cw = W; ch = H; }
      top = std::floor((H - ch) / 2); left = std::floor((W - cw) / 2);
    }
    const double theta = (-c.degrees + 2.0 * c.degrees * ua) * 3.14159265358979323846 / 180.0;
    p[0] = (float)top; p[1] = (float)left; p[2] = (float)ch; p[3] = (float)cw;
    p[4] = (float)std::cos(theta); p[5] = (float)std::sin(theta); p[6] = uf < 0.5 ? 1.f : 0.f; p[7] = 0.f;
  }

  void run() {
    const PrefetchConfig& c = cfg_;
    const size_t img_bytes = (size_t)c.H * c.W * 3;
    const size_t n = indices_.size();
    std::unique_ptr<DecodePool> pool;
    if (c.stream) pool.reset(new DecodePool(c.stream->threads));
    for (size_t b0 = 0; b0 < n; b0 += c.mb) {
      int slot;
      cudaEvent_t ev;
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_free_.wait(lk, [this] { return !free_.empty() || quit_; });
        if (quit_) {                      // stopped mid-epoch: a consumer blocked in next() must wake up
          done_ = true;
          lk.unlock();
          cv_ready_.notify_all();
          return;
        }
        slot = free_.front();
        free_.pop_front();
        ev = events_[slot];
        events_[slot] = nullptr;
      }
      if (ev) cudaEventSynchronize(ev);               // previous occupant's H2D copy has finished
      const int k = (int)std::min<size_t>(c.mb, n - b0);
      uint8_t* img = c.ring_img + (size_t)slot * c.mb * img_bytes;
      float* par = c.ring_par + (size_t)slot * c.mb * 8;
      int64_t* lab = c.ring_lab + (size_t)slot * c.mb;
      if (c.hw) {
        uint8_t* bytes = c.ring_img + (size_t)slot * c.slot_bytes;
        int64_t* geom = c.ring_geom + (size_t)slot * c.mb * 5;
        int64_t at = 0;
        for (int i = 0; i < k; ++i) {
          const int64_t src = indices_[b0 + i];
          const int H = (int)c.hw[src * 2], W = (int)c.hw[src * 2 + 1];
          const size_t n = (size_t)H * W * 3;
          if (c.offsets) std::memcpy(bytes + at, c.cache + c.offsets[src], n);
          int64_t* g = geom + (size_t)i * 5;
          g[0] = at; g[1] = H; g[2] = W;
          if (c.train) { g[3] = c.resize; g[4] = c.resize; }         // data/transforms.py::resized_dims
          else if (H <= W) { g[3] = c.resize; g[4] = std::max((int64_t)((double)c.resize * W / H), (int64_t)1); }
          else { g[3] = std::max((int64_t)((double)c.resize * H / W), (int64_t)1); g[4] = c.resize; }
          at += (int64_t)n;
          lab[i] = c.labels[src];
          sample_params(par + (size_t)i * 8, H, W);
        }
        if (c.stream) {
          const std::string err = fill_stream(*pool, slot, &indices_[b0], k);
          if (!err.empty()) {
            {
              std::lock_guard<std::mutex> lk(mu_);
              error_ = err;
              done_ = true;
            }
            cv_ready_.notify_all();
            return;
          }
        }
      } else {
        for (int i = 0; i < k; ++i) {
          const int64_t src = indices_[b0 + i];
          std::memcpy(img + (size_t)i * img_bytes, c.cache + (size_t)src * img_bytes, img_bytes);
          lab[i] = c.labels[src];
          sample_params(par + (size_t)i * 8, c.H, c.W);
        }
      }
      {
        std::lock_guard<std::mutex> lk(mu_);
        ready_.emplace_back(slot, k);
      }
      cv_ready_.notify_one();
    }
    {
      std::lock_guard<std::mutex> lk(mu_);
      done_ = true;
    }
    cv_ready_.notify_all();
  }

  // Lays the batch idx[0..k) out in the slot's stream arrays and decodes it on the pool.
  std::string fill_stream(DecodePool& pool, int slot, const int64_t* idx, int k) {
    const StreamConfig& s = *cfg_.stream;
    const int mb = cfg_.mb;
    int16_t* coef = s.ring_coef + (size_t)slot * s.coef_cap;
    int32_t* quant = s.ring_quant + (size_t)slot * mb * 3 * 64;
    uint8_t* raw = s.ring_raw + (size_t)slot * s.raw_cap;
    int32_t* desc = s.ring_desc + (size_t)slot * mb * kJpegDesc;
    int64_t blk = 0, at = 0;
    for (int i = 0; i < k; ++i) {
      const ImageHeader& h = s.headers[idx[i]];
      int32_t* d = desc + (size_t)i * kJpegDesc;
      std::fill(d, d + kJpegDesc, 0);
      d[3] = (int32_t)blk;
      if (h.kind == kFileJpeg) {
        d[0] = h.ncomp;
        d[1] = h.ncomp == 3 ? h.h[0] : 1;
        d[2] = h.ncomp == 3 ? h.v[0] : 1;
        for (int c = 0; c < h.ncomp; ++c) {
          jpeg_block_grid(h, c, d[5 + c], d[8 + c]);
          d[11 + c] = i * 3 + c;
        }
        blk += h.blocks;
      } else {
        const int64_t* hw = cfg_.hw + 2 * idx[i];
        d[4] = (int32_t)at;
        at += hw[0] * hw[1] * 3;
      }
    }
    if (blk * 64 > s.coef_cap || at > s.raw_cap) return "stream prefetcher: a batch does not fit its slot";
    return pool.run(k, [&](int i) {
      const int64_t src = idx[i];
      const ImageHeader& h = s.headers[src];
      const int32_t* d = desc + (size_t)i * kJpegDesc;
      const int64_t H = cfg_.hw[2 * src], W = cfg_.hw[2 * src + 1];
      if (h.kind == kFileJpeg) {
        jpeg_entropy_decode(s.paths[src], h, coef + (int64_t)d[3] * 64, quant + (size_t)i * 3 * 64);
      } else if (h.kind == kFilePng) {
        PngImage img;
        if (!decode_png_file(s.paths[src], img) || img.h != H || img.w != W)
          throw std::runtime_error(s.paths[src] + ": PNG decode failed or its size changed since the header scan");
        std::memcpy(raw + d[4], img.rgb.data(), img.rgb.size());
      } else {
        std::memcpy(raw + d[4], s.other + s.other_off[src], (size_t)(H * W * 3));
      }
    });
  }

  PrefetchConfig cfg_;
  std::vector<int64_t> indices_;
  std::deque<int> free_;
  std::deque<std::pair<int, int>> ready_;
  std::vector<cudaEvent_t> events_;
  std::mutex mu_;
  std::condition_variable cv_free_, cv_ready_;
  std::thread worker_;
  std::mt19937_64 rng_;
  bool done_ = false, quit_ = false;
  std::string error_;
};

BatchPrefetcher* prefetcher_create(const PrefetchConfig& c) { return new BatchPrefetcher(c); }
void prefetcher_destroy(BatchPrefetcher* p) { delete p; }
void prefetcher_start(BatchPrefetcher* p, std::vector<int64_t> idx, uint64_t seed) { p->start_epoch(std::move(idx), seed); }
bool prefetcher_next(BatchPrefetcher* p, int& slot, int& count) { return p->next(slot, count); }
void prefetcher_release(BatchPrefetcher* p, int slot, uint64_t cuda_event) {
  p->release(slot, reinterpret_cast<cudaEvent_t>(cuda_event));
}
void prefetcher_stop(BatchPrefetcher* p) { p->stop(); }

}  // namespace b200
