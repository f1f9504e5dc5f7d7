// video_pipeline.cu -- f-2: the file-driven frame loop of fast_artistic_video.lua:93-170 as a native host pipeline around the
// host-buffer session (session.cu).  The reference decodes, uploads, stylizes, downloads and encodes one frame after the other
// (image.load / flowFile.load in interpreted Lua, image.save); at H100 speeds that host work bounds the frame rate by two
// orders of magnitude.  Here:
//   decoder threads   read the PAYLOADS of frame PPM, certainty PGM and Middlebury .flo straight into PINNED ring slots
//                     (cudaHostAlloc); byte -> fp32 / 255, 1 - cert, (u,v) -> (dy,dx) planes happen on the GPU behind the H2D
//                     copy (session.cu: decode_bytes_kernel); the wait-for-file protocol of the flow / occlusion producers
//                     (utils.lua:74-80) and the [fmt] / {fmt} filename patterns (fast_artistic_video.lua:70-77) are kept
//   calling thread    only enqueues frames on the session (3 CUDA streams inside: H2D / compute / D2H)
//   completer thread  waits for the session's per-frame completion events in order (fav_session_frame_done)
//   encoder threads   deflate the landed Sub-filtered scanlines (quantised like image.save -- clamp, x255, round -- on the GPU
//                     before the D2H copy: session.cu: encode_rows_kernel) and write "<prefix>-%05d.png"
//                     (fast_artistic_video.lua:161); any PNG decoder returns the same pixels as the synchronous driver's files
// FAV_PIPE_STATS=1 prints where the host time went.
// Host code only (no kernels); compiled by nvcc for the CUDA runtime calls.
#include <zlib.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include <math.h>
#include <string.h>
#include <sys/stat.h>

#include "fav_common.cuh"

namespace fav {
namespace {

// {fmt} is formatted with the from-index, [fmt] with the to-index (fast_artistic_video.lua:70-77)
std::string format_flow_name(const std::string &pattern, int fromIndex, int toIndex) {
  std::string out;
  for (size_t i = 0; i < pattern.size();) {
    const char ch = pattern[i];
    const char close = ch == '{' ? '}' : (ch == '[' ? ']' : 0);
    size_t j = close ? pattern.find(close, i + 1) : std::string::npos;
    if (close && j != std::string::npos) {
      char buf[64];
      snprintf(buf, sizeof(buf), pattern.substr(i + 1, j - i - 1).c_str(), ch == '{' ? fromIndex : toIndex);
      out += buf;
      i = j + 1;
    } else {
      out += ch;
      ++i;
    }
  }
  return out;
}
std::string format_index(const std::string &pattern, int idx) {
  char buf[4096];
  snprintf(buf, sizeof(buf), pattern.c_str(), idx);
  return buf;
}
bool file_exists(const std::string &p) {
  struct stat st;
  return stat(p.c_str(), &st) == 0 && S_ISREG(st.st_mode);
}

void put_be32(std::vector<unsigned char> &v, uint32_t x) {
  v.push_back(x >> 24); v.push_back(x >> 16); v.push_back(x >> 8); v.push_back(x);
}
void png_chunk(std::vector<unsigned char> &out, const char type[4], const unsigned char *data, size_t n) {
  put_be32(out, (uint32_t)n);
  const size_t start = out.size();
  out.insert(out.end(), type, type + 4);
  if (n) out.insert(out.end(), data, data + n);
  put_be32(out, (uint32_t)crc32(0, out.data() + start, (uInt)(n + 4)));
}
// 8-bit PNG (colour type 2 RGB or 0 gray, no interlace) from scanlines that are already Sub-filtered (filter byte 1 + C*W bytes
// per row).  level 0 = stored; level 1 = zlib level 1 with Z_RLE (what libpng recommends for filtered rows when speed matters:
// on a stylized 720p frame 32 ms instead of 72 ms at the same size); level >= 2 = that zlib level with Z_FILTERED.
// nthreads > 1: the rows are cut into bands that are deflated concurrently as raw streams ending in a full flush (the last one
// in Z_FINISH) and concatenated behind one zlib header, the Adler-32 of the whole image combined from the bands' -- the
// 12288 x 2048 cube-map strips of the VR driver take seconds on one core.
int deflate_band(const unsigned char *raw, size_t n, int level, bool last, std::vector<unsigned char> &z, uLong *adler) {
  z_stream zs;
  memset(&zs, 0, sizeof(zs));
  if (deflateInit2(&zs, level, Z_DEFLATED, -15, 9, level <= 1 ? Z_RLE : Z_FILTERED) != Z_OK) return FAV_ERR_IO;
  z.resize(deflateBound(&zs, (uLong)n) + 16);
  zs.next_in = const_cast<unsigned char *>(raw); zs.avail_in = (uInt)n;
  zs.next_out = z.data(); zs.avail_out = (uInt)z.size();
  const int zrc = deflate(&zs, last ? Z_FINISH : Z_FULL_FLUSH);
  const bool ok = last ? zrc == Z_STREAM_END : (zrc == Z_OK && zs.avail_in == 0 && zs.avail_out > 0);
  z.resize(zs.total_out);
  deflateEnd(&zs);
  *adler = adler32(adler32(0L, Z_NULL, 0), raw, (uInt)n);
  return ok ? FAV_OK : FAV_ERR_IO;
}

int write_png_rows(const std::string &path, const unsigned char *raw, int W, int H, int C, int level, int nthreads,
                   std::vector<unsigned char> &out) {
  const size_t row = 1 + (size_t)C * W;
  const int max_bands = (int)std::max<size_t>(1, (row * H) / (1u << 20));  // >= 1 MiB of scanlines per band
  const int nb = std::max(1, std::min(std::min(nthreads, H), max_bands));
  std::vector<std::vector<unsigned char>> z(nb);
  std::vector<uLong> adl(nb);
  std::vector<size_t> len(nb);
  std::vector<int> rc(nb, FAV_OK);
  auto band = [&](int b) {
    const int y0 = (int)((int64_t)H * b / nb), y1 = (int)((int64_t)H * (b + 1) / nb);
    len[b] = (size_t)(y1 - y0) * row;
    rc[b] = deflate_band(raw + (size_t)y0 * row, len[b], level, b == nb - 1, z[b], &adl[b]);
  };
  if (nb == 1) {
    band(0);
  } else {
    std::vector<std::thread> th;
    for (int b = 0; b < nb; ++b) th.emplace_back(band, b);
    for (std::thread &t : th) t.join();
  }
  size_t zn = 2 + 4;
  uLong adler = adl[0];
  for (int b = 0; b < nb; ++b) {
    if (rc[b] != FAV_OK) return rc[b];
    zn += z[b].size();
    if (b) adler = adler32_combine(adler, adl[b], (z_off_t)len[b]);
  }
  out.clear();
  out.reserve(zn + 64);
  const unsigned char sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
  out.insert(out.end(), sig, sig + 8);
  std::vector<unsigned char> ihdr;
  put_be32(ihdr, (uint32_t)W); put_be32(ihdr, (uint32_t)H);
  const unsigned char tail[5] = {8, (unsigned char)(C == 3 ? 2 : 0), 0, 0, 0};
  ihdr.insert(ihdr.end(), tail, tail + 5);
  png_chunk(out, "IHDR", ihdr.data(), ihdr.size());
  put_be32(out, (uint32_t)zn);  // IDAT: zlib header, the bands, Adler-32
  const size_t start = out.size();
  out.insert(out.end(), {'I', 'D', 'A', 'T', 0x78, 0x01});
  for (int b = 0; b < nb; ++b) out.insert(out.end(), z[b].begin(), z[b].end());
  put_be32(out, (uint32_t)adler);
  put_be32(out, (uint32_t)crc32(crc32(0L, Z_NULL, 0), out.data() + start, (uInt)(out.size() - start)));
  png_chunk(out, "IEND", nullptr, 0);
  FILE *f = fopen(path.c_str(), "wb");
  if (!f) return FAV_ERR_IO;
  const bool ok = fwrite(out.data(), 1, out.size(), f) == out.size();
  fclose(f);
  return ok ? FAV_OK : FAV_ERR_IO;
}

inline double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

struct Slot {  // pinned; file payloads in, PNG scanlines out (the byte <-> float conversions happen on the GPU)
  unsigned char *rgb = nullptr, *cert = nullptr, *rows = nullptr;
  float *flo = nullptr;
};

}  // namespace
}  // namespace fav

using namespace fav;

extern "C" {

// image.save(path, img) for an 8-bit image that is already quantised: pixels = H x W x C bytes (C = 3 RGB or 1 gray, interleaved);
// Sub-filters the rows and writes the PNG with `nthreads` concurrent deflate bands (fast_artistic_video.lua:161,
// fast_artistic_video_vr.lua:541-556 write 8-bit PNGs through the `image` rock; any decoder returns the same pixels).
int fav_png_write(const char *path, const unsigned char *pixels, int W, int H, int C, int png_level, int nthreads) {
  FAV_REQUIRE(path && pixels && W > 0 && H > 0 && (C == 1 || C == 3), "fav_png_write: bad argument");
  FAV_REQUIRE((uint64_t)W * C * (uint64_t)H < (1ull << 31), "fav_png_write: image too large for one IDAT chunk");
  png_level = png_level < 0 ? 1 : (png_level > 9 ? 9 : png_level);
  const size_t row = 1 + (size_t)C * W;
  std::vector<unsigned char> raw(row * H), file;
  const int nt = nthreads < 1 ? 1 : (nthreads > 64 ? 64 : nthreads);
  auto filter = [&](int y0, int y1) {
    for (int y = y0; y < y1; ++y) {
      unsigned char *dst = raw.data() + (size_t)y * row;
      const unsigned char *src = pixels + (size_t)y * C * W;
      *dst++ = 1;
      for (int i = 0; i < C * W; ++i) dst[i] = (unsigned char)(src[i] - (i >= C ? src[i - C] : 0));
    }
  };
  if (nt == 1 || H < 64) {
    filter(0, H);
  } else {
    std::vector<std::thread> th;
    for (int t = 0; t < nt; ++t) th.emplace_back(filter, (int)((int64_t)H * t / nt), (int)((int64_t)H * (t + 1) / nt));
    for (std::thread &t : th) t.join();
  }
  if (write_png_rows(path, raw.data(), W, H, C, png_level, nt, file) != FAV_OK) {
    set_error("fav_png_write: cannot write %s", path);
    return FAV_ERR_IO;
  }
  return FAV_OK;
}

// Runs the whole clip; blocks until the last PNG is on disk.  Frames are <input_pattern % i>, i = 1..; the loop ends at
// num_frames or at the first missing frame file (func_load_image returning nil, fast_artistic_video.lua:93-97).
// frames_done / seconds (may be NULL) report what was processed.
int fav_video_pipeline_run(fav_session_t *sess, int H, int W, const char *input_pattern, const char *flow_pattern,
                           const char *occlusions_pattern, const char *output_prefix, int num_frames, int min_filter_r,
                           int invert_occlusion, int n_decode, int n_encode, int depth, int png_level, int *frames_done,
                           double *seconds) {
  FAV_REQUIRE(sess && input_pattern && flow_pattern && occlusions_pattern && output_prefix, "fav_video_pipeline_run: null argument");
  FAV_REQUIRE(H > 0 && W > 0 && num_frames >= 0, "fav_video_pipeline_run: bad size");
  n_decode = n_decode < 1 ? 1 : n_decode; n_encode = n_encode < 1 ? 1 : n_encode;
  depth = depth < 4 ? 4 : (depth > 60 ? 60 : depth);  // <= the session's ring of 64 per-frame completion events
  png_level = png_level < 0 ? 1 : (png_level > 9 ? 9 : png_level);
  int n = 0;
  while (n < num_frames && file_exists(format_index(input_pattern, n + 1))) ++n;
  if (frames_done) *frames_done = n;
  if (seconds) *seconds = 0;
  if (n == 0) return FAV_OK;
  const size_t HW = (size_t)H * W;
  std::vector<Slot> slots(depth);
  const size_t row_bytes = (size_t)H * (1 + 3 * (size_t)W);
  auto free_slots = [&]() {
    for (Slot &s : slots) { cudaFreeHost(s.rgb); cudaFreeHost(s.flo); cudaFreeHost(s.cert); cudaFreeHost(s.rows); }
  };
  for (Slot &s : slots)
    if (cudaHostAlloc((void **)&s.rgb, 3 * HW, cudaHostAllocDefault) != cudaSuccess ||
        cudaHostAlloc((void **)&s.flo, 2 * HW * 4, cudaHostAllocDefault) != cudaSuccess ||
        cudaHostAlloc((void **)&s.cert, HW, cudaHostAllocDefault) != cudaSuccess ||
        cudaHostAlloc((void **)&s.rows, row_bytes, cudaHostAllocDefault) != cudaSuccess) {
      (void)cudaGetLastError();
      free_slots();
      set_error("fav_video_pipeline_run: cannot allocate %d pinned frame slots", depth);
      return FAV_ERR_CUDA;
    }
  std::mutex mu;
  std::condition_variable cv_free, cv_dec, cv_enq, cv_done;  // one per class of waiter (no thundering herd of ~50 threads)
  std::atomic<int> next_decode{1}, next_encode{1};
  std::vector<int> ready(n + 2, 0);  // per frame: 1 decoded, 2 enqueued on the GPU, 3 landed in host memory, 4 written
  int err = FAV_OK;
  std::string err_msg;
  auto fail = [&](int code, const std::string &msg) {
    std::lock_guard<std::mutex> lk(mu);
    if (err == FAV_OK) { err = code; err_msg = msg; }
    cv_free.notify_all(); cv_dec.notify_all(); cv_enq.notify_all(); cv_done.notify_all();
  };
  auto wait_for_file = [&](const std::string &path) {  // utils.lua:74-80
    if (file_exists(path)) return true;
    fprintf(stderr, "Waiting for file \"%s\"\n", path.c_str());
    while (!file_exists(path)) {
      { std::lock_guard<std::mutex> lk(mu); if (err != FAV_OK) return false; }
      std::this_thread::sleep_for(std::chrono::seconds(1));
    }
    std::this_thread::sleep_for(std::chrono::seconds(1));
    return true;
  };
  const std::string in_pat(input_pattern), flow_pat(flow_pattern), occ_pat(occlusions_pattern), out_prefix(output_prefix);

  std::atomic<long long> t_decode{0}, t_png{0}, t_enc_wait{0}, t_dec_wait{0}, t_enq_wait{0};  // microseconds, all threads
  auto us = [](double a, double b) { return (long long)((b - a) * 1e6); };
  auto decoder = [&]() {
    for (;;) {
      const int i = next_decode.fetch_add(1);
      if (i > n) return;
      Slot &s = slots[(i - 1) % depth];
      const double w0 = now_s();
      {  // the slot is free once frame i - depth has been written
        std::unique_lock<std::mutex> lk(mu);
        cv_free.wait(lk, [&] { return err != FAV_OK || i <= depth || ready[i - depth] == 4; });
        if (err != FAV_OK) return;
      }
      const double w1 = now_s();
      int w = 0, h = 0, c = 0;
      const std::string frame_name = format_index(in_pat, i);
      int rc = fav_pnm_read_u8(frame_name.c_str(), s.rgb, 3 * HW, &w, &h, &c);
      if (rc == FAV_OK && (w != W || h != H || c != 3)) { fail(FAV_ERR_IO, frame_name + ": not a " + std::to_string(W) + "x" + std::to_string(H) + " P6 image"); return; }
      if (rc == FAV_OK && i > 1) {
        const std::string cert_name = format_flow_name(occ_pat, i - 1, i), flow_name = format_flow_name(flow_pat, i - 1, i);
        if (!wait_for_file(cert_name)) return;  // func_load_cert :99-103
        rc = fav_pnm_read_u8(cert_name.c_str(), s.cert, HW, &w, &h, &c);
        if (rc == FAV_OK && (w != W || h != H || c != 1)) { fail(FAV_ERR_IO, cert_name + ": size / type mismatch"); return; }
        if (rc == FAV_OK) {
          if (!wait_for_file(flow_name)) return;
          rc = fav_flo_read_raw(flow_name.c_str(), s.flo, 2 * HW, &w, &h);
          if (rc == FAV_OK && (w != W || h != H)) { fail(FAV_ERR_IO, flow_name + ": size mismatch"); return; }
        }
      }
      if (rc != FAV_OK) { fail(rc, fav_last_error()); return; }
      { std::lock_guard<std::mutex> lk(mu); ready[i] = 1; }
      cv_dec.notify_all();
      t_dec_wait += us(w0, w1); t_decode += us(w1, now_s());
    }
  };
  auto encoder = [&]() {
    std::vector<unsigned char> file;
    for (;;) {
      const int i = next_encode.fetch_add(1);
      if (i > n) return;
      const double w0 = now_s();
      {
        std::unique_lock<std::mutex> lk(mu);
        cv_done.wait(lk, [&] { return err != FAV_OK || ready[i] == 3; });
        if (err != FAV_OK) return;
      }
      const double w1 = now_s();
      const Slot &s = slots[(i - 1) % depth];
      char name[4096];
      snprintf(name, sizeof(name), "%s-%05d.png", out_prefix.c_str(), i);
      if (write_png_rows(name, s.rows, W, H, 3, png_level, 1, file) != FAV_OK) { fail(FAV_ERR_IO, std::string("cannot write ") + name); return; }
      { std::lock_guard<std::mutex> lk(mu); ready[i] = 4; }
      cv_free.notify_all();
      t_enc_wait += us(w0, w1); t_png += us(w1, now_s());
    }
  };
  // frames complete in order: ONE thread waits on the session's per-frame events (dozens of encoder threads blocking in the
  // CUDA runtime contend with the enqueueing thread for the context lock: measured 150-200 instead of 600+ frames/s)
  auto completer = [&]() {
    for (int i = 1; i <= n; ++i) {
      {
        std::unique_lock<std::mutex> lk(mu);
        cv_enq.wait(lk, [&] { return err != FAV_OK || ready[i] == 2; });
        if (err != FAV_OK) return;
      }
      if (fav_session_frame_done(sess, (uint64_t)(i - 1), 1) != FAV_OK) { fail(FAV_ERR_CUDA, fav_last_error()); return; }
      { std::lock_guard<std::mutex> lk(mu); ready[i] = 3; }
      cv_done.notify_all();
    }
  };

  const auto t0 = std::chrono::steady_clock::now();
  std::vector<std::thread> threads;
  for (int t = 0; t < n_decode; ++t) threads.emplace_back(decoder);
  for (int t = 0; t < n_encode; ++t) threads.emplace_back(encoder);
  threads.emplace_back(completer);
  for (int i = 1; i <= n; ++i) {
    {
      const double w0 = now_s();
      std::unique_lock<std::mutex> lk(mu);
      cv_dec.wait(lk, [&] { return err != FAV_OK || ready[i] == 1; });
      t_enq_wait += us(w0, now_s());
      if (err != FAV_OK) break;
    }
    Slot &s = slots[(i - 1) % depth];
    const int rc = fav_session_run_frame_bytes(sess, s.rgb, i == 1 ? nullptr : s.flo, i == 1 ? nullptr : s.cert, invert_occlusion,
                                               min_filter_r, FAV_BORDER_PER_TAP, s.rows);
    if (rc != FAV_OK) { fail(rc, fav_last_error()); break; }
    { std::lock_guard<std::mutex> lk(mu); ready[i] = 2; }
    cv_enq.notify_all();
  }
  for (std::thread &t : threads) t.join();
  fav_session_sync(sess);
  const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  free_slots();
  if (seconds) *seconds = dt;
  if (getenv("FAV_PIPE_STATS"))  // where the host time went: per-frame averages over all worker threads
    fprintf(stderr, "{\"pipeline_stats\": {\"frames\": %d, \"seconds\": %.4f, \"decode_ms\": %.2f, \"decode_wait_slot_ms\": %.2f, "
            "\"deflate_write_ms\": %.2f, \"encode_wait_frame_ms\": %.2f, \"enqueue_wait_decode_ms\": %.2f, "
            "\"n_decode\": %d, \"n_encode\": %d, \"depth\": %d, \"png_level\": %d}}\n",
            n, dt, t_decode / 1e3 / n, t_dec_wait / 1e3 / n, t_png / 1e3 / n, t_enc_wait / 1e3 / n,
            t_enq_wait / 1e3 / n, n_decode, n_encode, depth, png_level);
  if (err != FAV_OK) { set_error("fav_video_pipeline_run: %s", err_msg.c_str()); return err; }
  return FAV_OK;
}
}
