// Letterbox of photos of any size into the S x S model input: ImageOps.contain + ImageOps.pad with Pillow's 8-bit
// BICUBIC resampler, byte for byte (reference demo.py:27-51; the arithmetic is restated in oracle/letterbox_ref.py).
//
// The host computes, per photo, the contained size, the pad offsets and the int32 coefficient rows of both axes in
// double exactly as Pillow does (rows for a repeated (in, out) size are shared within a call) and uploads them with
// the per-photo descriptors in one copy.  The device then runs two launches for the whole batch:
//   first pass   photo -> uint8 workspace: normally the horizontal pass over only the photo rows the vertical windows
//                touch; for a photo more than 100x taller than wide that gets shorter, the vertical pass (Pillow's
//                Image.resize orders the passes that way for such photos).  Skipped for a photo whose width stays.
//   last pass    workspace (or the photo) -> the padded S x S output, pad included: the other axis, or a one-tap
//                identity row when that axis keeps its size (exact: (2^21 + p 2^22) >> 22 = p).
// Each thread makes one output byte (channel c of pixel x), so stores and the vertical taps are coalesced.
#include "common.cuh"

#include <algorithm>
#include <cmath>
#include <map>
#include <utility>
#include <vector>

using namespace mhmr;

namespace {

constexpr int kPrecisionBits = 22;  // 32 - 8 - 2: the fractional bits of Pillow's 8-bit coefficients
constexpr int kThreads = 256;

struct LbPass {
  const uint8_t* src;  // uint8 RGB rows, `pitch` bytes apart
  int64_t pitch;
  int row0;            // photo row of src's row 0 (the first row the horizontal pass kept), else 0
  int axis;            // 0: taps along x (output index = column); 1: taps along y (output index = row)
  int table;           // int32 offset of the coefficient rows: (xmin, n, k[taps]) per output index
  int taps;
};

struct LbImage {
  LbPass first, last;  // first: photo -> ws (absent when ws_rows == 0); last: -> out, pad included
  uint8_t* ws;         // [ws_rows, ws_cols, 3]
  int ws_rows, ws_cols;
  int x0, y0, nw, nh;  // the resized photo's box in the S x S output
  uint8_t* out;        // resize only: the [nh, nw, 3] output, `out_pitch` bytes per row
  int64_t out_pitch;
};

// One output byte: clip8((2^21 + sum_t src * k[t]) >> 22), summed in int32 as Pillow does.  The sum cannot overflow:
// the host checks 255 * sum|k| + 2^21 < 2^31 for every coefficient row (normalised Keys rows have sum|k| < 1.3 * 2^22,
// since the negative lobes hold well under a third of the positive mass).  Taps stay inside [0, in) of their axis, so
// no read leaves the photo's (or the workspace's) own rows and columns.
__device__ __forceinline__ uint8_t resample_byte(const LbPass& p, const int32_t* __restrict__ tab, int r, int x, int c) {
  const int32_t* e = tab + p.table + static_cast<int64_t>(p.axis == 0 ? x : r) * (p.taps + 2);
  const int xmin = __ldg(e), n = __ldg(e + 1);
  const uint8_t* s;
  int64_t step;
  if (p.axis == 0) {
    s = p.src + static_cast<int64_t>(r + p.row0) * p.pitch + 3ll * xmin + c;
    step = 3;
  } else {
    s = p.src + static_cast<int64_t>(xmin - p.row0) * p.pitch + 3ll * x + c;
    step = p.pitch;
  }
  int acc = 1 << (kPrecisionBits - 1);
  for (int t = 0; t < n; ++t) acc += static_cast<int>(__ldg(s + t * step)) * __ldg(e + 2 + t);
  return static_cast<uint8_t>(min(max(acc >> kPrecisionBits, 0), 255));
}

__global__ void __launch_bounds__(kThreads) letterbox_first_pass_kernel(const LbImage* __restrict__ imgs,
                                                                        const int32_t* __restrict__ tab) {
  const LbImage& im = imgs[blockIdx.z];
  const int j = blockIdx.x * kThreads + threadIdx.x;
  if (j >= 3 * im.ws_cols) return;
  const int x = j / 3, c = j - 3 * x;
  for (int r = blockIdx.y; r < im.ws_rows; r += gridDim.y)
    im.ws[static_cast<int64_t>(r) * 3 * im.ws_cols + j] = resample_byte(im.first, tab, r, x, c);
}

__global__ void __launch_bounds__(kThreads) letterbox_last_pass_kernel(const LbImage* __restrict__ imgs,
                                                                       const int32_t* __restrict__ tab, uint8_t* out,
                                                                       int S, int pad) {
  const LbImage& im = imgs[blockIdx.z];
  const int j = blockIdx.x * kThreads + threadIdx.x;
  if (j >= 3 * S) return;
  const int x = j / 3, c = j - 3 * x;
  const bool in_x = x >= im.x0 && x < im.x0 + im.nw;
  for (int y = blockIdx.y; y < S; y += gridDim.y) {
    uint8_t v = static_cast<uint8_t>(pad);
    if (in_x && y >= im.y0 && y < im.y0 + im.nh) v = resample_byte(im.last, tab, y - im.y0, x - im.x0, c);
    out[(static_cast<int64_t>(blockIdx.z) * S + y) * 3 * S + j] = v;
  }
}

// Image.resize's last pass: one output byte per thread, straight into each photo's own output rows.
__global__ void __launch_bounds__(kThreads) resize_last_pass_kernel(const LbImage* __restrict__ imgs,
                                                                    const int32_t* __restrict__ tab) {
  const LbImage& im = imgs[blockIdx.z];
  const int j = blockIdx.x * kThreads + threadIdx.x;
  if (j >= 3 * im.nw) return;
  const int x = j / 3, c = j - 3 * x;
  for (int y = blockIdx.y; y < im.nh; y += gridDim.y)
    im.out[static_cast<int64_t>(y) * im.out_pitch + j] = resample_byte(im.last, tab, y, x, c);
}

// ---- host: Pillow's arithmetic (plain double operations; the x86-64 host build emits no fused multiply-add) --------
double bicubic(double x) {  // Keys cubic, a = -0.5
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1.0;
  if (x < 2.0) return (((x - 5.0) * x + 8.0) * x - 4.0) * a;
  return 0.0;
}

int round_half_even(double v) { return static_cast<int>(std::nearbyint(v)); }  // Python's round(), default FE_TONEAREST

struct Tables {
  std::vector<int32_t> data;
  std::map<std::pair<int, int>, std::pair<int, int>> at;  // (in, out) -> (offset, taps)

  // Coefficient rows of one axis resampled from `in` to `out` samples, shared by every photo of the call that needs
  // them; in == out gives one-tap identity rows (the axis Pillow skips).  Returns false if a row could overflow the
  // int32 sum (not reached by normalised bicubic rows; checked rather than assumed).
  bool get(int in, int out, int* offset, int* taps) {
    auto it = at.find({in, out});
    if (it != at.end()) {
      *offset = it->second.first;
      *taps = it->second.second;
      return true;
    }
    *offset = static_cast<int>(data.size());
    if (in == out) {
      *taps = 1;
      for (int i = 0; i < out; ++i) data.insert(data.end(), {i, 1, 1 << kPrecisionBits});
    } else {
      const double scale = static_cast<double>(in) / out;
      const double filterscale = std::max(scale, 1.0);
      const double support = 2.0 * filterscale;
      const double inv = 1.0 / filterscale;
      *taps = static_cast<int>(std::ceil(support)) * 2 + 1;
      std::vector<double> w(*taps);
      for (int i = 0; i < out; ++i) {
        const double center = (i + 0.5) * scale;
        const int xmin = std::max(static_cast<int>(center - support + 0.5), 0);  // truncation, as in C
        const int n = std::min(static_cast<int>(center + support + 0.5), in) - xmin;
        double ww = 0.0;
        for (int t = 0; t < n; ++t) {
          w[t] = bicubic((t + xmin - center + 0.5) * inv);
          ww += w[t];
        }
        data.push_back(xmin);
        data.push_back(n);
        int64_t mass = 0;
        for (int t = 0; t < *taps; ++t) {
          const double v = t < n ? (ww != 0.0 ? w[t] / ww : w[t]) : 0.0;
          const double s = v * static_cast<double>(1 << kPrecisionBits);
          const int32_t k = static_cast<int32_t>(v < 0.0 ? -0.5 + s : 0.5 + s);  // half away from zero
          mass += k < 0 ? -static_cast<int64_t>(k) : k;
          data.push_back(k);
        }
        if (255 * mass + (1 << (kPrecisionBits - 1)) >= (1ll << 31)) return false;
      }
    }
    at[{in, out}] = {*offset, *taps};
    return true;
  }
  const int32_t* row(int offset, int taps, int i) const { return data.data() + offset + static_cast<int64_t>(i) * (taps + 2); }
};

// Image.resize((nw, nh), BICUBIC) of one photo as passes over the shared coefficient rows: which axis goes first, the
// workspace it needs, and the source of the last pass (see the top of this file).  False if a coefficient row could
// overflow the int32 sum.
bool plan(Tables& tab, const uint8_t* src, int64_t pitch, int64_t H, int64_t W, int nw, int nh, LbImage& im) {
  int hoff, htaps, voff, vtaps;
  if (!tab.get(static_cast<int>(W), nw, &hoff, &htaps) || !tab.get(static_cast<int>(H), nh, &voff, &vtaps)) return false;
  const LbPass horiz{src, pitch, 0, 0, hoff, htaps}, vert{src, pitch, 0, 1, voff, vtaps};
  if (H > 100 * W && nh < H) {  // vertical first: photo -> ws [nh, W], then horizontal ws -> out
    im.first = vert;
    im.ws_rows = nh;
    im.ws_cols = static_cast<int>(W);
    im.last = horiz;
    im.last.pitch = 3 * W;
  } else if (nw != W) {  // horizontal over the rows the vertical windows touch, then vertical ws -> out
    const int y_first = tab.row(voff, vtaps, 0)[0];
    const int32_t* lastrow = tab.row(voff, vtaps, nh - 1);
    im.first = horiz;
    im.first.row0 = y_first;
    im.ws_rows = lastrow[0] + lastrow[1] - y_first;
    im.ws_cols = nw;
    im.last = vert;
    im.last.row0 = y_first;
    im.last.pitch = 3ll * nw;
  } else {  // the width stays: one (vertical or identity) pass from the photo
    im.ws_rows = 0;
    im.ws_cols = 0;
    im.last = vert;
  }
  return true;
}

}  // namespace

extern "C" {

int mhmr_op_letterbox_u8(const int64_t* photos, int B, int S, int pad, uint8_t* out, int32_t* boxes, void* stream) {
  MHMR_REQUIRE(photos != nullptr && out != nullptr, "null argument");
  MHMR_REQUIRE(B >= 1 && B <= 65535, "letterbox: 1 <= B <= 65535 photos");
  MHMR_REQUIRE(S >= 1 && S <= 32768, "letterbox: 1 <= S <= 32768");
  MHMR_REQUIRE(pad >= 0 && pad <= 255, "letterbox: the pad value is a byte");
  std::vector<LbImage> imgs(B);
  std::vector<int> box(4 * B);
  Tables tab;
  for (int b = 0; b < B; ++b) {
    const int64_t* d = photos + 4 * b;
    const int64_t H = d[1], W = d[2], pitch = d[3];
    MHMR_REQUIRE(d[0] != 0, "letterbox: null photo");
    MHMR_REQUIRE(H >= 1 && W >= 1 && H <= (1 << 20) && W <= (1 << 20), "letterbox: photo sides in [1, 2^20]");
    MHMR_REQUIRE(pitch >= 3 * W, "letterbox: row pitch below 3 W bytes");
    // ImageOps.contain: the long side becomes S, the short one round(short / long * S) (half to even)
    int nw = S, nh = S;
    const double ratio = static_cast<double>(W) / static_cast<double>(H);
    if (ratio != 1.0) {
      if (ratio > 1.0)
        nh = round_half_even(static_cast<double>(H) / static_cast<double>(W) * S);
      else
        nw = round_half_even(static_cast<double>(W) / static_cast<double>(H) * S);
    }
    MHMR_REQUIRE(nw >= 1 && nh >= 1, "letterbox: the photo's short side rounds to 0 pixels (Pillow raises too)");
    LbImage& im = imgs[b];
    im.nw = nw;
    im.nh = nh;
    im.x0 = round_half_even((S - nw) * 0.5);  // ImageOps.pad, centering 0.5
    im.y0 = round_half_even((S - nh) * 0.5);
    MHMR_REQUIRE(plan(tab, reinterpret_cast<const uint8_t*>(d[0]), pitch, H, W, nw, nh, im),
                 "letterbox: a coefficient row could overflow the int32 sum");
    box[4 * b] = im.x0; box[4 * b + 1] = im.y0; box[4 * b + 2] = nw; box[4 * b + 3] = nh;
  }
  MHMR_REQUIRE(tab.data.size() < (1ull << 31), "letterbox: coefficient tables too large");

  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallScratch ws(st);
  const size_t r_imgs = ws.region(sizeof(LbImage) * B, true), r_tab = ws.region(4 * tab.data.size(), true);
  std::vector<size_t> r_ws(B);
  for (int b = 0; b < B; ++b) r_ws[b] = ws.region(static_cast<size_t>(imgs[b].ws_rows) * 3 * imgs[b].ws_cols);
  TRY(ws.allocate());
  int max_cols = 0, max_rows = 0;
  for (int b = 0; b < B; ++b) {
    LbImage& im = imgs[b];
    if (im.ws_rows > 0) {
      im.ws = ws.dev<uint8_t>(r_ws[b]);
      im.last.src = im.ws;
      max_cols = std::max(max_cols, im.ws_cols);
      max_rows = std::max(max_rows, im.ws_rows);
    }
  }
  std::copy_n(imgs.data(), B, ws.host<LbImage>(r_imgs));
  std::copy_n(tab.data.data(), tab.data.size(), ws.host<int32_t>(r_tab));
  const LbImage* d_imgs = ws.dev<const LbImage>(r_imgs);
  const int32_t* d_tab = ws.dev<const int32_t>(r_tab);
  TRY(ws.upload());
  if (max_rows > 0) {
    const dim3 grid((3 * max_cols + kThreads - 1) / kThreads, std::min(max_rows, 65535), B);
    letterbox_first_pass_kernel<<<grid, kThreads, 0, st>>>(d_imgs, d_tab);
    MHMR_CUDA_CHECK(cudaGetLastError());
  }
  const dim3 grid((3 * S + kThreads - 1) / kThreads, std::min(S, 65535), B);
  letterbox_last_pass_kernel<<<grid, kThreads, 0, st>>>(d_imgs, d_tab, out, S, pad);
  MHMR_CUDA_CHECK(cudaGetLastError());
  TRY(ws.release());
  if (boxes != nullptr) std::copy(box.begin(), box.end(), boxes);
  return MHMR_OK;
}

int mhmr_op_resize_u8(const int64_t* photos, int B, void* stream) {
  MHMR_REQUIRE(B >= 0 && B <= 65535, "resize: 0 <= B <= 65535 photos");
  if (B == 0) return MHMR_OK;
  MHMR_REQUIRE(photos != nullptr, "null argument");
  std::vector<LbImage> imgs(B);
  Tables tab;
  int max_nw = 0, max_nh = 0;
  for (int b = 0; b < B; ++b) {
    const int64_t* d = photos + 8 * b;
    const int64_t H = d[1], W = d[2], pitch = d[3], nh = d[5], nw = d[6], out_pitch = d[7];
    MHMR_REQUIRE(d[0] != 0 && d[4] != 0, "resize: null photo or output");
    MHMR_REQUIRE(H >= 1 && W >= 1 && H <= (1 << 20) && W <= (1 << 20), "resize: photo sides in [1, 2^20]");
    MHMR_REQUIRE(nh >= 1 && nw >= 1 && nh <= (1 << 20) && nw <= (1 << 20), "resize: output sides in [1, 2^20]");
    MHMR_REQUIRE(pitch >= 3 * W && out_pitch >= 3 * nw, "resize: row pitch below 3 W bytes");
    LbImage& im = imgs[b];
    im.nw = static_cast<int>(nw);
    im.nh = static_cast<int>(nh);
    im.out = reinterpret_cast<uint8_t*>(d[4]);
    im.out_pitch = out_pitch;
    MHMR_REQUIRE(plan(tab, reinterpret_cast<const uint8_t*>(d[0]), pitch, H, W, im.nw, im.nh, im),
                 "resize: a coefficient row could overflow the int32 sum");
    max_nw = std::max(max_nw, im.nw);
    max_nh = std::max(max_nh, im.nh);
  }
  MHMR_REQUIRE(tab.data.size() < (1ull << 31), "resize: coefficient tables too large");

  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallScratch ws(st);
  const size_t r_imgs = ws.region(sizeof(LbImage) * B, true), r_tab = ws.region(4 * tab.data.size(), true);
  std::vector<size_t> r_ws(B);
  for (int b = 0; b < B; ++b) r_ws[b] = ws.region(static_cast<size_t>(imgs[b].ws_rows) * 3 * imgs[b].ws_cols);
  TRY(ws.allocate());
  int max_cols = 0, max_rows = 0;
  for (int b = 0; b < B; ++b) {
    LbImage& im = imgs[b];
    if (im.ws_rows > 0) {
      im.ws = ws.dev<uint8_t>(r_ws[b]);
      im.last.src = im.ws;
      max_cols = std::max(max_cols, im.ws_cols);
      max_rows = std::max(max_rows, im.ws_rows);
    }
  }
  std::copy_n(imgs.data(), B, ws.host<LbImage>(r_imgs));
  std::copy_n(tab.data.data(), tab.data.size(), ws.host<int32_t>(r_tab));
  const LbImage* d_imgs = ws.dev<const LbImage>(r_imgs);
  const int32_t* d_tab = ws.dev<const int32_t>(r_tab);
  TRY(ws.upload());
  if (max_rows > 0) {
    const dim3 grid((3 * max_cols + kThreads - 1) / kThreads, std::min(max_rows, 65535), B);
    letterbox_first_pass_kernel<<<grid, kThreads, 0, st>>>(d_imgs, d_tab);
    MHMR_CUDA_CHECK(cudaGetLastError());
  }
  const dim3 grid((3 * max_nw + kThreads - 1) / kThreads, std::min(max_nh, 65535), B);
  resize_last_pass_kernel<<<grid, kThreads, 0, st>>>(d_imgs, d_tab);
  MHMR_CUDA_CHECK(cudaGetLastError());
  TRY(ws.release());
  return MHMR_OK;
}

}  // extern "C"
