// letterbox.cu -- dataset congealing's pre-processing on the device: prepare_data.py:53-77 border_pad (Pillow's LANCZOS
// resize of 8-bit RGB + np.pad(mode='edge')) followed by congeal_dataset.py:23-26 prepro, for a ragged batch of images
// packed in one uint8 buffer.  Replaces two PIL calls, a float32 conversion and a full-resolution fp32 upload per image.
//
// Pillow resamples 8-bit images in two separable fixed-point passes over a uint8 intermediate; a pass is skipped when its
// axis keeps its size.  The coefficients (Resample.c precompute_coeffs + normalize_coeffs_8bpc) are computed here in
// float64 with every operation rounded on its own, then rounded to 22 fractional bits.  Pillow 12.2 runs the horizontal
// pass first unless the image is more than 100 times as tall as it is wide and shrinks vertically (nh < h): such an
// image is resampled vertically first, an upsampling vertical pass still comes second.
//
// Launches: (1) the coefficient tables of every pass, one thread per output index; (2) the first pass of the images
// that need two, into the workspace; (3) per output pixel of the S x S square: the edge pad and the mirror as index
// arithmetic, the last pass (or the copy), and the normalisation.  The last pass is recomputed for the padded rows or
// columns (they repeat an edge of the resized image), which is cheaper than a third pass over memory.
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"

namespace gg {
namespace {

constexpr int kThreads = 256;
constexpr int kPrecisionBits = 22;   // Pillow's PRECISION_BITS for 8-bit images: 32 - 8 - 2

// Pillow's sinc_filter / lanczos_filter (support 3).
__device__ __forceinline__ double sinc(double x) {
  if (x == 0.0) return 1.0;
  x = __dmul_rn(x, 3.14159265358979323846);
  return __ddiv_rn(sin(x), x);
}

__device__ __forceinline__ double lanczos(double x) {
  if (-3.0 <= x && x < 3.0) return __dmul_rn(sinc(x), sinc(__ddiv_rn(x, 3.0)));
  return 0.0;
}

__device__ __forceinline__ double tap_weight(int x, int xmin, double center, double ss) {
  return lanczos(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss));
}

// One output index of one pass: (first input index, count, ksize weights) as precompute_coeffs + normalize_coeffs_8bpc.
__global__ void __launch_bounds__(kThreads)
letterbox_coeffs_kernel(int* __restrict__ coef, const GGLetterboxImage* __restrict__ info) {
  const GGLetterboxImage im = info[blockIdx.y];
  const bool horizontal = blockIdx.z == 0;
  const int64_t base = horizontal ? im.coef_h : im.coef_v;
  const int in = horizontal ? im.w : im.h, out = horizontal ? im.nw : im.nh, ksize = horizontal ? im.ksize_h : im.ksize_v;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (base < 0 || i >= out) return;
  const double scale = __ddiv_rn(static_cast<double>(in), static_cast<double>(out));
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = __dmul_rn(3.0, filterscale);
  const double ss = __ddiv_rn(1.0, filterscale);
  const double center = __dmul_rn(__dadd_rn(static_cast<double>(i), 0.5), scale);
  int xmin = static_cast<int>(__dadd_rn(__dsub_rn(center, support), 0.5));
  if (xmin < 0) xmin = 0;
  int xmax = static_cast<int>(__dadd_rn(__dadd_rn(center, support), 0.5));
  if (xmax > in) xmax = in;
  xmax -= xmin;
  double ww = 0.0;
  for (int x = 0; x < xmax; ++x) ww = __dadd_rn(ww, tap_weight(x, xmin, center, ss));
  int* row = coef + base + static_cast<int64_t>(i) * (ksize + 2);
  row[0] = xmin;
  row[1] = xmax;
  for (int x = 0; x < xmax; ++x) {
    double k = tap_weight(x, xmin, center, ss);
    if (ww != 0.0) k = __ddiv_rn(k, ww);
    const double scaled = __dmul_rn(k, static_cast<double>(1 << kPrecisionBits));
    row[2 + x] = static_cast<int>(k < 0.0 ? __dadd_rn(-0.5, scaled) : __dadd_rn(0.5, scaled));
  }
}

__device__ __forceinline__ unsigned char clip8(int v) {
  if (v >= (255 << kPrecisionBits)) return 255;
  if (v <= 0) return 0;
  return static_cast<unsigned char>(v >> kPrecisionBits);
}

// One resampled RGB pixel: count taps from p (3 bytes each, `step` bytes apart) with the fixed-point weights w.
__device__ __forceinline__ void resample_pixel(const unsigned char* __restrict__ p, int64_t step,
                                               const int* __restrict__ w, int count, unsigned char v[3]) {
  int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
  for (int k = 0; k < count; ++k) {
    const int c = __ldg(w + k);
    s0 += static_cast<int>(__ldg(p)) * c;
    s1 += static_cast<int>(__ldg(p + 1)) * c;
    s2 += static_cast<int>(__ldg(p + 2)) * c;
    p += step;
  }
  v[0] = clip8(s0);
  v[1] = clip8(s1);
  v[2] = clip8(s2);
}

// First pass of the images that need two: horizontal (h x nw) or vertical (nh x w) into the workspace.
__global__ void __launch_bounds__(kThreads)
letterbox_first_pass_kernel(unsigned char* __restrict__ ws, const int* __restrict__ coef,
                            const unsigned char* __restrict__ images, const GGLetterboxImage* __restrict__ info) {
  const GGLetterboxImage im = info[blockIdx.y];
  if (im.order < 3) return;
  const bool horizontal = im.order == 3;
  const int tw = horizontal ? im.nw : im.w;
  const int64_t total = static_cast<int64_t>(horizontal ? im.h : im.nh) * tw;
  const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int y = static_cast<int>(idx / tw), x = static_cast<int>(idx % tw);
  const unsigned char* src = images + im.offset;
  const int* row;
  const unsigned char* p;
  int64_t step;
  if (horizontal) {
    row = coef + im.coef_h + static_cast<int64_t>(x) * (im.ksize_h + 2);
    p = src + (static_cast<int64_t>(y) * im.w + __ldg(row)) * 3;
    step = 3;
  } else {
    row = coef + im.coef_v + static_cast<int64_t>(y) * (im.ksize_v + 2);
    p = src + (static_cast<int64_t>(__ldg(row)) * im.w + x) * 3;
    step = static_cast<int64_t>(im.w) * 3;
  }
  unsigned char v[3];
  resample_pixel(p, step, row + 2, __ldg(row + 1), v);
  unsigned char* o = ws + im.tmp_offset + idx * 3;
  o[0] = v[0];
  o[1] = v[1];
  o[2] = v[2];
}

// One output pixel (3 planes) of image blockIdx.y: mirror, edge pad, last pass or copy, normalisation.
__global__ void __launch_bounds__(kThreads)
letterbox_output_kernel(float* __restrict__ out, const unsigned char* __restrict__ ws, const int* __restrict__ coef,
                        const unsigned char* __restrict__ images, const GGLetterboxImage* __restrict__ info,
                        const unsigned char* __restrict__ flip, int S) {
  const int64_t plane = static_cast<int64_t>(S) * S;
  const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= plane) return;
  const int n = blockIdx.y;
  const GGLetterboxImage im = info[n];
  const int oy = static_cast<int>(idx / S), ox = static_cast<int>(idx % S);
  int ry = oy, rx = (flip != nullptr && __ldg(flip + n) != 0) ? S - 1 - ox : ox;
  if (im.h <= im.w) {   // border_pad pads the rows of a landscape (or square) image, the columns otherwise
    ry = min(max(ry - (S - im.nh) / 2, 0), im.nh - 1);
  } else {
    rx = min(max(rx - (S - im.nw) / 2, 0), im.nw - 1);
  }
  const unsigned char* src = images + im.offset;
  const unsigned char* tmp = ws + im.tmp_offset;
  unsigned char v[3];
  const int* row;
  switch (im.order) {
    case 0: {
      const unsigned char* p = src + (static_cast<int64_t>(ry) * im.w + rx) * 3;
      v[0] = __ldg(p);
      v[1] = __ldg(p + 1);
      v[2] = __ldg(p + 2);
      break;
    }
    case 1:   // horizontal only, from the image
      row = coef + im.coef_h + static_cast<int64_t>(rx) * (im.ksize_h + 2);
      resample_pixel(src + (static_cast<int64_t>(ry) * im.w + __ldg(row)) * 3, 3, row + 2, __ldg(row + 1), v);
      break;
    case 2:   // vertical only, from the image
      row = coef + im.coef_v + static_cast<int64_t>(ry) * (im.ksize_v + 2);
      resample_pixel(src + (static_cast<int64_t>(__ldg(row)) * im.w + rx) * 3, static_cast<int64_t>(im.w) * 3, row + 2,
                     __ldg(row + 1), v);
      break;
    case 3:   // vertical, from the (h, nw) intermediate
      row = coef + im.coef_v + static_cast<int64_t>(ry) * (im.ksize_v + 2);
      resample_pixel(tmp + (static_cast<int64_t>(__ldg(row)) * im.nw + rx) * 3, static_cast<int64_t>(im.nw) * 3, row + 2,
                     __ldg(row + 1), v);
      break;
    default:  // horizontal, from the (nh, w) intermediate
      row = coef + im.coef_h + static_cast<int64_t>(rx) * (im.ksize_h + 2);
      resample_pixel(tmp + (static_cast<int64_t>(ry) * im.w + __ldg(row)) * 3, 3, row + 2, __ldg(row + 1), v);
      break;
  }
  float* o = out + static_cast<int64_t>(n) * 3 * plane + idx;
#pragma unroll
  for (int c = 0; c < 3; ++c)   // torch.from_numpy(x).float().div_(255.0).add_(-0.5).mul_(2.0)
    o[c * plane] = __fmul_rn(__fadd_rn(__fdiv_rn(static_cast<float>(v[c]), 255.f), -0.5f), 2.f);
}

// Pillow's ksize for `in` -> `out`: (int)ceil(support) * 2 + 1 with support = 3 * max(in / out, 1).
int pillow_ksize(int in, int out) {
  double filterscale = static_cast<double>(in) / out;
  if (filterscale < 1.0) filterscale = 1.0;
  return static_cast<int>(std::ceil(3.0 * filterscale)) * 2 + 1;
}

// Derived fields of info[0..N) from (offset, h, w); returns the workspace bytes, or a negative GG_ERR_* code.
int64_t plan(GGLetterboxImage* info, int64_t N, int S, int resize, int64_t images_bytes) {
  if (N < 1 || N > 65535 || S < 1 || (resize != 0 && resize != 1) || images_bytes < 0)
    return fail(GG_ERR_BAD_ARG, "letterbox: 1 <= N <= 65535, S >= 1, resize 0 or 1, images_bytes >= 0");
  if (static_cast<int64_t>(S) * S > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "letterbox: S * S exceeds 2^31");
  int64_t n_coef = 0, n_tmp = 0;
  for (int64_t n = 0; n < N; ++n) {
    GGLetterboxImage& im = info[n];
    const int64_t h = im.h, w = im.w;
    if (h < 1 || w < 1 || im.offset < 0 || im.offset > images_bytes || h * w * 3 > images_bytes - im.offset)
      return fail(GG_ERR_BAD_ARG, "letterbox: image %lld (%lld x %lld at byte %lld) is empty or outside the %lld-byte buffer",
                  static_cast<long long>(n), static_cast<long long>(h), static_cast<long long>(w),
                  static_cast<long long>(im.offset), static_cast<long long>(images_bytes));
    int64_t nh = h, nw = w;
    if (resize) {   // border_pad: int(np.around(S * h / w)) -- Python's true division, rounded half to even
      if (h <= w) {
        nw = S;
        nh = static_cast<int64_t>(std::nearbyint(static_cast<double>(S * h) / static_cast<double>(w)));
      } else {
        nh = S;
        nw = static_cast<int64_t>(std::nearbyint(static_cast<double>(S * w) / static_cast<double>(h)));
      }
      if (nh < 1 || nw < 1)
        return fail(GG_ERR_BAD_ARG, "letterbox: image %lld (%lld x %lld) resizes to an empty image at S = %d",
                    static_cast<long long>(n), static_cast<long long>(h), static_cast<long long>(w), S);
    } else if (std::max(h, w) != S) {
      return fail(GG_ERR_BAD_ARG, "letterbox: without resize S must equal max(h, w) (image %lld is %lld x %lld, S = %d)",
                  static_cast<long long>(n), static_cast<long long>(h), static_cast<long long>(w), S);
    }
    const bool need_h = nw != w, need_v = nh != h;
    im.nh = static_cast<int32_t>(nh);
    im.nw = static_cast<int32_t>(nw);
    im.order = need_h && need_v ? (h > 100 * w && nh < h ? 4 : 3) : need_h ? 1 : need_v ? 2 : 0;
    im.ksize_h = need_h ? pillow_ksize(static_cast<int>(w), static_cast<int>(nw)) : 0;
    im.ksize_v = need_v ? pillow_ksize(static_cast<int>(h), static_cast<int>(nh)) : 0;
    im.reserved = 0;
    im.coef_h = need_h ? n_coef : -1;
    n_coef += need_h ? nw * (im.ksize_h + 2) : 0;
    im.coef_v = need_v ? n_coef : -1;
    n_coef += need_v ? nh * (im.ksize_v + 2) : 0;
    im.tmp_offset = im.order >= 3 ? n_tmp : -1;
    n_tmp += im.order == 3 ? h * nw * 3 : im.order == 4 ? nh * w * 3 : 0;
    n_tmp = (n_tmp + 15) & ~int64_t(15);
  }
  const int64_t coef_bytes = (n_coef * 4 + 15) & ~int64_t(15);
  for (int64_t n = 0; n < N; ++n)
    if (info[n].tmp_offset >= 0) info[n].tmp_offset += coef_bytes;
  return coef_bytes + n_tmp;
}

inline unsigned blocks_for(int64_t total) { return static_cast<unsigned>((total + kThreads - 1) / kThreads); }

}  // namespace
}  // namespace gg

using namespace gg;

extern "C" {

int gg_letterbox_plan(GGLetterboxImage* info_host, int64_t N, int S, int resize, int64_t images_bytes,
                      int64_t* workspace_bytes_host) {
  if (!info_host || !workspace_bytes_host) return fail(GG_ERR_BAD_ARG, "letterbox_plan: null info or workspace size");
  const int64_t ws = plan(info_host, N, S, resize, images_bytes);
  if (ws < 0) return static_cast<int>(ws);
  *workspace_bytes_host = ws;
  return GG_OK;
}

int gg_letterbox(float* out, void* workspace, int64_t workspace_bytes, const unsigned char* images, int64_t images_bytes,
                 const GGLetterboxImage* info_host, const GGLetterboxImage* info, const unsigned char* flip, int64_t N,
                 int S, int resize, void* stream) {
  if (!out || !images || !info_host || !info) return fail(GG_ERR_BAD_ARG, "letterbox: null output, images or info");
  if (!aligned8(info)) return fail(GG_ERR_BAD_ARG, "letterbox: info must be 8-byte aligned");
  if (N < 1 || N > 65535) return fail(GG_ERR_BAD_ARG, "letterbox: 1 <= N <= 65535");
  std::vector<GGLetterboxImage> want(info_host, info_host + N);
  const int64_t ws_bytes = plan(want.data(), N, S, resize, images_bytes);
  if (ws_bytes < 0) return static_cast<int>(ws_bytes);
  if (std::memcmp(want.data(), info_host, sizeof(GGLetterboxImage) * N) != 0)
    return fail(GG_ERR_BAD_ARG, "letterbox: info differs from gg_letterbox_plan's");
  if (workspace_bytes < ws_bytes)
    return fail(GG_ERR_BAD_ARG, "letterbox: the workspace needs %lld bytes (got %lld)", static_cast<long long>(ws_bytes),
                static_cast<long long>(workspace_bytes));
  if (ws_bytes > 0 && (!workspace || !aligned16(workspace)))
    return fail(GG_ERR_BAD_ARG, "letterbox: the workspace must be non-null and 16-byte aligned");
  int max_out = 0;
  int64_t max_tmp = 0;
  for (const GGLetterboxImage& im : want) {
    max_out = std::max(max_out, std::max(im.ksize_h ? im.nw : 0, im.ksize_v ? im.nh : 0));
    if (im.order == 3) max_tmp = std::max(max_tmp, static_cast<int64_t>(im.h) * im.nw);
    if (im.order == 4) max_tmp = std::max(max_tmp, static_cast<int64_t>(im.nh) * im.w);
  }
  auto st = static_cast<cudaStream_t>(stream);
  auto* coef = static_cast<int*>(workspace);
  auto* ws = static_cast<unsigned char*>(workspace);
  if (max_out > 0) {
    letterbox_coeffs_kernel<<<dim3(blocks_for(max_out), static_cast<unsigned>(N), 2), kThreads, 0, st>>>(coef, info);
    GG_CHECK_LAUNCH("letterbox coefficients launch");
  }
  if (max_tmp > 0) {
    letterbox_first_pass_kernel<<<dim3(blocks_for(max_tmp), static_cast<unsigned>(N)), kThreads, 0, st>>>(ws, coef, images,
                                                                                                          info);
    GG_CHECK_LAUNCH("letterbox first pass launch");
  }
  letterbox_output_kernel<<<dim3(blocks_for(static_cast<int64_t>(S) * S), static_cast<unsigned>(N)), kThreads, 0, st>>>(
      out, ws, coef, images, info, flip, S);
  GG_CHECK_LAUNCH("letterbox output launch");
  return GG_OK;
}

}  // extern "C"
