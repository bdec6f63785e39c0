// grid.cuh -- torchvision make_grid's layout and the images2grid quantisation, shared by the uint8 grid writers
// (splat.cu: gg_splat_composite_grid; trainvis.cu: gg_image_grid, gg_flow_image_grid).
//
// make_grid(nrow, padding, pad_value=0): xmaps = min(nrow, N) images per row, ymaps = ceil(N / xmaps) rows, each cell
// (H + pad) x (W + pad) with `pad` rows / columns of padding before it and after the last; a single image is returned as
// it is (no padding).  Padding and the cells past the last image hold 0, which images2grid maps to 0.
#pragma once

#include <cstdint>

namespace gg {

struct GridLayout {
  int64_t n;                 // images
  int h, w;                  // image size
  int xmaps, pad, hg, wg;    // images per row, padding, grid size
};

// The layout of N images of h x w.  -> false when one grid exceeds 2^31 bytes (HWC uint8).
inline bool make_grid_layout(GridLayout& g, int64_t n, int h, int w, int nrow, int padding) {
  g.n = n; g.h = h; g.w = w;
  g.xmaps = static_cast<int>(n < nrow ? n : nrow);
  const int64_t ymaps = (n + g.xmaps - 1) / g.xmaps;
  g.pad = n == 1 ? 0 : padding;                      // make_grid returns a single image as it is
  const int64_t hg = ymaps * (h + g.pad) + g.pad, wg = static_cast<int64_t>(g.xmaps) * (w + g.pad) + g.pad;
  if (hg * wg * 3 > 0x7fffffffLL) return false;
  g.hg = static_cast<int>(hg); g.wg = static_cast<int>(wg);
  return true;
}

// Grid pixel (gx, gy) -> the image it shows (y, x within it), or -1 for padding and empty cells.
__device__ __forceinline__ int64_t grid_source(const GridLayout& g, int gx, int gy, int& y, int& x) {
  const int yy = gy - g.pad, xx = gx - g.pad;
  if (yy < 0 || xx < 0) return -1;
  const int ch = g.h + g.pad, cw = g.w + g.pad;
  y = yy % ch;
  x = xx % cw;
  const int64_t k = static_cast<int64_t>(yy / ch) * g.xmaps + xx / cw;
  if (y >= g.h || x >= g.w || k >= g.n) return -1;
  return k;
}

// make_grid's normalize with range (lo, hi) -- clamp(lo, hi), sub(lo), div(max(hi - lo, 1e-5)) -- then images2grid's
// mul(255), add(0.5), clamp(0, 255) and truncating uint8 cast, each rounded on its own.  hi - lo is formed in double by
// make_grid and rounded once to float: for float lo and hi that is the correctly rounded float difference.  The division
// is the correctly rounded quotient, as make_grid computes it on CPU tensors.  On CUDA tensors torch's result was seen to
// differ from both the quotient and the product with the float reciprocal at some values chosen next to quantisation
// steps, so a per-image range (not (-1, 1) or (0, 1), whose divisors are exact) may differ from it there by one step.
__device__ __forceinline__ unsigned char quantise_range(float v, float lo, float hi) {
  v = fminf(fmaxf(v, lo), hi);
  v = __fdiv_rn(__fsub_rn(v, lo), fmaxf(__fsub_rn(hi, lo), 1e-5f));
  v = __fadd_rn(__fmul_rn(v, 255.f), 0.5f);
  v = fminf(fmaxf(v, 0.f), 255.f);
  return static_cast<unsigned char>(static_cast<int>(v));
}

}  // namespace gg
