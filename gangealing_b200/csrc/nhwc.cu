// nhwc.cu -- channels-last (N, H, W, C) variants of the StyledConv tail family (sm_90a).
//
// Why: cuDNN's tensor-core convolution kernels are NHWC-native; with NCHW activations every convolution of the step
// is bracketed by nchwToNhwc / nhwcToNchw conversion kernels.
// Keeping the generator's activations channels-last end to end removes them -- provided the hand-written kernels
// between the convolutions speak NHWC too.  In this layout a pixel's channels are contiguous, so with C % 4 == 0
// EVERYTHING is 16-byte aligned: the blur can use a real 4-D TMA tensor map (cp.async.bulk.tensor, SASS UTMALDG)
// whose out-of-bounds zero fill implements the padding of upfirdn2d for free.
//
// Every kernel is templated on the STORAGE type T (fp32, or bf16 for BASELINE config 3: bf16 activations, fp32
// arithmetic); an activation is always moved 16 bytes at a time (V = 4 fp32 / 8 bf16 channels, ChanVec<T>).
//
// Same math / reference citations as the NCHW kernels (bias_act.cu, upfirdn2d.cu):
//   gg_noise_bias_act_nhwc       lrelu(rs[n,c]*x + nw*noise[n,p] + b[c])*gain                networks.py:291-298,346-348
//   gg_bias_act_backward_nhwc    gx = (out>0 ? g : a*g)*gain ; grad_bias[c] = sum gx          op/fused_act.py:20-38
//   gg_channel_scale_nhwc        x*s[n,c] (+ row_dot[n,c] = sum_p x*y)                        networks.py:236,243
//   gg_blur_nhwc                 upfirdn2d(up=down=1, <=4x4 separable or not) [+ fused tail]   networks.py:266 (+346-348)
#include <cuda.h>

#include "common.cuh"
#include "nhwc_reduce.cuh"

namespace gg {
namespace {

constexpr int kT = 256;

// ------------------------------------------------------------------------------------------------ elementwise
template <typename T>
__global__ void __launch_bounds__(kT)
noise_bias_act_nhwc_kernel(T* __restrict__ out, const T* __restrict__ x, const float* __restrict__ noise,
                           const float* __restrict__ noise_weight, const float* __restrict__ bias,
                           const float* __restrict__ row_scale, float alpha, float gain, int64_t n_vec, int cv,
                           int64_t hw) {
  constexpr int V = ChanVec<T>::V;
  const float nw = noise ? (noise_weight ? __ldg(noise_weight) : 1.f) : 0.f;
  const int64_t base = (static_cast<int64_t>(blockIdx.x) * 4) * kT + threadIdx.x;
  uint4 xv[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int64_t v = base + static_cast<int64_t>(u) * kT;
    if (v < n_vec) xv[u] = ldg_stream16(x + v * V);
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int64_t v = base + static_cast<int64_t>(u) * kT;
    if (v < n_vec) {
      // index arithmetic in 32 bits whenever the tensor allows it (a 64-bit division costs ~80 instructions: with two of
      // them per vector this streaming kernel was ISSUE-bound in bf16, 83 % issue utilisation at 80 % of the HBM peak);
      // the sample index is only needed for the per-(sample, channel) row scale
      int64_t pix, n = 0;
      int cq;
      if (n_vec <= 0xffffffffLL) {
        const unsigned v32 = static_cast<unsigned>(v), p32 = v32 / static_cast<unsigned>(cv);
        cq = static_cast<int>(v32 - p32 * static_cast<unsigned>(cv));
        pix = p32;
        if (row_scale) n = p32 / static_cast<unsigned>(hw);
      } else {
        pix = v / cv;
        cq = static_cast<int>(v - pix * cv);
        if (row_scale) n = pix / hw;
      }
      const float nz = noise ? nw * __ldg(noise + pix) : 0.f;
      float xf[V], o[V];
      ChanVec<T>::unpack(xv[u], xf);
#pragma unroll
      for (int q = 0; q < V / 4; ++q) {
        const float4 b = bias ? __ldg(reinterpret_cast<const float4*>(bias) + cq * (V / 4) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float4 r = row_scale ? __ldg(reinterpret_cast<const float4*>(row_scale + n * cv * V) + cq * (V / 4) + q)
                                   : make_float4(1.f, 1.f, 1.f, 1.f);
        const float bb[4] = {b.x, b.y, b.z, b.w}, rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float t = fmaf(xf[4 * q + k], rr[k], bb[k]) + nz;
          o[4 * q + k] = (t > 0.f ? t : t * alpha) * gain;
        }
      }
      stg_stream16(out + v * V, ChanVec<T>::pack(o));
    }
  }
}

// One CTA = `chunk` consecutive pixels of one sample x all channels.  Thread = (channel vector, pixel lane); per-channel
// sums are reduced across the CTA's pixel lanes in shared memory and written as one partial row per CTA.
// MODE 0: channel_scale (out = x*s, dot = sum x*y)   MODE 1: bias_act backward (out = act'(ref)*x*gain, dot = sum out)
template <typename T, int MODE>
__global__ void __launch_bounds__(kT)
rowwise_nhwc_kernel(T* __restrict__ out, float* __restrict__ partial, const T* __restrict__ x,
                    const T* __restrict__ y, const float* __restrict__ s, float alpha, float gain, int cv,
                    int64_t hw, int chunk, int chunks_per_sample) {
  constexpr int V = ChanVec<T>::V;
  extern __shared__ float red[];                       // [pixel lanes][C] partial sums
  const int64_t n = blockIdx.x / chunks_per_sample;
  const int ck = blockIdx.x - n * chunks_per_sample;
  const int64_t p0 = static_cast<int64_t>(ck) * chunk, p1 = min(p0 + chunk, hw);
  const int lanes_p = kT / cv > 0 ? kT / cv : 1;       // pixel lanes when C/V <= 256
  float acc[V];
#pragma unroll
  for (int k = 0; k < V; ++k) acc[k] = 0.f;
  const int cq = threadIdx.x % cv;
  const int pl = threadIdx.x / cv;
  if (pl < lanes_p) {
    float sv[V];
#pragma unroll
    for (int k = 0; k < V; ++k) sv[k] = (MODE == 0) ? __ldg(s + n * cv * V + cq * V + k) : 1.f;
    const bool has_y = (MODE == 1) || y != nullptr;
    auto body = [&](const uint4 xr, const uint4 yr, int64_t off) {
      float xf[V], yf[V], o[V];
      ChanVec<T>::unpack(xr, xf);
      ChanVec<T>::unpack(yr, yf);
#pragma unroll
      for (int k = 0; k < V; ++k) {
        if (MODE == 0) {
          o[k] = xf[k] * sv[k];
          if (has_y) acc[k] = fmaf(xf[k], yf[k], acc[k]);
        } else {                                 // y = saved forward output
          o[k] = (yf[k] > 0.f ? xf[k] : xf[k] * alpha) * gain;
          acc[k] += o[k];
        }
      }
      *reinterpret_cast<uint4*>(out + off) = ChanVec<T>::pack(o);
    };
    const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
    int64_t p = p0 + pl;
    // 4 pixels per trip: all loads issued before the first dependent store (memory-level parallelism)
    for (; p + 3 * lanes_p < p1; p += 4 * lanes_p) {
      uint4 xv[4], yv[4];
      int64_t off[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        off[u] = ((n * hw + p + u * lanes_p) * cv + cq) * V;
        xv[u] = ldg_stream16(x + off[u]);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) yv[u] = has_y ? ldg_stream16(y + off[u]) : zero;
#pragma unroll
      for (int u = 0; u < 4; ++u) body(xv[u], yv[u], off[u]);
    }
    for (; p < p1; p += lanes_p) {
      const int64_t off = ((n * hw + p) * cv + cq) * V;
      const uint4 xv = ldg_stream16(x + off);
      const uint4 yv = has_y ? ldg_stream16(y + off) : zero;
      body(xv, yv, off);
    }
  }
  if (partial) {
    const int C = cv * V;
    if (pl < lanes_p) {
#pragma unroll
      for (int q = 0; q < V / 4; ++q)
        reinterpret_cast<float4*>(red + pl * C + cq * V)[q] = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += kT) {
      float t = 0.f;
      for (int l = 0; l < lanes_p; ++l) t += red[l * C + c];
      partial[static_cast<int64_t>(blockIdx.x) * C + c] = t;
    }
  }
}

// ------------------------------------------------------------------------------------------------ to-RGB (1x1, 3 outputs)
// out[n,o,p] = sum_i wm[n,o,i] * x[n,p,i] + bias[o] + skip[n,o,p]   x: NHWC, out/skip: planar (N, 3, HW)
// One pass over x (the only large operand).  A group of 8 lanes owns 4 consecutive pixels: every lane streams its
// channel quads (l + 8j) of the 4 pixels (4 independent 128-bit loads per trip), the 3 x C modulated filter sits in
// shared memory, and the 12 partial dot products are combined with 3 butterfly steps.
__global__ void __launch_bounds__(kT)
to_rgb_nhwc_fwd_kernel(float* __restrict__ out, const float* __restrict__ x, const float* __restrict__ wm,
                       const float* __restrict__ bias, const float* __restrict__ skip, int c4, int64_t hw, int chunk,
                       int chunks_per_sample) {
  extern __shared__ __align__(16) float wsm[];          // [3][C]
  const int64_t n = blockIdx.x / chunks_per_sample;
  const int ck = blockIdx.x - n * chunks_per_sample;
  const int64_t p0 = static_cast<int64_t>(ck) * chunk, p1 = min(p0 + chunk, hw);
  {
    const float4* src = reinterpret_cast<const float4*>(wm + n * 3 * c4 * 4);
    float4* dst = reinterpret_cast<float4*>(wsm);
    for (int i = threadIdx.x; i < 3 * c4; i += kT) dst[i] = __ldg(src + i);
  }
  __syncthreads();
  const float4* w4 = reinterpret_cast<const float4*>(wsm);
  const int l = threadIdx.x & 7, grp = threadIdx.x >> 3;
  const bool vec_ok = (hw & 3) == 0;
  const unsigned gmask = 0xffu << (threadIdx.x & 24);     // groups of one warp may leave the loop at different trips
  for (int64_t pb = p0 + grp * 4; pb < p1; pb += (kT / 8) * 4) {
    float acc[4][3];
#pragma unroll
    for (int u = 0; u < 4; ++u) acc[u][0] = acc[u][1] = acc[u][2] = 0.f;
    const float4* xp[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int64_t pu = min(pb + u, p1 - 1);             // clamped: a tail pixel is recomputed, never stored
      xp[u] = reinterpret_cast<const float4*>(x + (n * hw + pu) * c4 * 4);
    }
    for (int q = l; q < c4; q += 8) {
      float4 xv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) xv[u] = __ldcs(xp[u] + q);
      const float4 w0 = w4[q], w1 = w4[c4 + q], w2 = w4[2 * c4 + q];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        acc[u][0] = fmaf(xv[u].x, w0.x, fmaf(xv[u].y, w0.y, fmaf(xv[u].z, w0.z, fmaf(xv[u].w, w0.w, acc[u][0]))));
        acc[u][1] = fmaf(xv[u].x, w1.x, fmaf(xv[u].y, w1.y, fmaf(xv[u].z, w1.z, fmaf(xv[u].w, w1.w, acc[u][1]))));
        acc[u][2] = fmaf(xv[u].x, w2.x, fmaf(xv[u].y, w2.y, fmaf(xv[u].z, w2.z, fmaf(xv[u].w, w2.w, acc[u][2]))));
      }
    }
#pragma unroll
    for (int m = 4; m >= 1; m >>= 1)
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int o = 0; o < 3; ++o) acc[u][o] += __shfl_xor_sync(gmask, acc[u][o], m);
    if (l < 3) {                                           // lane o of the group stores output plane o
      const int o = l;
      float r[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) r[u] = (o == 0 ? acc[u][0] : o == 1 ? acc[u][1] : acc[u][2]) + (bias ? __ldg(bias + o) : 0.f);
      const int64_t off = (n * 3 + o) * hw + pb;
      if (vec_ok && pb + 3 < p1) {
        if (skip) {
          const float4 sk = __ldg(reinterpret_cast<const float4*>(skip + off));
          r[0] += sk.x; r[1] += sk.y; r[2] += sk.z; r[3] += sk.w;
        }
        *reinterpret_cast<float4*>(out + off) = make_float4(r[0], r[1], r[2], r[3]);
      } else {
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (pb + u < p1) out[off + u] = r[u] + (skip ? __ldg(skip + off + u) : 0.f);
      }
    }
  }
}

// Backward: gx[n,p,i] = sum_o wm[n,o,i] g[n,o,p]  and  gwm[n,o,i] = sum_p g[n,o,p] x[n,p,i], one pass over x / gx.
// Thread = (channel quad, pixel lane) as in rowwise_nhwc_kernel; the three g planes are warp-broadcast loads.
__global__ void __launch_bounds__(kT)
to_rgb_nhwc_bwd_kernel(float* __restrict__ gx, float* __restrict__ partial, const float* __restrict__ g,
                       const float* __restrict__ x, const float* __restrict__ wm, int c4, int64_t hw, int chunk,
                       int chunks_per_sample) {
  extern __shared__ float red[];                          // [pixel lanes][3][C]
  const int64_t n = blockIdx.x / chunks_per_sample;
  const int ck = blockIdx.x - n * chunks_per_sample;
  const int64_t p0 = static_cast<int64_t>(ck) * chunk, p1 = min(p0 + chunk, hw);
  const int lanes_p = kT / c4 > 0 ? kT / c4 : 1;
  const int cq = threadIdx.x % c4, pl = threadIdx.x / c4;
  float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, a2 = a0;
  if (pl < lanes_p) {
    const float4* wp = reinterpret_cast<const float4*>(wm + n * 3 * c4 * 4);
    const float4 w0 = __ldg(wp + cq), w1 = __ldg(wp + c4 + cq), w2 = __ldg(wp + 2 * c4 + cq);
    const float* g0 = g + n * 3 * hw;
    auto body = [&](int64_t p, const float4 xv, float s0, float s1, float s2) {
      float4 o;
      o.x = fmaf(w2.x, s2, fmaf(w1.x, s1, w0.x * s0)); o.y = fmaf(w2.y, s2, fmaf(w1.y, s1, w0.y * s0));
      o.z = fmaf(w2.z, s2, fmaf(w1.z, s1, w0.z * s0)); o.w = fmaf(w2.w, s2, fmaf(w1.w, s1, w0.w * s0));
      if (gx) *reinterpret_cast<float4*>(gx + ((n * hw + p) * c4 + cq) * 4) = o;
      a0.x = fmaf(s0, xv.x, a0.x); a0.y = fmaf(s0, xv.y, a0.y); a0.z = fmaf(s0, xv.z, a0.z); a0.w = fmaf(s0, xv.w, a0.w);
      a1.x = fmaf(s1, xv.x, a1.x); a1.y = fmaf(s1, xv.y, a1.y); a1.z = fmaf(s1, xv.z, a1.z); a1.w = fmaf(s1, xv.w, a1.w);
      a2.x = fmaf(s2, xv.x, a2.x); a2.y = fmaf(s2, xv.y, a2.y); a2.z = fmaf(s2, xv.z, a2.z); a2.w = fmaf(s2, xv.w, a2.w);
    };
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    int64_t p = p0 + pl;
    for (; p + 3 * lanes_p < p1; p += 4 * lanes_p) {
      float4 xv[4];
      float s[4][3];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t pu = p + u * lanes_p;
        xv[u] = partial ? __ldcs(reinterpret_cast<const float4*>(x + ((n * hw + pu) * c4 + cq) * 4)) : zero;
        s[u][0] = __ldg(g0 + pu); s[u][1] = __ldg(g0 + hw + pu); s[u][2] = __ldg(g0 + 2 * hw + pu);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) body(p + u * lanes_p, xv[u], s[u][0], s[u][1], s[u][2]);
    }
    for (; p < p1; p += lanes_p) {
      const float4 xv = partial ? __ldcs(reinterpret_cast<const float4*>(x + ((n * hw + p) * c4 + cq) * 4)) : zero;
      body(p, xv, __ldg(g0 + p), __ldg(g0 + hw + p), __ldg(g0 + 2 * hw + p));
    }
  }
  if (partial) {
    float4* r4 = reinterpret_cast<float4*>(red);
    if (pl < lanes_p) {
      r4[(pl * 3 + 0) * c4 + cq] = a0; r4[(pl * 3 + 1) * c4 + cq] = a1; r4[(pl * 3 + 2) * c4 + cq] = a2;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 3 * c4; i += kT) {
      float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int q = 0; q < lanes_p; ++q) {
        const float4 v = r4[q * 3 * c4 + i];
        t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
      }
      reinterpret_cast<float4*>(partial + static_cast<int64_t>(blockIdx.x) * 3 * c4 * 4)[i] = t;
    }
  }
}

// ------------------------------------------------------------------------------------------------ blur (TMA tiled)
// Tile geometry per storage type: a thread always owns 16 bytes of channels (V = 4 fp32 / 8 bf16) so that a pixel of the
// tile is 128 bytes (8 threads, conflict-free LDS.128); it owns COLS adjacent output columns (2 for fp32, 1 for bf16:
// the register window is 4 rows x COLS x V floats either way).
template <typename T> struct BlurGeom {
  static constexpr int V = ChanVec<T>::V;
  static constexpr int CB = 8 * V;                 // channels per CTA (128 B per pixel in the tile)
  static constexpr int COLS = (V == 4) ? 2 : 1;    // output columns per thread
  static constexpr int BX = 32 * COLS;             // output columns per CTA
  static constexpr int TW = BX + 3;                // tile width (3 halo columns)
  static constexpr int STAGE_ELEMS = 4 * TW * CB;  // kRY = 4 rows per stage
};
constexpr int kRY = 4;      // input rows per pipeline stage
constexpr int kNS = 3;      // stages

struct BlurNhwcParams {
  int n, c, in_h, in_w, out_h, out_w;
  int pad_x0, pad_y0;
  int seg_rows;             // output rows per CTA (grid.y segments)
  int act;                  // FUSED: 1 linear, 3 lrelu
  float alpha, gain;
};

__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* tmap, int c0, int x0, int y0, int n0,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
      ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(c0), "r"(x0), "r"(y0), "r"(n0), "r"(smem_u32(bar))
      : "memory");
}

// CTA = (sample n, BX-column block, CB-channel chunk, row segment).  Input rows stream through a 3-stage ring of
// {CB ch x TW px x 4 rows} TMA boxes (zero-filled outside the image = upfirdn2d's padding); each thread slides a
// 4-row window of horizontal results for its COLS columns x V channels down the whole segment, so a row is read from
// shared memory once and from HBM once (+3 halo rows per segment, +3/BX halo columns).
//   MODE 0  plain blur                                                  out = B(in)
//   MODE 1  fused StyledConv tail: o = lrelu(rs*B(in) + nw*noise + b)*gain; writes `out` = o and/or `out2` = o*scale2[n,c]
//           (the NEXT modulated convolution's input: its style modulation rides in this epilogue, networks.py:236,243)
//   MODE 2  adjoint epilogue (backward of MODE 1's blur): t = B(in); `out` = t*rs[n,c]; partial[cta][c] = sum t*mul[n,y,x,c]
//           (the gradient of the demodulation coefficients, <B^T g, raw>, reduced inside the pass that produces B^T g)
//   FAST    (MODE 1) the gain-folded epilogue `max(T, T*slope)` is valid for the launch (gain > 0, 0 <= slope <= 1 or linear):
//           a compile-time variant -- as a run-time flag the compiler predicated BOTH epilogues into the row loop (FSETP /
//           FSEL / FMUL of the general path: 16 % of the issue slots of the bf16 kernel, which is issue-bound)
//   MODE 3  MODE 1 whose `out` receives the sign mask of o (common.cuh), (N, H, W, C/32) uint32, instead of o: all that a
//           backward pass without reductions over o needs of it
template <typename T, int MODE, bool SEP, bool FAST = false>
__global__ void __launch_bounds__(kT, 2)
blur_nhwc_kernel(T* __restrict__ out, T* __restrict__ out2, const __grid_constant__ CUtensorMap tmap,
                 const float* __restrict__ filt, int kh, int kw, const float* __restrict__ noise,
                 const float* __restrict__ noise_weight, const float* __restrict__ bias,
                 const float* __restrict__ row_scale, const float* __restrict__ scale2, const T* __restrict__ mul,
                 float* __restrict__ partial, BlurNhwcParams p) {
  using G = BlurGeom<T>;
  constexpr int V = G::V, CB = G::CB, COLS = G::COLS, BX = G::BX, TW = G::TW;
  constexpr bool FUSED = MODE == 1 || MODE == 3;
  constexpr bool MASK = MODE == 3;
  extern __shared__ __align__(128) unsigned char tiles_raw[];
  T* tiles = reinterpret_cast<T*>(tiles_raw);
  __shared__ uint64_t full_bar[kNS];
  const int tid = threadIdx.x;
  const int cq = tid & 7;                 // channel vector within the CB-channel chunk
  const int xg = tid >> 3;                // 0..31 -> columns COLS*xg .. of the block
  const int chunks = p.c / CB;
  const int bx = blockIdx.x / chunks, cc = blockIdx.x - bx * chunks;
  const int n = blockIdx.z;
  const int oy0 = blockIdx.y * p.seg_rows;
  const int rows_out = min(p.seg_rows, p.out_h - oy0);
  const int x_out0 = bx * BX;             // first output column of the block
  const int c0 = cc * CB;
  // input row/col of tap (0,0) for output (oy0, x_out0)
  const int iy0 = oy0 - p.pad_y0, ix0 = x_out0 - p.pad_x0;
  const int rows_in = rows_out + 3;
  const int n_stage_iters = (rows_in + kRY - 1) / kRY;
  constexpr uint32_t kStageBytes = G::STAGE_ELEMS * sizeof(T);

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < kNS; ++s) mbar_init(&full_bar[s], 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < kNS - 1; ++s)
      if (s < n_stage_iters) {
        mbar_expect_tx(&full_bar[s], kStageBytes);
        tma_load_4d(tiles + s * G::STAGE_ELEMS, &tmap, c0, ix0, iy0 + s * kRY, n, &full_bar[s]);
      }
  }

  // taps (flipped: true convolution), rank-1 factorisation when possible
  float kf[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
      kf[a][b] = (a < kh && b < kw) ? __ldg(filt + (kh - 1 - a) * kw + (kw - 1 - b)) : 0.f;
  float ku[4], kv[4];
  {
    int a0 = 0, b0 = 0;
    float big = 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b)
        if (fabsf(kf[a][b]) > big) { big = fabsf(kf[a][b]); a0 = a; b0 = b; }
    float piv = 1.f;
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b)
        if (a == a0 && b == b0) piv = kf[a][b];
    const float inv = big > 0.f ? 1.f / piv : 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      float col = 0.f;
#pragma unroll
      for (int b = 0; b < 4; ++b) if (b == b0) col = kf[a][b];
      ku[a] = col * inv;
    }
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      float row = 0.f;
#pragma unroll
      for (int a = 0; a < 4; ++a) if (a == a0) row = kf[a][b];
      kv[b] = row;
    }
  }

  // per-thread channel constants (a thread keeps its V channels for the whole segment)
  float bq[V], rq[V], sq[V], dacc[V];
#pragma unroll
  for (int k = 0; k < V; ++k) { bq[k] = 0.f; rq[k] = 1.f; sq[k] = 1.f; dacc[k] = 0.f; }
  float nw = 0.f;
  const int64_t nc0 = static_cast<int64_t>(n) * p.c + c0 + cq * V;
  if (MODE != 0) {
    if (row_scale) {
#pragma unroll
      for (int k = 0; k < V; ++k) rq[k] = __ldg(row_scale + nc0 + k);
    }
  }
  if (FUSED) {
    if (bias) {
#pragma unroll
      for (int k = 0; k < V; ++k) bq[k] = __ldg(bias + c0 + cq * V + k);
    }
    if (scale2) {
#pragma unroll
      for (int k = 0; k < V; ++k) sq[k] = __ldg(scale2 + nc0 + k);
    }
    nw = noise ? (noise_weight ? __ldg(noise_weight) : 1.f) : 0.f;
  }
  // lrelu(t)*gain == max(T, T*slope) with T = gain*t when gain > 0 and 0 <= slope <= 1: the gain is folded into the
  // row scale, the bias and the noise weight, the row scale into the vertical taps (2 epilogue ops per output)
  constexpr bool fast = FUSED && FAST;    // the host checks gain > 0 && ((act == 3 && 0 <= alpha <= 1) || act == 1)
  const float neg = (p.act == 3) ? p.alpha : 1.f;
  if (fast) {
#pragma unroll
    for (int k = 0; k < V; ++k) { rq[k] *= p.gain; bq[k] *= p.gain; }
    nw *= p.gain;
  }
  const int xo = x_out0 + COLS * xg;      // first of this thread's output columns
  // element offset of this thread's first channel at output (n, oy0 + ro, xo): kept as a RUNNING 64-bit value (ro advances
  // by one per input row) -- recomputing ((n*H + oy)*W + x)*C + c per row and column cost ~30 integer instructions a row
  const int64_t row_stride = static_cast<int64_t>(p.out_w) * p.c;
  const int64_t obase = ((static_cast<int64_t>(n) * p.out_h + oy0) * p.out_w + xo) * p.c + c0 + cq * V;   // ro = 0
  int64_t ocur = obase - 3 * row_stride;                                                                  // ro = r_in - 3
  bool okc[COLS];
#pragma unroll
  for (int j = 0; j < COLS; ++j) okc[j] = xo + j < p.out_w;
  // noise of the rows a stage completes is fetched one stage ahead (its latency hides behind the previous stage)
  float nzn[kRY][COLS];
#pragma unroll
  for (int rr = 0; rr < kRY; ++rr)
#pragma unroll
    for (int j = 0; j < COLS; ++j) nzn[rr][j] = 0.f;
  const float* noise_base = noise ? noise + (static_cast<int64_t>(n) * p.out_h + oy0) * p.out_w + xo : nullptr;   // row ro = 0
  auto fetch_noise = [&](int it_) {
#pragma unroll
    for (int rr = 0; rr < kRY; ++rr) {
      const int ro = it_ * kRY + rr - 3;
#pragma unroll
      for (int j = 0; j < COLS; ++j) nzn[rr][j] = 0.f;
      if (ro >= 0 && ro < rows_out) {
        const float* np_ = noise_base + static_cast<int64_t>(ro) * p.out_w;
#pragma unroll
        for (int j = 0; j < COLS; ++j)
          if (okc[j]) nzn[rr][j] = __ldg(np_ + j);
      }
    }
  };
  if (FUSED && noise) fetch_noise(0);

  // MODE 2: the `mul` operand of the row an iteration completes is fetched one input row earlier (its HBM latency hides
  // behind that row's shared-memory reads and arithmetic)
  uint4 mcur[COLS], mnext[COLS];
#pragma unroll
  for (int j = 0; j < COLS; ++j) mcur[j] = mnext[j] = make_uint4(0u, 0u, 0u, 0u);
  auto fetch_mul = [&](int ro_) {
    if (ro_ >= 0 && ro_ < rows_out) {
      const int64_t mo = obase + ro_ * row_stride;
#pragma unroll
      for (int j = 0; j < COLS; ++j)
        if (okc[j]) mnext[j] = __ldg(reinterpret_cast<const uint4*>(mul + mo + static_cast<int64_t>(j) * p.c));
    }
  };
  if (MODE == 2 && mul) { fetch_mul(-3 + 3); }   // row 0 is completed by input row 3

  // window: sep -> horizontal results hwin[4 rows][COLS][V]; else raw inputs rwin[4 rows][COLS+3][V]
  float hwin[SEP ? 4 : 1][COLS][V];
  float rwin[SEP ? 1 : 4][COLS + 3][V];
  int r_in = 0;                            // input rows consumed so far (relative to iy0)
  for (int it = 0; it < n_stage_iters; ++it) {
    const int stage = it % kNS;
    if (tid == 0) {
      const int nxt = it + kNS - 1;
      if (nxt < n_stage_iters) {
        const int ns = nxt % kNS;
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_expect_tx(&full_bar[ns], kStageBytes);
        tma_load_4d(tiles + ns * G::STAGE_ELEMS, &tmap, c0, ix0, iy0 + nxt * kRY, n, &full_bar[ns]);
      }
    }
    float nzc[kRY][COLS];
#pragma unroll
    for (int rr = 0; rr < kRY; ++rr)
#pragma unroll
      for (int j = 0; j < COLS; ++j) nzc[rr][j] = nzn[rr][j];
    if (FUSED && noise && it + 1 < n_stage_iters) fetch_noise(it + 1);
    if (MODE == 2 && mul && it + 1 < n_stage_iters) {
      // pull the `mul` rows the NEXT stage completes into L2 now (no registers held): the one-row-ahead register fetch
      // below then only has to cover an L2 hit
#pragma unroll
      for (int rr = 0; rr < kRY; ++rr) {
        const int ro = (it + 1) * kRY + rr - 3;
        if (ro >= 0 && ro < rows_out) {
          const T* mp = mul + obase + ro * row_stride;
#pragma unroll
          for (int j = 0; j < COLS; ++j)
            if (okc[j]) asm volatile("prefetch.global.L2 [%0];" ::"l"(mp + static_cast<int64_t>(j) * p.c));
        }
      }
    }
    mbar_wait(&full_bar[stage], static_cast<uint32_t>((it / kNS) & 1));
    const T* st = tiles + stage * G::STAGE_ELEMS;
#pragma unroll
    for (int rr = 0; rr < kRY; ++rr, ++r_in, ocur += row_stride) {
      if (MODE == 2 && mul) {
#pragma unroll
        for (int j = 0; j < COLS; ++j) mcur[j] = mnext[j];
        fetch_mul(r_in - 3 + 1);           // the row the NEXT iteration completes
      }
      // COLS+3 input pixels (columns COLS*xg .. of the tile) x V channels of this thread
      const uint4* rowp = reinterpret_cast<const uint4*>(st + (rr * TW + COLS * xg) * CB) + cq;
      float q[COLS + 3][V];
#pragma unroll
      for (int i = 0; i < COLS + 3; ++i) ChanVec<T>::unpack(rowp[i * 8], q[i]);     // pixel pitch = 8 x 16 B
      if constexpr (SEP) {
        // explicit _rn intrinsics: the products are rounded exactly as written (no contraction into other FMAs)
#pragma unroll
        for (int j = 0; j < COLS; ++j)
#pragma unroll
          for (int k = 0; k < V; ++k) {
            float h = __fmul_rn(kv[0], q[j][k]);
            h = __fmaf_rn(kv[1], q[j + 1][k], h);
            h = __fmaf_rn(kv[2], q[j + 2][k], h);
            h = __fmaf_rn(kv[3], q[j + 3][k], h);
            hwin[rr][j][k] = h;
          }
      } else {
#pragma unroll
        for (int i = 0; i < COLS + 3; ++i)
#pragma unroll
          for (int k = 0; k < V; ++k) rwin[rr][i][k] = q[i][k];
      }
      const int ro = r_in - 3;             // output row (relative to oy0) completed by this input row
      if (ro >= 0 && ro < rows_out) {
#pragma unroll
        for (int j = 0; j < COLS; ++j) {
          float a4[V];
          if constexpr (SEP) {
#pragma unroll
            for (int k = 0; k < V; ++k) {         // rows r_in-3 .. r_in in order
              float a = __fmul_rn(ku[0], hwin[(rr + 1) & 3][j][k]);
              a = __fmaf_rn(ku[1], hwin[(rr + 2) & 3][j][k], a);
              a = __fmaf_rn(ku[2], hwin[(rr + 3) & 3][j][k], a);
              a = __fmaf_rn(ku[3], hwin[rr][j][k], a);
              a4[k] = a;
            }
          } else {
#pragma unroll
            for (int k = 0; k < V; ++k) a4[k] = 0.f;
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
              for (int b = 0; b < 4; ++b)
#pragma unroll
                for (int k = 0; k < V; ++k) a4[k] = fmaf(kf[a][b], rwin[(rr + 1 + a) & 3][j + b][k], a4[k]);
          }
          const int64_t ooff = ocur + j * p.c;
          if (FUSED) {
            const float nzj = nw * nzc[rr][j];
            float o2[V];
#pragma unroll
            for (int k = 0; k < V; ++k) {
              float t = __fmaf_rn(a4[k], rq[k], __fadd_rn(bq[k], nzj));
              const float tn = __fmul_rn(t, neg);
              if (fast) t = fmaxf(t, tn);
              else t = (t > 0.f ? t : tn) * p.gain;
              a4[k] = t;
              o2[k] = __fmul_rn(t, sq[k]);
            }
            uint32_t word = 0u;
            if (MASK) word = sign_word<V>(sign_bits<T>(a4), cq, 0xffffffffu);   // `ro` is uniform: every lane is here
            if (okc[j]) {
              if (MASK) {
                if ((cq * V & 31) == 0) reinterpret_cast<uint32_t*>(out)[ooff >> 5] = word;
              } else if (out) {
                *reinterpret_cast<uint4*>(out + ooff) = ChanVec<T>::pack(a4);
              }
              if (out2) *reinterpret_cast<uint4*>(out2 + ooff) = ChanVec<T>::pack(o2);
            }
          } else if (MODE == 2) {
            if (okc[j]) {
              if (mul) {
                float mf[V];
                ChanVec<T>::unpack(mcur[j], mf);
#pragma unroll
                for (int k = 0; k < V; ++k) dacc[k] = fmaf(a4[k], mf[k], dacc[k]);
              }
#pragma unroll
              for (int k = 0; k < V; ++k) a4[k] *= rq[k];
              *reinterpret_cast<uint4*>(out + ooff) = ChanVec<T>::pack(a4);
            }
          } else {
            if (okc[j]) *reinterpret_cast<uint4*>(out + ooff) = ChanVec<T>::pack(a4);
          }
        }
      }
    }
    __syncthreads();   // the stage is free for the producer
  }
  if (MODE == 2 && partial) {
    // sum over the 32 column groups of the CTA: [xg][CB] in the (now idle) first stage, then one row per CTA at
    // partial[n][bx * gridDim.y + seg][C] (summed over the middle index by nhwc_finish_kernel)
    float* red = reinterpret_cast<float*>(tiles_raw);
#pragma unroll
    for (int k = 0; k < V; ++k) red[xg * CB + cq * V + k] = dacc[k];
    __syncthreads();
    if (tid < CB) {
      float t = 0.f;
#pragma unroll 8
      for (int g = 0; g < 32; ++g) t += red[g * CB + tid];
      const int64_t K = static_cast<int64_t>(gridDim.x / chunks) * gridDim.y;
      const int64_t kidx = static_cast<int64_t>(bx) * gridDim.y + blockIdx.y;
      partial[(static_cast<int64_t>(n) * K + kidx) * p.c + c0 + tid] = t;
    }
  }
}

// ---- host: tensor map through the driver entry point (no link-time libcuda dependency)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

inline int grid1(int64_t total, int per_cta) {
  int64_t g = (total + per_cta - 1) / per_cta;
  return static_cast<int>(g > 0 ? g : 1);
}

}  // namespace
}  // namespace gg

using namespace gg;

extern "C" {

static inline int vec_of(int dtype) { return dtype == GG_BF16 ? 8 : 4; }

int gg_noise_bias_act_nhwc(void* out, const void* x, const float* noise, const float* noise_weight, const float* bias,
                           const float* row_scale, int dtype, float alpha, float scale, int64_t N, int C, int64_t HW,
                           void* stream) {
  if (N < 0 || C < 0 || HW < 0) return fail(GG_ERR_BAD_ARG, "noise_bias_act_nhwc: negative size");
  if (dtype != GG_F32 && dtype != GG_BF16) return fail(GG_ERR_UNSUPPORTED, "noise_bias_act_nhwc: dtype %d not supported", dtype);
  const int64_t numel = N * HW * C;
  if (numel == 0) return GG_OK;
  const int V = vec_of(dtype);
  if (C % V != 0) return fail(GG_ERR_UNSUPPORTED, "noise_bias_act_nhwc: C must be a multiple of %d", V);
  if (!out || !x) return fail(GG_ERR_BAD_ARG, "noise_bias_act_nhwc: null tensor");
  if (!aligned16(bias) || !aligned16(row_scale))   // read as float4
    return fail(GG_ERR_BAD_ARG, "noise_bias_act_nhwc: bias and row_scale must be 16-byte aligned");
  const int64_t n_vec = numel / V;
  const int64_t grid = (n_vec + 4 * kT - 1) / (4 * kT);
  if (grid > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "noise_bias_act_nhwc: tensor too large");
  GG_DISPATCH_T(dtype, "noise_bias_act_nhwc",
                (noise_bias_act_nhwc_kernel<T_><<<static_cast<unsigned>(grid), kT, 0, static_cast<cudaStream_t>(stream)>>>(
                    static_cast<T_*>(out), static_cast<const T_*>(x), noise, noise_weight, bias, row_scale, alpha, scale,
                    n_vec, C / V, HW)));
  GG_CHECK_LAUNCH("noise_bias_act_nhwc launch");
  return GG_OK;
}

// Pixels per CTA: enough CTAs to fill the machine ~8x over, at least 4 trips of the CTA's pixel lanes each.
static int64_t rowwise_chunk(int64_t N, int cv, int64_t HW) {
  const int lanes_p = kT / cv > 0 ? kT / cv : 1;
  const int64_t target = 8LL * sm_count();
  int64_t k = (target + N - 1) / N;
  const int64_t kmax = (HW + 4 * lanes_p - 1) / (4 * lanes_p);
  if (k > kmax) k = kmax;
  if (k < 1) k = 1;
  return (HW + k - 1) / k;
}

int64_t gg_nhwc_rowwise_workspace(int64_t N, int C, int64_t HW) {
  if (N <= 0 || C <= 0 || HW <= 0 || C % 4 != 0) return 0;
  // the fp32 geometry has the most CTAs (4 channels per thread): sized for either storage type
  const int64_t chunk = rowwise_chunk(N, C / 4, HW);
  const int64_t chunk8 = (C % 8 == 0) ? rowwise_chunk(N, C / 8, HW) : chunk;
  const int64_t k = (HW + (chunk < chunk8 ? chunk : chunk8) - 1) / (chunk < chunk8 ? chunk : chunk8);
  return N * k * C * static_cast<int64_t>(sizeof(float));
}

static int launch_rowwise(int mode, void* out, float* dst, void* workspace, const void* x, const void* y, const float* s,
                          int dtype, float alpha, float gain, int64_t N, int C, int64_t HW, bool per_sample, void* stream) {
  if (N < 0 || C < 0 || HW < 0) return fail(GG_ERR_BAD_ARG, "nhwc rowwise: negative size");
  if (dtype != GG_F32 && dtype != GG_BF16) return fail(GG_ERR_UNSUPPORTED, "nhwc rowwise: dtype %d not supported", dtype);
  if (N * HW * C == 0) {
    // a sum over no pixels is 0: row_dot[N][C] (per sample) or grad_bias[C]
    const int64_t sums = (per_sample ? N : 1) * C;
    if (dst && sums > 0) {
      cudaError_t e = cudaMemsetAsync(dst, 0, sums * sizeof(float), static_cast<cudaStream_t>(stream));
      if (e != cudaSuccess) return cuda_fail(e, "nhwc rowwise memset");
    }
    return GG_OK;
  }
  const int V = vec_of(dtype);
  if (C % V != 0 || C / V > kT) return fail(GG_ERR_UNSUPPORTED, "nhwc rowwise: C must be a multiple of %d and <= %d", V, V * kT);
  if (!out || !x) return fail(GG_ERR_BAD_ARG, "nhwc rowwise: null tensor");
  if (dst && !workspace) return fail(GG_ERR_BAD_ARG, "nhwc rowwise: reduction needs a workspace");
  const int cv = C / V;
  const int64_t chunk64 = rowwise_chunk(N, cv, HW);
  if (chunk64 > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "nhwc rowwise: plane too large");
  const int chunk = static_cast<int>(chunk64);
  const int K = static_cast<int>((HW + chunk - 1) / chunk);
  const int64_t grid = N * K;
  if (grid > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "nhwc rowwise: too many CTAs");
  const int lanes_p = kT / cv > 0 ? kT / cv : 1;
  const size_t smem = static_cast<size_t>(lanes_p) * C * sizeof(float);
  float* partial = dst ? static_cast<float*>(workspace) : nullptr;
  auto st = static_cast<cudaStream_t>(stream);
  const unsigned g = static_cast<unsigned>(grid);
  if (mode == 0) {
    GG_DISPATCH_T(dtype, "nhwc rowwise",
                  (rowwise_nhwc_kernel<T_, 0><<<g, kT, smem, st>>>(static_cast<T_*>(out), partial, static_cast<const T_*>(x),
                                                                 dst ? static_cast<const T_*>(y) : nullptr, s, alpha, gain,
                                                                 cv, HW, chunk, K)));
  } else {
    GG_DISPATCH_T(dtype, "nhwc rowwise",
                  (rowwise_nhwc_kernel<T_, 1><<<g, kT, smem, st>>>(static_cast<T_*>(out), partial, static_cast<const T_*>(x),
                                                                 static_cast<const T_*>(y), s, alpha, gain, cv, HW, chunk, K)));
  }
  GG_CHECK_LAUNCH("nhwc rowwise launch");
  if (dst) {
    const int64_t rows = per_sample ? N : 1;
    const int kk = per_sample ? K : static_cast<int>(N * K);
    nhwc_finish_kernel<<<static_cast<unsigned>(rows * ((C + 31) / 32)), dim3(32, 32), 0, st>>>(dst, partial, rows, kk, C);
    GG_CHECK_LAUNCH("nhwc finish launch");
  }
  return GG_OK;
}

int gg_channel_scale_nhwc(void* out, float* row_dot, void* workspace, const void* x, const void* y, const float* s,
                          int dtype, int64_t N, int C, int64_t HW, void* stream) {
  if (!s) return fail(GG_ERR_BAD_ARG, "channel_scale_nhwc: null scale");
  if (row_dot && !y) return fail(GG_ERR_BAD_ARG, "channel_scale_nhwc: row_dot needs y");
  return launch_rowwise(0, out, row_dot, workspace, x, y, s, dtype, 0.f, 1.f, N, C, HW, true, stream);
}

int gg_bias_act_backward_nhwc(void* gx, float* grad_bias, void* workspace, const void* g, const void* out_saved,
                              int dtype, float alpha, float scale, int64_t N, int C, int64_t HW, void* stream) {
  if (!out_saved) return fail(GG_ERR_BAD_ARG, "bias_act_backward_nhwc: null saved output");
  return launch_rowwise(1, gx, grad_bias, workspace, g, out_saved, nullptr, dtype, alpha, scale, N, C, HW, false, stream);
}

int64_t gg_to_rgb_nhwc_workspace(int64_t N, int C, int64_t HW) { return 3 * gg_nhwc_rowwise_workspace(N, C, HW); }

int gg_to_rgb_nhwc_forward(float* out, const float* x, const float* wm, const float* bias, const float* skip, int64_t N,
                           int C, int64_t HW, void* stream) {
  if (N < 0 || C < 0 || HW < 0) return fail(GG_ERR_BAD_ARG, "to_rgb_nhwc: negative size");
  if (N * HW == 0) return GG_OK;
  if (C < 32 || C % 32 != 0 || C > 1024) return fail(GG_ERR_UNSUPPORTED, "to_rgb_nhwc: C must be a multiple of 32, <= 1024");
  if (!out || !x || !wm) return fail(GG_ERR_BAD_ARG, "to_rgb_nhwc: null tensor");
  // wm is read as float4; skip too, and out written as float4, when the planes are whole quads (HW % 4 == 0)
  if (!aligned16(wm) || (HW % 4 == 0 && (!aligned16(skip) || !aligned16(out))))
    return fail(GG_ERR_BAD_ARG, "to_rgb_nhwc: wm (and skip, out when HW %% 4 == 0) must be 16-byte aligned");
  // pixels per CTA: a multiple of the 128 pixels one trip covers, ~8 CTAs per SM over the whole batch
  const int64_t target = 8LL * sm_count();
  int64_t k = (target + N - 1) / N;
  const int64_t kmax = (HW + 127) / 128;
  if (k > kmax) k = kmax;
  if (k < 1) k = 1;
  int64_t chunk = ((HW + k - 1) / k + 127) / 128 * 128;
  if (chunk > 0x7fffff00LL) return fail(GG_ERR_BAD_ARG, "to_rgb_nhwc: plane too large");
  const int K = static_cast<int>((HW + chunk - 1) / chunk);
  const int64_t grid = N * K;
  if (grid > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "to_rgb_nhwc: too many CTAs");
  to_rgb_nhwc_fwd_kernel<<<static_cast<unsigned>(grid), kT, static_cast<size_t>(3) * C * sizeof(float),
                           static_cast<cudaStream_t>(stream)>>>(out, x, wm, bias, skip, C / 4, HW, static_cast<int>(chunk), K);
  GG_CHECK_LAUNCH("to_rgb_nhwc forward launch");
  return GG_OK;
}

int gg_to_rgb_nhwc_backward(float* gx, float* gwm, void* workspace, const float* g, const float* x, const float* wm,
                            int64_t N, int C, int64_t HW, void* stream) {
  if (N < 0 || C < 0 || HW < 0) return fail(GG_ERR_BAD_ARG, "to_rgb_nhwc backward: negative size");
  if (N * HW == 0 || C == 0) {
    if (gwm && N * C > 0) {   // gwm sums over no pixels: 0
      cudaError_t e = cudaMemsetAsync(gwm, 0, N * 3 * C * sizeof(float), static_cast<cudaStream_t>(stream));
      if (e != cudaSuccess) return cuda_fail(e, "to_rgb_nhwc backward memset");
    }
    return GG_OK;
  }
  if (C % 4 != 0 || C > 1024) return fail(GG_ERR_UNSUPPORTED, "to_rgb_nhwc backward: C must be a multiple of 4, <= 1024");
  if (!g || !wm || (!gx && !gwm)) return fail(GG_ERR_BAD_ARG, "to_rgb_nhwc backward: null tensor");
  if (gwm && (!x || !workspace)) return fail(GG_ERR_BAD_ARG, "to_rgb_nhwc backward: gwm needs x and a workspace");
  if (!aligned16(wm)) return fail(GG_ERR_BAD_ARG, "to_rgb_nhwc backward: wm must be 16-byte aligned");   // read as float4
  const int c4 = C / 4;
  const int64_t chunk64 = rowwise_chunk(N, c4, HW);
  if (chunk64 > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "to_rgb_nhwc backward: plane too large");
  const int chunk = static_cast<int>(chunk64);
  const int K = static_cast<int>((HW + chunk - 1) / chunk);
  const int64_t grid = N * K;
  if (grid > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "to_rgb_nhwc backward: too many CTAs");
  const int lanes_p = kT / c4 > 0 ? kT / c4 : 1;
  const size_t smem = static_cast<size_t>(lanes_p) * 3 * C * sizeof(float);
  auto st = static_cast<cudaStream_t>(stream);
  float* partial = gwm ? static_cast<float*>(workspace) : nullptr;
  to_rgb_nhwc_bwd_kernel<<<static_cast<unsigned>(grid), kT, smem, st>>>(gx, partial, g, x, wm, c4, HW, chunk, K);
  GG_CHECK_LAUNCH("to_rgb_nhwc backward launch");
  if (gwm) {
    nhwc_finish_kernel<<<static_cast<unsigned>(N * ((3 * C + 31) / 32)), dim3(32, 32), 0, st>>>(gwm, partial, N, K, 3 * C);
    GG_CHECK_LAUNCH("to_rgb_nhwc finish launch");
  }
  return GG_OK;
}

// ---- blur: geometry shared by the launch and the workspace query
struct BlurPlan {
  int out_h, out_w, xblocks, chunks, segs, seg_rows;
};
static int blur_plan(BlurPlan* pl, int dtype, int64_t N, int C, int in_h, int in_w, int kernel_h, int kernel_w, int pad_x0,
                     int pad_x1, int pad_y0, int pad_y1) {
  const int V = vec_of(dtype);
  const int CB = 8 * V, BX = (V == 4) ? 64 : 32;
  if (C % CB != 0) return fail(GG_ERR_UNSUPPORTED, "blur_nhwc: C must be a multiple of %d", CB);
  pl->out_h = in_h + pad_y0 + pad_y1 - kernel_h + 1;
  pl->out_w = in_w + pad_x0 + pad_x1 - kernel_w + 1;
  if (pl->out_h < 1 || pl->out_w < 1) return fail(GG_ERR_BAD_ARG, "blur_nhwc: empty output");
  pl->xblocks = (pl->out_w + BX - 1) / BX;
  pl->chunks = C / CB;
  // row segments: enough CTAs to fill the machine twice, at least 16 rows each (3 halo rows per segment)
  const int64_t base_ctas = static_cast<int64_t>(pl->xblocks) * pl->chunks * (N > 0 ? N : 1);
  int segs = static_cast<int>((2LL * 2 * sm_count() + base_ctas - 1) / base_ctas);
  int seg_rows = (pl->out_h + segs - 1) / segs;
  if (seg_rows < 16) seg_rows = pl->out_h < 16 ? pl->out_h : 16;
  seg_rows = (seg_rows + 3) / 4 * 4;
  pl->seg_rows = seg_rows;
  pl->segs = (pl->out_h + seg_rows - 1) / seg_rows;
  return GG_OK;
}

int64_t gg_blur_nhwc_workspace(int dtype, int64_t N, int C, int in_h, int in_w, int kernel_h, int kernel_w, int pad_x0,
                               int pad_x1, int pad_y0, int pad_y1) {
  BlurPlan pl;
  if (N <= 0 || C <= 0 || (dtype != GG_F32 && dtype != GG_BF16)) return 0;
  if (blur_plan(&pl, dtype, N, C, in_h, in_w, kernel_h, kernel_w, pad_x0, pad_x1, pad_y0, pad_y1) != GG_OK) return 0;
  return N * static_cast<int64_t>(pl.xblocks) * pl.segs * C * static_cast<int64_t>(sizeof(float));
}

}  // extern "C"

template <typename T>
static int launch_blur(void* out, void* out2, const void* in, const float* kernel, const float* noise,
                       const float* noise_weight, const float* bias, const float* row_scale, const float* scale2,
                       const void* mul, float* row_dot, void* workspace, int64_t N, int C, int in_h, int in_w, int kernel_h,
                       int kernel_w, int separable, int pad_x0, int pad_x1, int pad_y0, int pad_y1, int mode, int act,
                       float alpha, float scale, void* stream, int dtype, bool out_is_mask) {
  using G = BlurGeom<T>;
  BlurPlan pl;
  int rc = blur_plan(&pl, dtype, N, C, in_h, in_w, kernel_h, kernel_w, pad_x0, pad_x1, pad_y0, pad_y1);
  if (rc != GG_OK) return rc;
  EncodeTiledFn enc = encode_fn();
  if (!enc) return fail(GG_ERR_CUDA, "blur_nhwc: cuTensorMapEncodeTiled is not available from this driver");
  // descriptors are memoised per (address, shape, type): a training loop (or a captured graph's warm-up) presents the
  // same few activations again and again
  struct MapKey { const void* ptr; int64_t n; int c, h, w, es; };
  struct MapEnt { MapKey key; CUtensorMap map; bool valid; };
  static thread_local MapEnt cache[16] = {};
  static thread_local unsigned cache_next = 0;
  const MapKey key = {in, N, C, in_h, in_w, static_cast<int>(sizeof(T))};
  const CUtensorMap* cached = nullptr;
  for (int i = 0; i < 16 && !cached; ++i)
    if (cache[i].valid && cache[i].key.ptr == key.ptr && cache[i].key.n == key.n && cache[i].key.c == key.c &&
        cache[i].key.h == key.h && cache[i].key.w == key.w && cache[i].key.es == key.es)
      cached = &cache[i].map;
  CUtensorMap tmap;
  if (cached) tmap = *cached;
  const cuuint64_t es = sizeof(T);
  const cuuint64_t gdim[4] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(in_w), static_cast<cuuint64_t>(in_h),
                              static_cast<cuuint64_t>(N)};
  const cuuint64_t gstr[3] = {static_cast<cuuint64_t>(C) * es, static_cast<cuuint64_t>(in_w) * C * es,
                              static_cast<cuuint64_t>(in_h) * in_w * C * es};
  const cuuint32_t box[4] = {G::CB, G::TW, kRY, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  if (!cached) {
    const CUresult r = enc(&tmap, sizeof(T) == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4,
                           const_cast<void*>(in), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(GG_ERR_CUDA, "blur_nhwc: cuTensorMapEncodeTiled failed (%d)", static_cast<int>(r));
    MapEnt& e = cache[cache_next++ % 16];
    e.key = key; e.map = tmap; e.valid = true;
  }
  BlurNhwcParams p;
  p.n = static_cast<int>(N); p.c = C; p.in_h = in_h; p.in_w = in_w; p.out_h = pl.out_h; p.out_w = pl.out_w;
  p.pad_x0 = pad_x0; p.pad_y0 = pad_y0;
  p.act = act; p.alpha = alpha; p.gain = scale;
  p.seg_rows = pl.seg_rows;
  const dim3 grid(static_cast<unsigned>(pl.xblocks * pl.chunks), static_cast<unsigned>(pl.segs), static_cast<unsigned>(N));
  const size_t smem = static_cast<size_t>(kNS) * G::STAGE_ELEMS * sizeof(T);
  static DeviceOnce configured;
  if (configured.needed()) {
    cudaError_t e = cudaSuccess;
    const void* kernels[12] = {reinterpret_cast<const void*>(blur_nhwc_kernel<T, 0, true>),
                              reinterpret_cast<const void*>(blur_nhwc_kernel<T, 0, false>),
                              reinterpret_cast<const void*>(blur_nhwc_kernel<T, 1, true, false>),
                              reinterpret_cast<const void*>(blur_nhwc_kernel<T, 1, false, false>),
                              reinterpret_cast<const void*>(blur_nhwc_kernel<T, 1, true, true>),
                              reinterpret_cast<const void*>(blur_nhwc_kernel<T, 1, false, true>),
                              reinterpret_cast<const void*>(blur_nhwc_kernel<T, 3, true, false>),
                              reinterpret_cast<const void*>(blur_nhwc_kernel<T, 3, false, false>),
                              reinterpret_cast<const void*>(blur_nhwc_kernel<T, 3, true, true>),
                              reinterpret_cast<const void*>(blur_nhwc_kernel<T, 3, false, true>),
                              reinterpret_cast<const void*>(blur_nhwc_kernel<T, 2, true>),
                              reinterpret_cast<const void*>(blur_nhwc_kernel<T, 2, false>)};
    for (int i = 0; i < 12 && e == cudaSuccess; ++i)
      e = cudaFuncSetAttribute(kernels[i], cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return cuda_fail(e, "blur_nhwc smem opt-in");
    configured.done();
  }
  auto st = static_cast<cudaStream_t>(stream);
  float* partial = (mode == 2 && row_dot) ? static_cast<float*>(workspace) : nullptr;
  const bool fast = scale > 0.f && ((act == 3 && alpha >= 0.f && alpha <= 1.f) || act == 1);
#define GG_BLUR(M_, S_, F_)                                                                                          \
  blur_nhwc_kernel<T, M_, S_, F_><<<grid, kT, smem, st>>>(static_cast<T*>(out), static_cast<T*>(out2), tmap, kernel, kernel_h, \
                                                         kernel_w, noise, noise_weight, bias, row_scale, scale2,     \
                                                         static_cast<const T*>(mul), partial, p)
  if (mode == 1 && out_is_mask) {
    if (fast) { if (separable) GG_BLUR(3, true, true); else GG_BLUR(3, false, true); }
    else { if (separable) GG_BLUR(3, true, false); else GG_BLUR(3, false, false); }
  }
  else if (mode == 1) {
    if (fast) { if (separable) GG_BLUR(1, true, true); else GG_BLUR(1, false, true); }
    else { if (separable) GG_BLUR(1, true, false); else GG_BLUR(1, false, false); }
  }
  else if (mode == 2) { if (separable) GG_BLUR(2, true, false); else GG_BLUR(2, false, false); }
  else { if (separable) GG_BLUR(0, true, false); else GG_BLUR(0, false, false); }
#undef GG_BLUR
  GG_CHECK_LAUNCH("blur_nhwc launch");
  if (partial) {
    const int K = pl.xblocks * pl.segs;
    nhwc_finish_kernel<<<static_cast<unsigned>(N * ((C + 31) / 32)), dim3(32, 32), 0, st>>>(row_dot, partial, N, K, C);
    GG_CHECK_LAUNCH("blur_nhwc finish launch");
  }
  return GG_OK;
}

extern "C" {

int gg_blur_nhwc(void* out, void* out2, const void* in, const float* kernel, const float* noise, const float* noise_weight,
                 const float* bias, const float* row_scale, const float* scale2, const void* mul, float* row_dot,
                 void* workspace, int dtype, int64_t N, int C, int in_h, int in_w, int kernel_h, int kernel_w, int separable,
                 int pad_x0, int pad_x1, int pad_y0, int pad_y1, int mode, int act, float alpha, float scale, void* stream) {
  if (N < 0 || C < 0 || in_h < 1 || in_w < 1) return fail(GG_ERR_BAD_ARG, "blur_nhwc: bad shape");
  if (kernel_h < 1 || kernel_w < 1 || kernel_h > 4 || kernel_w > 4) return fail(GG_ERR_UNSUPPORTED, "blur_nhwc: filter must be <= 4x4");
  if (mode < 0 || mode > 2) return fail(GG_ERR_BAD_ARG, "blur_nhwc: mode must be 0 (blur), 1 (fused tail) or 2 (adjoint epilogue)");
  if (act != 1 && act != 3) return fail(GG_ERR_UNSUPPORTED, "blur_nhwc: act must be 1 or 3");
  if (dtype != GG_F32 && dtype != GG_BF16) return fail(GG_ERR_UNSUPPORTED, "blur_nhwc: dtype %d not supported (fp32 or bf16)", dtype);
  if (N == 0 || C == 0) return GG_OK;
  if (!in || !kernel) return fail(GG_ERR_BAD_ARG, "blur_nhwc: null tensor");
  if (mode == 1 ? (!out && !out2) : !out) return fail(GG_ERR_BAD_ARG, "blur_nhwc: null output");
  if (mode != 1 && out2) return fail(GG_ERR_BAD_ARG, "blur_nhwc: out2 belongs to the fused tail (mode 1)");
  if (mode == 2 && row_dot && (!mul || !workspace)) return fail(GG_ERR_BAD_ARG, "blur_nhwc: row_dot needs `mul` and a workspace");
  if (N > 65535) return fail(GG_ERR_UNSUPPORTED, "blur_nhwc: batch > 65535");
  if (mode == 0) { noise = nullptr; noise_weight = nullptr; bias = nullptr; row_scale = nullptr; scale2 = nullptr; }
  GG_DISPATCH_T(dtype, "blur_nhwc",
                return launch_blur<T_>(out, out2, in, kernel, noise, noise_weight, bias, row_scale, scale2, mul, row_dot,
                                       workspace, N, C, in_h, in_w, kernel_h, kernel_w, separable, pad_x0, pad_x1, pad_y0,
                                       pad_y1, mode, act, alpha, scale, stream, dtype, false));
  return GG_OK;
}

int gg_blur_nhwc_mask(void* mask, void* out2, const void* in, const float* kernel, const float* noise,
                      const float* noise_weight, const float* bias, const float* row_scale, const float* scale2, int dtype,
                      int64_t N, int C, int in_h, int in_w, int kernel_h, int kernel_w, int separable, int pad_x0, int pad_x1,
                      int pad_y0, int pad_y1, int act, float alpha, float scale, void* stream) {
  if (N < 0 || C < 0 || in_h < 1 || in_w < 1) return fail(GG_ERR_BAD_ARG, "blur_nhwc_mask: bad shape");
  if (kernel_h < 1 || kernel_w < 1 || kernel_h > 4 || kernel_w > 4) return fail(GG_ERR_UNSUPPORTED, "blur_nhwc_mask: filter must be <= 4x4");
  if (act != 1 && act != 3) return fail(GG_ERR_UNSUPPORTED, "blur_nhwc_mask: act must be 1 or 3");
  if (dtype != GG_F32 && dtype != GG_BF16) return fail(GG_ERR_UNSUPPORTED, "blur_nhwc_mask: dtype %d not supported (fp32 or bf16)", dtype);
  if (N == 0 || C == 0) return GG_OK;
  if (!in || !kernel) return fail(GG_ERR_BAD_ARG, "blur_nhwc_mask: null tensor");
  if (!mask) return fail(GG_ERR_BAD_ARG, "blur_nhwc_mask: null mask");
  if (out2 && !scale2) return fail(GG_ERR_BAD_ARG, "blur_nhwc_mask: out2 needs scale2");
  if (N > 65535) return fail(GG_ERR_UNSUPPORTED, "blur_nhwc_mask: batch > 65535");
  GG_DISPATCH_T(dtype, "blur_nhwc_mask",
                return launch_blur<T_>(mask, out2, in, kernel, noise, noise_weight, bias, row_scale, scale2, nullptr, nullptr,
                                       nullptr, N, C, in_h, in_w, kernel_h, kernel_w, separable, pad_x0, pad_x1, pad_y0,
                                       pad_y1, 1, act, alpha, scale, stream, dtype, true));
  return GG_OK;
}

}  // extern "C"
