// flow.cu -- flow composition of the flow STN head in one pass, forward and backward (sm_90a).
//
// Replaces ~20 ATen launches of reference models/spatial_transformers/warping_heads.py:
//   upsample_flow (:180-193)  softmax over the 9 mask logits, F.unfold(8*flow, 3x3), weighted sum, 2 permutes
//   FlowHead.forward (:239-244) flow = identity_flow + delta_flow; apply_affine(base_warp, flow) (:268-277);
//                               identity_flow.lerp(flow, alpha)
// One thread per full-resolution flow pixel; tensors are KB-sized, so the cost is launch latency and the
// win is launch count.  Algorithmic bytes per sample (K=1, 16x16 -> 128x128): mask 0.59 MB + outputs 0.26 MB.
#include "flow_compose.cuh"

namespace gg {
namespace {

struct FlowParams {
  int64_t n;       // samples (N*K)
  int h, w;        // low-res size
  int s;           // flow_downsample (8)
};

// index helpers: mask is (N, 9*s*s, H, W) viewed (N, 9, s, s, H, W) (warping_heads.py:184)
__device__ __forceinline__ int64_t mask_index(const FlowParams& p, int64_t n, int k, int sy, int sx, int h, int w) {
  return ((((n * 9 + k) * p.s + sy) * p.s + sx) * p.h + h) * static_cast<int64_t>(p.w) + w;
}

// thread index -> (n, sy, sx, h, w) in mask memory order (w fastest): coalesced mask reads
__device__ __forceinline__ void decode(const FlowParams& p, int64_t idx, int64_t& n, int& sy, int& sx, int& h, int& w) {
  w = static_cast<int>(idx % p.w); idx /= p.w;
  h = static_cast<int>(idx % p.h); idx /= p.h;
  sx = static_cast<int>(idx % p.s); idx /= p.s;
  sy = static_cast<int>(idx % p.s); idx /= p.s;
  n = idx;
}

__global__ void __launch_bounds__(256)
flow_compose_fwd_kernel(float* __restrict__ delta_out, float* __restrict__ flow_out, const float* __restrict__ low,
                        const float* __restrict__ mask, const float* __restrict__ identity,
                        const float* __restrict__ base, const float* __restrict__ alpha, FlowParams p, int64_t total) {
  for (int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    int64_t n; int sy, sx, h, w;
    decode(p, idx, n, sy, sx, h, w);
    float pk[9], fx[9], fy[9];
    const float2 u = convex_upsample(low, mask, n, p.h, p.w, p.s, sy, sx, h, w, pk, fx, fy);
    const int Y = h * p.s + sy, X = w * p.s + sx;
    const int64_t pix = (static_cast<int64_t>(Y) * (p.w * p.s) + X) * 2;
    const int64_t o = n * (p.h * p.s) * static_cast<int64_t>(p.w * p.s) * 2 + pix;
    *reinterpret_cast<float2*>(delta_out + o) = u;
    if (flow_out) {
      const float2 id = *reinterpret_cast<const float2*>(identity + pix);
      *reinterpret_cast<float2*>(flow_out + o) = compose_flow(id, u.x, u.y, base, alpha, n);
    }
  }
}

// backward of one full-resolution pixel: the forward's convex up-sampling (softmax weights, scaled neighbourhood), the
// gradient arriving at delta (gdx, gdy) and, with g_flow and base, this pixel's terms of d loss / d base (v, zero otherwise)
struct PixelGrad {
  float pk[9], fx[9], fy[9];
  float gdx, gdy;
  float v[6];
};

__device__ __forceinline__ void pixel_grad(const FlowParams& p, int64_t n, int sy, int sx, int h, int w,
                                           const float* __restrict__ g_delta, const float* __restrict__ g_flow,
                                           const float* __restrict__ low, const float* __restrict__ mask,
                                           const float* __restrict__ identity, const float* __restrict__ base,
                                           const float* __restrict__ alpha, PixelGrad& r) {
  const int Y = h * p.s + sy, X = w * p.s + sx;
  const int64_t pix = (static_cast<int64_t>(Y) * (p.w * p.s) + X) * 2;
  const int64_t o = n * (p.h * p.s) * static_cast<int64_t>(p.w * p.s) * 2 + pix;
  const float2 d = convex_upsample(low, mask, n, p.h, p.w, p.s, sy, sx, h, w, r.pk, r.fx, r.fy);
#pragma unroll
  for (int q = 0; q < 6; ++q) r.v[q] = 0.f;
  // gradient arriving at delta
  float gdx = 0.f, gdy = 0.f;
  if (g_delta) { const float2 g = *reinterpret_cast<const float2*>(g_delta + o); gdx = g.x; gdy = g.y; }
  if (g_flow) {
    float2 gf = *reinterpret_cast<const float2*>(g_flow + o);
    if (alpha) { const float a = alpha[n]; gf.x *= a; gf.y *= a; }
    if (base) {
      const float2 id = *reinterpret_cast<const float2*>(identity + pix);
      const float gx = id.x + d.x, gy = id.y + d.y;
      const float* M = base + n * 6;
      r.v[0] = gf.x * gx; r.v[1] = gf.x * gy; r.v[2] = gf.x;
      r.v[3] = gf.y * gx; r.v[4] = gf.y * gy; r.v[5] = gf.y;
      const float px = M[0] * gf.x + M[3] * gf.y;
      const float py = M[1] * gf.x + M[4] * gf.y;
      gf.x = px; gf.y = py;
    }
    gdx += gf.x; gdy += gf.y;
  }
  r.gdx = gdx; r.gdy = gdy;
}

// backward, g_mask: one thread per full-resolution pixel (its 9 logits)
__global__ void __launch_bounds__(256)
flow_compose_bwd_kernel(float* __restrict__ g_mask, const float* __restrict__ g_delta, const float* __restrict__ g_flow,
                        const float* __restrict__ low, const float* __restrict__ mask,
                        const float* __restrict__ identity, const float* __restrict__ base,
                        const float* __restrict__ alpha, FlowParams p, int64_t total) {
  for (int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    int64_t n; int sy, sx, h, w;
    decode(p, idx, n, sy, sx, h, w);
    PixelGrad r;
    pixel_grad(p, n, sy, sx, h, w, g_delta, g_flow, low, mask, identity, base, alpha, r);
    // through the convex combination: d/dlogit_k = p_k (t_k - sum_j p_j t_j), t_k = <g, f_k>
    float t[9], tbar = 0.f;
#pragma unroll
    for (int k = 0; k < 9; ++k) { t[k] = r.gdx * r.fx[k] + r.gdy * r.fy[k]; tbar = fmaf(r.pk[k], t[k], tbar); }
#pragma unroll
    for (int k = 0; k < 9; ++k) g_mask[mask_index(p, n, k, sy, sx, h, w)] = r.pk[k] * (t[k] - tbar);
  }
}

// The two reductions of the backward pass are GATHERED, without atomics, so that they are the same in every run.
// g_low: one warp per low-resolution entry (n, hh, ww); its lanes walk, in a fixed order, the 9*s*s full-resolution pixels
// whose 3x3 neighbourhood holds it, and meet in a butterfly sum.
__global__ void __launch_bounds__(256)
flow_low_bwd_kernel(float* __restrict__ g_low, const float* __restrict__ g_delta, const float* __restrict__ g_flow,
                    const float* __restrict__ low, const float* __restrict__ mask, const float* __restrict__ identity,
                    const float* __restrict__ base, const float* __restrict__ alpha, FlowParams p, int64_t entries) {
  const int lane = threadIdx.x & 31;
  const int ss = p.s * p.s;
  for (int64_t e = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; e < entries;
       e += (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5) {
    const int ww = static_cast<int>(e % p.w);
    const int hh = static_cast<int>((e / p.w) % p.h);
    const int64_t n = e / (static_cast<int64_t>(p.w) * p.h);
    float ax = 0.f, ay = 0.f;
    for (int j = lane; j < 9 * ss; j += 32) {
      const int k = j / ss, sy = (j % ss) / p.s, sx = j % p.s;
      const int h = hh - k / 3 + 1, w = ww - k % 3 + 1;      // the pixel block whose neighbour k is (hh, ww)
      if (h < 0 || h >= p.h || w < 0 || w >= p.w) continue;
      PixelGrad r;
      pixel_grad(p, n, sy, sx, h, w, g_delta, g_flow, low, mask, identity, base, alpha, r);
      const float sc = static_cast<float>(p.s) * r.pk[k];
      ax = fmaf(sc, r.gdx, ax);
      ay = fmaf(sc, r.gdy, ay);
    }
    ax = warp_sum(ax);
    ay = warp_sum(ay);
    if (lane == 0) *reinterpret_cast<float2*>(g_low + e * 2) = make_float2(ax, ay);
  }
}

// g_base: one CTA per sample, a fixed-order block reduction of the 6 terms of its pixels
constexpr int kBaseThreads = 256;
__global__ void __launch_bounds__(kBaseThreads)
flow_base_bwd_kernel(float* __restrict__ g_base, const float* __restrict__ g_delta, const float* __restrict__ g_flow,
                     const float* __restrict__ low, const float* __restrict__ mask, const float* __restrict__ identity,
                     const float* __restrict__ base, const float* __restrict__ alpha, FlowParams p) {
  const int64_t n = blockIdx.x;
  const int64_t per_sample = static_cast<int64_t>(p.s) * p.s * p.h * p.w;
  float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int64_t i = threadIdx.x; i < per_sample; i += kBaseThreads) {
    int64_t nn; int sy, sx, h, w;
    decode(p, n * per_sample + i, nn, sy, sx, h, w);
    PixelGrad r;
    pixel_grad(p, nn, sy, sx, h, w, g_delta, g_flow, low, mask, identity, base, alpha, r);
#pragma unroll
    for (int q = 0; q < 6; ++q) acc[q] += r.v[q];
  }
  __shared__ float part[kBaseThreads / 32][6];
#pragma unroll
  for (int q = 0; q < 6; ++q) {
    const float v = warp_sum(acc[q]);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5][q] = v;
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    float t = 0.f;
    for (int wi = 0; wi < kBaseThreads / 32; ++wi) t += part[wi][threadIdx.x];
    g_base[n * 6 + threadIdx.x] = t;
  }
}

}  // namespace
}  // namespace gg

using namespace gg;

extern "C" {

int gg_flow_compose_forward(float* delta_flow, float* flow, const float* low_flow, const float* mask,
                            const float* identity_flow, const float* base_warp, const float* alpha, int64_t N,
                            int H, int W, int S, void* stream) {
  if (N < 0 || H < 1 || W < 1 || S < 1) return fail(GG_ERR_BAD_ARG, "flow_compose_forward: bad shape");
  if (N == 0) return GG_OK;
  if (!delta_flow || !low_flow || !mask) return fail(GG_ERR_BAD_ARG, "flow_compose_forward: null tensor");
  if (flow && !identity_flow) return fail(GG_ERR_BAD_ARG, "flow_compose_forward: flow output needs identity_flow");
  FlowParams p{N, H, W, S};
  const int64_t total = N * S * S * H * static_cast<int64_t>(W);
  flow_compose_fwd_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      delta_flow, flow, low_flow, mask, identity_flow, base_warp, alpha, p, total);
  GG_CHECK_LAUNCH("flow_compose_fwd launch");
  return GG_OK;
}

int gg_flow_compose_backward(float* grad_mask, float* grad_low_flow, float* grad_base_warp, const float* grad_delta,
                             const float* grad_flow, const float* low_flow, const float* mask,
                             const float* identity_flow, const float* base_warp, const float* alpha, int64_t N,
                             int H, int W, int S, void* stream) {
  if (N < 0 || H < 1 || W < 1 || S < 1) return fail(GG_ERR_BAD_ARG, "flow_compose_backward: bad shape");
  if (N == 0) return GG_OK;
  if (!low_flow || !mask) return fail(GG_ERR_BAD_ARG, "flow_compose_backward: null tensor");
  if (grad_flow && base_warp && !identity_flow) return fail(GG_ERR_BAD_ARG, "flow_compose_backward: identity_flow required");
  FlowParams p{N, H, W, S};
  const int64_t total = N * S * S * H * static_cast<int64_t>(W);
  auto st = static_cast<cudaStream_t>(stream);
  if (grad_mask)
    flow_compose_bwd_kernel<<<grid_for(total, 256), 256, 0, st>>>(grad_mask, grad_delta, grad_flow, low_flow, mask, identity_flow,
                                                             base_warp, alpha, p, total);
  if (grad_low_flow) {
    const int64_t entries = N * H * static_cast<int64_t>(W);
    flow_low_bwd_kernel<<<grid_for(entries * 32, 256), 256, 0, st>>>(grad_low_flow, grad_delta, grad_flow, low_flow, mask,
                                                                 identity_flow, base_warp, alpha, p, entries);
  }
  if (grad_base_warp && grad_flow && base_warp) {
    if (N > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "flow_compose_backward: too many samples");
    flow_base_bwd_kernel<<<static_cast<unsigned>(N), kBaseThreads, 0, st>>>(grad_base_warp, grad_delta, grad_flow, low_flow,
                                                                           mask, identity_flow, base_warp, alpha, p);
  }
  GG_CHECK_LAUNCH("flow_compose_bwd launch");
  return GG_OK;
}

}  // extern "C"
