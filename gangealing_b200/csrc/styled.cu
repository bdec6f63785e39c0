// styled.cu -- the generator's StyledConv / ToRGB tails fused ACROSS layer boundaries on channels-last activations (sm_90a).
//
// The weight-shared modulated convolution conv(scale*W, x*s) (op/modconv.py) needs the activation scaled per (sample,
// channel) by the NEXT layer's style.  Round 1 paid for that with a separate streaming pass per convolution
// (`channel_scale`: read + write of the whole activation forward, read + read + write backward: 15.7 % of the step).
// Here the scaling rides in the epilogue of the kernel that PRODUCES the activation, the to-RGB 1x1 convolution
// (3 outputs per pixel -- no tensor-core shape) rides there too, and the backward of all of it is one pass:
//
//   gg_styled_tail_nhwc   raw -> o = lrelu(demod[n,c]*raw + nw*noise[n,p] + bias[c])*gain           networks.py:291-298,346-348
//                          writes  out = o            (optional: only when a backward pass will need it)
//                                  xs  = o*s_next[n,c] (optional: the next modulated convolution's input, networks.py:236,243)
//                                  rgb[n,:,p] = wm[n,:,:] . o + rgb_bias + skip[n,:,p]  (optional: ToRGB, networks.py:389-405)
//                          ONE read of raw; at the last layer without a backward pass nothing but the image is written.
//   gg_styled_tail_backward_nhwc   g_o = g_xs*s_next + wm^T g_rgb ; g_t = lrelu'(out)*gain*g_o ; g_raw = g_t*demod
//                          + per-(sample, channel) sums  d_s_next = sum_p g_xs*out,  d_demod = sum_p g_t*raw,
//                            d_wm[o] = sum_p g_rgb[o]*out          (deterministic two-stage reductions)
//                          ONE pass over (g_xs, out[, raw]) -> g_raw, replacing channel_scale-backward, the gradient
//                          add of the RGB branch, to_rgb-backward, bias_act-backward and the demodulation row-dot.
// (The blur tail of the up-sampling layers is csrc/nhwc.cu's blur kernel with the same `out2 = o*scale2` epilogue, and its
// adjoint with the `*demod, sum t*raw` epilogue.)
//
// Storage type T = fp32 or bf16 (BASELINE config 3); arithmetic is fp32; 16 bytes of channels per access.
#include "common.cuh"
#include "nhwc_reduce.cuh"

namespace gg {
namespace {

constexpr int kT = 256;
constexpr int kGroup = 8;      // lanes that share one pixel (a 128-byte line of the activation per load instruction)
constexpr int kPix = 4;        // consecutive pixels per group per trip

struct TailFwdParams {
  const void* raw; void* out; void* xs; float* rgb; const float* skip;
  const float* noise; const float* noise_weight; const float* bias; const float* demod; const float* s_next;
  const float* wm; const float* rgb_bias;
  float alpha, gain;
  int act;
  int C;
  int64_t hw;
  int chunk, chunks_per_sample;
};

// CTA = `chunk` consecutive pixels of one sample.  The per-channel constants of that sample (demod*gain, bias*gain, s_next,
// the three to-RGB rows) are staged once in shared memory; a group of 8 lanes owns 4 consecutive pixels per trip and walks
// the channel vectors v = lane + 8j: 4 independent 16-byte loads in flight per lane, every constant fetched once per 4 pixels.
// FAST: the gain-folded epilogue max(T, T*slope) is valid for the launch (host check) -- compile-time, so that the general
// select-and-scale epilogue is not predicated into the pixel loop next to it.
// MASK: `out` is the sign mask (common.cuh) instead of the activation -- all a backward pass without reductions needs of o.
template <typename T, bool FAST, bool MASK>
__global__ void __launch_bounds__(kT, 2)
styled_tail_nhwc_kernel(const TailFwdParams p) {
  constexpr int V = ChanVec<T>::V;
  constexpr int Q = V / 4;                              // float4 quarters per channel vector
  // constants of this sample, one plane per quarter so that lane l reads float4 #v of a plane (16-byte stride between the
  // lanes of a group: conflict-free LDS.128): cst[k][q][nvec] float4, k = d, b, s, w0, w1, w2
  extern __shared__ __align__(16) float cst[];
  const int C = p.C;
  const int nvec = C / V, J = nvec / kGroup;
  const int64_t n = blockIdx.x / p.chunks_per_sample;
  const int ck = blockIdx.x - n * p.chunks_per_sample;
  const int64_t p0 = static_cast<int64_t>(ck) * p.chunk, p1 = min(p0 + p.chunk, p.hw);
  constexpr bool fast = FAST;   // gain > 0 && ((act == 3 && 0 <= alpha <= 1) || act == 1)
  const float neg = (p.act == 3) ? p.alpha : 1.f;
  const float gfold = fast ? p.gain : 1.f;   // lrelu(t)*g == max(T, T*slope) with T = g*t: the gain folds into d, b, nw
  for (int c = threadIdx.x; c < C; c += kT) {
    const int v = c / V, r = c - v * V, q = r >> 2, e = r & 3;
    const int slot = (q * nvec + v) * 4 + e;            // plane k starts at k*C
    cst[slot] = (p.demod ? __ldg(p.demod + n * C + c) : 1.f) * gfold;
    cst[C + slot] = (p.bias ? __ldg(p.bias + c) : 0.f) * gfold;
    cst[2 * C + slot] = p.s_next ? __ldg(p.s_next + n * C + c) : 1.f;
    if (p.rgb) {
      cst[3 * C + slot] = __ldg(p.wm + (n * 3 + 0) * C + c);
      cst[4 * C + slot] = __ldg(p.wm + (n * 3 + 1) * C + c);
      cst[5 * C + slot] = __ldg(p.wm + (n * 3 + 2) * C + c);
    }
  }
  const float nw = (p.noise ? (p.noise_weight ? __ldg(p.noise_weight) : 1.f) : 0.f) * gfold;
  __syncthreads();
  const float4* c4 = reinterpret_cast<const float4*>(cst);
  const int c4_plane = C / 4;                           // float4s per constant plane
  const int l = threadIdx.x & (kGroup - 1), grp = threadIdx.x / kGroup;
  const unsigned gmask = 0xffu << (threadIdx.x & 24);    // the groups of one warp may leave the loop at different trips
  // per-sample base pointers + 32-bit in-sample offsets (the host checks hw*C < 2^31): the pixel loop then needs no 64-bit
  // multiplies and half the index registers (the bf16 instantiation sits at the 128-register cap of 2 CTAs/SM)
  const int hw = static_cast<int>(p.hw);
  const T* raw = static_cast<const T*>(p.raw) + n * hw * C;
  T* out = (p.out && !MASK) ? static_cast<T*>(p.out) + n * hw * C : nullptr;
  uint32_t* mask = MASK ? static_cast<uint32_t*>(p.out) + n * hw * (C >> 5) : nullptr;
  T* xs = p.xs ? static_cast<T*>(p.xs) + n * hw * C : nullptr;
  const float* noise_n = p.noise ? p.noise + n * hw : nullptr;
  const int q0 = static_cast<int>(p0), q1 = static_cast<int>(p1);
  constexpr int kStride = (kT / kGroup) * kPix;
  // software pipeline over (trip, j): the 4 loads of step i+1 are issued before the arithmetic of step i
  auto pixel = [&](int pb_, int u) { return min(pb_ + u, q1 - 1); };   // clamped: a tail pixel is recomputed, never stored
  uint4 xn[kPix];
  int pb = q0 + grp * kPix;
  if (pb < q1) {
#pragma unroll
    for (int u = 0; u < kPix; ++u) xn[u] = ldg_stream16(raw + static_cast<unsigned>(pixel(pb, u) * C + l * V));
  }
  for (; pb < q1; pb += kStride) {
    float nz[kPix];
    unsigned po[kPix];                // element offset of the pixel's channel 0 inside the sample
#pragma unroll
    for (int u = 0; u < kPix; ++u) {
      const int px = pixel(pb, u);
      po[u] = static_cast<unsigned>(px) * static_cast<unsigned>(C);
      nz[u] = noise_n ? nw * __ldg(noise_n + px) : 0.f;
    }
    float acc[kPix][3];
#pragma unroll
    for (int u = 0; u < kPix; ++u) acc[u][0] = acc[u][1] = acc[u][2] = 0.f;
    for (int j = 0; j < J; ++j) {
      const int v = l + kGroup * j;
      uint4 xr[kPix];
#pragma unroll
      for (int u = 0; u < kPix; ++u) xr[u] = xn[u];
      {  // prefetch the next step: (pb, j+1) or (pb + stride, 0)
        const bool wrap = (j + 1 == J);
        const int pbn = wrap ? pb + kStride : pb;
        const int vn = wrap ? l : v + kGroup;
        if (pbn < q1) {
#pragma unroll
          for (int u = 0; u < kPix; ++u) xn[u] = ldg_stream16(raw + static_cast<unsigned>(pixel(pbn, u) * C + vn * V));
        }
      }
      float d[V], b[V], s[V], w0[V], w1[V], w2[V];
#pragma unroll
      for (int q = 0; q < Q; ++q) {
        const float4 dv = c4[q * nvec + v], bv = c4[c4_plane + q * nvec + v], sv = c4[2 * c4_plane + q * nvec + v];
        d[4 * q] = dv.x; d[4 * q + 1] = dv.y; d[4 * q + 2] = dv.z; d[4 * q + 3] = dv.w;
        b[4 * q] = bv.x; b[4 * q + 1] = bv.y; b[4 * q + 2] = bv.z; b[4 * q + 3] = bv.w;
        s[4 * q] = sv.x; s[4 * q + 1] = sv.y; s[4 * q + 2] = sv.z; s[4 * q + 3] = sv.w;
        if (p.rgb) {
          const float4 a0 = c4[3 * c4_plane + q * nvec + v], a1 = c4[4 * c4_plane + q * nvec + v], a2 = c4[5 * c4_plane + q * nvec + v];
          w0[4 * q] = a0.x; w0[4 * q + 1] = a0.y; w0[4 * q + 2] = a0.z; w0[4 * q + 3] = a0.w;
          w1[4 * q] = a1.x; w1[4 * q + 1] = a1.y; w1[4 * q + 2] = a1.z; w1[4 * q + 3] = a1.w;
          w2[4 * q] = a2.x; w2[4 * q + 1] = a2.y; w2[4 * q + 2] = a2.z; w2[4 * q + 3] = a2.w;
        }
      }
#pragma unroll
      for (int u = 0; u < kPix; ++u) {
        float x[V], o[V], o2[V];
        ChanVec<T>::unpack(xr[u], x);
#pragma unroll
        for (int k = 0; k < V; ++k) {
          float t = fmaf(x[k], d[k], b[k] + nz[u]);
          t = fast ? fmaxf(t, t * neg) : (t > 0.f ? t : t * neg) * p.gain;
          o[k] = t;
          o2[k] = t * s[k];
        }
        if (p.rgb) {
#pragma unroll
          for (int k = 0; k < V; ++k) {
            acc[u][0] = fmaf(w0[k], o[k], acc[u][0]);
            acc[u][1] = fmaf(w1[k], o[k], acc[u][1]);
            acc[u][2] = fmaf(w2[k], o[k], acc[u][2]);
          }
        }
        uint32_t word = 0u;
        if (MASK) word = sign_word<V>(sign_bits<T>(o), l, gmask);
        if (pb + u < q1) {
          const unsigned off = po[u] + static_cast<unsigned>(v * V);
          if (MASK) {
            if ((l * V & 31) == 0) mask[off >> 5] = word;
          } else if (out) {
            stg_stream16(out + off, ChanVec<T>::pack(o));
          }
          if (xs) stg_stream16(xs + off, ChanVec<T>::pack(o2));
        }
      }
    }
    if (p.rgb) {
#pragma unroll
      for (int m = kGroup / 2; m >= 1; m >>= 1)
#pragma unroll
        for (int u = 0; u < kPix; ++u)
#pragma unroll
          for (int o = 0; o < 3; ++o) acc[u][o] += __shfl_xor_sync(gmask, acc[u][o], m);
      if (l < 3) {                                         // lane o of the group stores output plane o
        const int o = l;
        const float rb = p.rgb_bias ? __ldg(p.rgb_bias + o) : 0.f;
        const int64_t off = (n * 3 + o) * p.hw + pb;
#pragma unroll
        for (int u = 0; u < kPix; ++u)
          if (pb + u < q1) {
            const float r = (o == 0 ? acc[u][0] : o == 1 ? acc[u][1] : acc[u][2]) + rb;
            p.rgb[off + u] = r + (p.skip ? __ldg(p.skip + off + u) : 0.f);
          }
      }
    }
  }
}

struct TailBwdParams {
  void* g_raw; float* partial;
  const void* g_xs; const void* out; const void* raw;   // MASK: `out` is the forward pass's sign mask
  const float* s_next; const float* demod; const float* g_rgb; const float* wm;
  float alpha, gain;
  int C;
  int64_t hw;
  int chunk, chunks_per_sample;
  int r_ds, r_dd, r_gw, n_red;      // rows of the reduction block (-1: absent): d_s_next, d_demod, d_wm[3]
};

// Thread = (channel vector, pixel lane): a thread keeps its V channels for the whole chunk, so the per-channel sums live in
// registers; they are combined across the CTA's pixel lanes through shared memory into one partial block per CTA.
// MASK: lrelu' comes from the sign mask; nothing is reduced, so neither the activation nor `raw` is read.
template <typename T, bool MASK>
__global__ void __launch_bounds__(kT, 2)
styled_tail_bwd_nhwc_kernel(const TailBwdParams p) {
  constexpr int V = ChanVec<T>::V;
  constexpr int U = (V == 4) ? 4 : 2;   // pixels in flight per thread: 3 x 16-byte loads each (register budget: 2 CTAs/SM)
  extern __shared__ float red[];                          // [pixel lanes][n_red][C]
  const int C = p.C, cv = C / V;
  const int64_t n = blockIdx.x / p.chunks_per_sample;
  const int ck = blockIdx.x - n * p.chunks_per_sample;
  const int64_t p0 = static_cast<int64_t>(ck) * p.chunk, p1 = min(p0 + p.chunk, p.hw);
  const int lanes_p = kT / cv > 0 ? kT / cv : 1;
  const int cq = threadIdx.x % cv, pl = threadIdx.x / cv;
  float a_ds[V], a_dd[V], a_g0[V], a_g1[V], a_g2[V];
#pragma unroll
  for (int k = 0; k < V; ++k) a_ds[k] = a_dd[k] = a_g0[k] = a_g1[k] = a_g2[k] = 0.f;
  const T* gxs = static_cast<const T*>(p.g_xs);
  const T* outp = static_cast<const T*>(p.out);
  const uint32_t* maskp = static_cast<const uint32_t*>(p.out) + n * p.hw * (C >> 5);     // this sample's words
  const int mw = C >> 5;
  auto load_out = [&](int64_t pu, int64_t off) {      // the activation vector, or (MASK) its V sign bits in .x
    return MASK ? make_uint4(sign_load<V>(maskp + pu * mw, cq), 0u, 0u, 0u) : ldg_stream16(outp + off);
  };
  const T* rawp = static_cast<const T*>(p.raw);
  T* graw = static_cast<T*>(p.g_raw);
  if (pl < lanes_p) {
    float sv[V], dv[V], w0[V], w1[V], w2[V];
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const int c = cq * V + k;
      sv[k] = p.s_next ? __ldg(p.s_next + n * C + c) : 1.f;
      dv[k] = p.demod ? __ldg(p.demod + n * C + c) : 1.f;
      w0[k] = p.g_rgb ? __ldg(p.wm + (n * 3 + 0) * C + c) : 0.f;
      w1[k] = p.g_rgb ? __ldg(p.wm + (n * 3 + 1) * C + c) : 0.f;
      w2[k] = p.g_rgb ? __ldg(p.wm + (n * 3 + 2) * C + c) : 0.f;
    }
    const float* g0 = p.g_rgb ? p.g_rgb + n * 3 * p.hw : nullptr;
    const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
    auto body = [&](int64_t off, const uint4 gr, const uint4 orw, const uint4 rr, float s0, float s1, float s2) {
      float g[V], o[V], r[V], gt[V];
      ChanVec<T>::unpack(gr, g);
      if (!MASK) ChanVec<T>::unpack(orw, o);
      ChanVec<T>::unpack(rr, r);
#pragma unroll
      for (int k = 0; k < V; ++k) {
        float go = g[k] * sv[k];
        if (p.g_rgb) go = fmaf(w2[k], s2, fmaf(w1[k], s1, fmaf(w0[k], s0, go)));
        const bool pos = MASK ? ((orw.x >> k) & 1u) != 0u : o[k] > 0.f;
        const float t = (pos ? go : go * p.alpha) * p.gain;
        gt[k] = t * dv[k];
        if (!MASK) {
          a_ds[k] = fmaf(g[k], o[k], a_ds[k]);
          a_dd[k] = fmaf(t, r[k], a_dd[k]);
          a_g0[k] = fmaf(s0, o[k], a_g0[k]);
          a_g1[k] = fmaf(s1, o[k], a_g1[k]);
          a_g2[k] = fmaf(s2, o[k], a_g2[k]);
        }
      }
      *reinterpret_cast<uint4*>(graw + off) = ChanVec<T>::pack(gt);
    };
    int64_t pp = p0 + pl;
    for (; pp + (U - 1) * lanes_p < p1; pp += U * lanes_p) {
      uint4 gr[U], orw[U], rr[U];
      float s[U][3];
      int64_t off[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t pu = pp + u * lanes_p;
        off[u] = ((n * p.hw + pu) * cv + cq) * V;
        orw[u] = load_out(pu, off[u]);
        gr[u] = gxs ? ldg_stream16(gxs + off[u]) : zero;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t pu = pp + u * lanes_p;
        rr[u] = rawp ? ldg_stream16(rawp + off[u]) : zero;
        s[u][0] = g0 ? __ldg(g0 + pu) : 0.f;
        s[u][1] = g0 ? __ldg(g0 + p.hw + pu) : 0.f;
        s[u][2] = g0 ? __ldg(g0 + 2 * p.hw + pu) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) body(off[u], gr[u], orw[u], rr[u], s[u][0], s[u][1], s[u][2]);
    }
    for (; pp < p1; pp += lanes_p) {
      const int64_t off = ((n * p.hw + pp) * cv + cq) * V;
      body(off, gxs ? ldg_stream16(gxs + off) : zero, load_out(pp, off), rawp ? ldg_stream16(rawp + off) : zero,
           g0 ? __ldg(g0 + pp) : 0.f, g0 ? __ldg(g0 + p.hw + pp) : 0.f, g0 ? __ldg(g0 + 2 * p.hw + pp) : 0.f);
    }
  }
  if (!MASK && p.partial && p.n_red > 0) {
    const int R = p.n_red;
    if (pl < lanes_p) {
      float* row = red + static_cast<int64_t>(pl) * R * C + cq * V;
#pragma unroll
      for (int k = 0; k < V; ++k) {
        if (p.r_ds >= 0) row[p.r_ds * C + k] = a_ds[k];
        if (p.r_dd >= 0) row[p.r_dd * C + k] = a_dd[k];
        if (p.r_gw >= 0) { row[p.r_gw * C + k] = a_g0[k]; row[(p.r_gw + 1) * C + k] = a_g1[k]; row[(p.r_gw + 2) * C + k] = a_g2[k]; }
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < R * C; i += kT) {
      float t = 0.f;
      for (int q = 0; q < lanes_p; ++q) t += red[static_cast<int64_t>(q) * R * C + i];
      p.partial[static_cast<int64_t>(blockIdx.x) * R * C + i] = t;
    }
  }
}

// pixels per CTA of the forward kernel: a multiple of the 128 pixels one trip covers, ~8 CTAs per SM over the batch
int64_t fwd_chunk(int64_t N, int64_t HW) {
  const int64_t trip = (kT / kGroup) * kPix;
  const int64_t target = 8LL * sm_count();
  int64_t k = (target + N - 1) / N;
  const int64_t kmax = (HW + trip - 1) / trip;
  if (k > kmax) k = kmax;
  if (k < 1) k = 1;
  return ((HW + k - 1) / k + trip - 1) / trip * trip;
}

int64_t bwd_chunk(int64_t N, int cv, int64_t HW) {
  const int lanes_p = kT / cv > 0 ? kT / cv : 1;
  const int64_t target = 8LL * sm_count();
  int64_t k = (target + N - 1) / N;
  const int64_t kmax = (HW + 4 * lanes_p - 1) / (4 * lanes_p);
  if (k > kmax) k = kmax;
  if (k < 1) k = 1;
  return (HW + k - 1) / k;
}

}  // namespace
}  // namespace gg

using namespace gg;

// `out_is_mask`: `out` receives the sign mask (N, HW, C/32) uint32 instead of the activation.
static int launch_tail_fwd(const char* who, void* out, bool out_is_mask, void* xs, float* rgb, const void* raw,
                           const float* noise, const float* noise_weight, const float* bias, const float* demod,
                           const float* s_next, const float* wm, const float* rgb_bias, const float* skip, int dtype, int act,
                           float alpha, float scale, int64_t N, int C, int64_t HW, void* stream) {
  if (N < 0 || C < 0 || HW < 0) return fail(GG_ERR_BAD_ARG, "%s: negative size", who);
  if (dtype != GG_F32 && dtype != GG_BF16) return fail(GG_ERR_UNSUPPORTED, "%s: dtype %d not supported (fp32 or bf16)", who, dtype);
  if (act != 1 && act != 3) return fail(GG_ERR_UNSUPPORTED, "%s: act must be 1 (linear) or 3 (lrelu)", who);
  if (N * HW * C == 0) return GG_OK;
  const int V = dtype == GG_BF16 ? 8 : 4;
  if (C % (V * kGroup) != 0 || C > 2048) return fail(GG_ERR_UNSUPPORTED, "%s: C must be a multiple of %d, <= 2048", who, V * kGroup);
  if (!raw || (!out && !xs && !rgb)) return fail(GG_ERR_BAD_ARG, "%s: null tensor", who);
  if (out_is_mask && !out) return fail(GG_ERR_BAD_ARG, "%s: null mask", who);
  if (xs && !s_next) return fail(GG_ERR_BAD_ARG, "%s: xs needs s_next", who);
  if (rgb && !wm) return fail(GG_ERR_BAD_ARG, "%s: rgb needs wm", who);
  const int64_t chunk = fwd_chunk(N, HW);
  if (chunk > 0x7fffff00LL || HW * C >= 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "%s: plane too large (H*W*C must be < 2^31)", who);
  const int K = static_cast<int>((HW + chunk - 1) / chunk);
  const int64_t grid = N * K;
  if (grid > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "%s: too many CTAs", who);
  TailFwdParams p;
  p.raw = raw; p.out = out; p.xs = xs; p.rgb = rgb; p.skip = rgb ? skip : nullptr;
  p.noise = noise; p.noise_weight = noise_weight; p.bias = bias; p.demod = demod; p.s_next = s_next;
  p.wm = wm; p.rgb_bias = rgb_bias; p.alpha = alpha; p.gain = scale; p.act = act; p.C = C; p.hw = HW;
  p.chunk = static_cast<int>(chunk); p.chunks_per_sample = K;
  const size_t smem = static_cast<size_t>(6) * C * sizeof(float);
  auto st = static_cast<cudaStream_t>(stream);
  const bool fast = p.gain > 0.f && ((p.act == 3 && p.alpha >= 0.f && p.alpha <= 1.f) || p.act == 1);
  const unsigned g = static_cast<unsigned>(grid);
#define GG_TAIL(T_, F_)                                                                   \
  do {                                                                                    \
    if (out_is_mask) styled_tail_nhwc_kernel<T_, F_, true><<<g, kT, smem, st>>>(p);       \
    else styled_tail_nhwc_kernel<T_, F_, false><<<g, kT, smem, st>>>(p);                  \
  } while (0)
  if (dtype == GG_F32) { if (fast) GG_TAIL(float, true); else GG_TAIL(float, false); }
  else { if (fast) GG_TAIL(__nv_bfloat16, true); else GG_TAIL(__nv_bfloat16, false); }
#undef GG_TAIL
  GG_CHECK_LAUNCH("styled_tail_nhwc launch");
  return GG_OK;
}

extern "C" {

int gg_styled_tail_nhwc(void* out, void* xs, float* rgb, const void* raw, const float* noise, const float* noise_weight,
                        const float* bias, const float* demod, const float* s_next, const float* wm, const float* rgb_bias,
                        const float* skip, int dtype, int act, float alpha, float scale, int64_t N, int C, int64_t HW,
                        void* stream) {
  return launch_tail_fwd("styled_tail_nhwc", out, false, xs, rgb, raw, noise, noise_weight, bias, demod, s_next, wm, rgb_bias,
                         skip, dtype, act, alpha, scale, N, C, HW, stream);
}

int gg_styled_tail_mask_nhwc(void* mask, void* xs, float* rgb, const void* raw, const float* noise, const float* noise_weight,
                             const float* bias, const float* demod, const float* s_next, const float* wm,
                             const float* rgb_bias, const float* skip, int dtype, int act, float alpha, float scale, int64_t N,
                             int C, int64_t HW, void* stream) {
  return launch_tail_fwd("styled_tail_mask_nhwc", mask, true, xs, rgb, raw, noise, noise_weight, bias, demod, s_next, wm,
                         rgb_bias, skip, dtype, act, alpha, scale, N, C, HW, stream);
}

int64_t gg_styled_tail_backward_workspace(int dtype, int64_t N, int C, int64_t HW) {
  if (N <= 0 || C <= 0 || HW <= 0) return 0;
  const int V = dtype == GG_BF16 ? 8 : 4;
  if (C % V != 0) return 0;
  const int64_t chunk = bwd_chunk(N, C / V, HW);
  return N * ((HW + chunk - 1) / chunk) * 5 * C * static_cast<int64_t>(sizeof(float));
}

int gg_styled_tail_backward_nhwc(void* g_raw, float* d_s_next, float* d_demod, float* d_wm, void* workspace,
                                 const void* g_xs, const float* g_rgb, const void* out_saved, const void* raw,
                                 const float* s_next, const float* demod, const float* wm, int dtype, float alpha,
                                 float scale, int64_t N, int C, int64_t HW, int64_t reduce_pitch, void* stream) {
  if (N < 0 || C < 0 || HW < 0) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_nhwc: negative size");
  if (dtype != GG_F32 && dtype != GG_BF16) return fail(GG_ERR_UNSUPPORTED, "styled_tail_backward_nhwc: dtype %d not supported", dtype);
  // rows of the reduction block: d_s_next, d_demod, d_wm[3] (each present only when requested)
  int r = 0;
  const int r_ds = d_s_next ? r++ : -1;
  const int r_dd = d_demod ? r++ : -1;
  const int r_gw = d_wm ? r : -1;
  if (d_wm) r += 3;
  if (r > 0 && reduce_pitch != C && reduce_pitch != 0 && reduce_pitch != r * C)
    return fail(GG_ERR_BAD_ARG, "styled_tail_backward_nhwc: reduce_pitch must be C (separate dense outputs) or r*C (packed block)");
  // the caller's destinations are slices of one (N, r, C) block when they are laid out that way (the Python face allocates
  // them so); otherwise each is a dense (N, rows, C) tensor of its own
  float* first = d_s_next ? d_s_next : (d_demod ? d_demod : d_wm);
  const bool packed = r > 0 && (!d_s_next || d_s_next == first + static_cast<int64_t>(r_ds) * C) &&
                      (!d_demod || d_demod == first + static_cast<int64_t>(r_dd) * C) &&
                      (!d_wm || d_wm == first + static_cast<int64_t>(r_gw) * C) && reduce_pitch == r * C;
  auto st = static_cast<cudaStream_t>(stream);
  if (N * HW * C == 0) {
    if (r > 0 && N * C > 0) {   // a sum over no pixels is 0
      cudaError_t e = cudaSuccess;
      if (packed) {
        e = cudaMemsetAsync(first, 0, N * r * C * sizeof(float), st);
      } else {
        if (d_s_next && e == cudaSuccess) e = cudaMemsetAsync(d_s_next, 0, N * C * sizeof(float), st);
        if (d_demod && e == cudaSuccess) e = cudaMemsetAsync(d_demod, 0, N * C * sizeof(float), st);
        if (d_wm && e == cudaSuccess) e = cudaMemsetAsync(d_wm, 0, N * 3 * C * sizeof(float), st);
      }
      if (e != cudaSuccess) return cuda_fail(e, "styled_tail_backward_nhwc memset");
    }
    return GG_OK;
  }
  const int V = dtype == GG_BF16 ? 8 : 4;
  if (C % V != 0 || C / V > kT) return fail(GG_ERR_UNSUPPORTED, "styled_tail_backward_nhwc: C must be a multiple of %d, <= %d", V, V * kT);
  if (!g_raw || !out_saved || (!g_xs && !g_rgb)) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_nhwc: null tensor");
  if (g_xs && !s_next) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_nhwc: g_xs needs s_next");
  if (g_rgb && !wm) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_nhwc: g_rgb needs wm");
  if (d_s_next && !g_xs) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_nhwc: d_s_next needs g_xs");
  if (d_demod && !raw) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_nhwc: d_demod needs raw");
  if (d_wm && !g_rgb) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_nhwc: d_wm needs g_rgb");
  if ((d_s_next || d_demod || d_wm) && !workspace) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_nhwc: reductions need a workspace");
  const int cv = C / V;
  const int64_t chunk64 = bwd_chunk(N, cv, HW);
  if (chunk64 > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_nhwc: plane too large");
  const int K = static_cast<int>((HW + chunk64 - 1) / chunk64);
  const int64_t grid = N * K;
  if (grid > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_nhwc: too many CTAs");
  TailBwdParams p;
  p.g_raw = g_raw; p.partial = static_cast<float*>(workspace); p.g_xs = g_xs; p.out = out_saved;
  p.raw = d_demod ? raw : nullptr; p.s_next = s_next; p.demod = demod; p.g_rgb = g_rgb; p.wm = wm;
  p.alpha = alpha; p.gain = scale; p.C = C; p.hw = HW; p.chunk = static_cast<int>(chunk64); p.chunks_per_sample = K;
  p.r_ds = r_ds; p.r_dd = r_dd; p.r_gw = r_gw; p.n_red = r;
  const int lanes_p = kT / cv > 0 ? kT / cv : 1;
  const size_t smem = static_cast<size_t>(lanes_p) * (r > 0 ? r : 1) * C * sizeof(float);
  if (smem > 48 * 1024) {
    static DeviceOnce configured;
    if (configured.needed()) {
      cudaError_t e = cudaFuncSetAttribute(styled_tail_bwd_nhwc_kernel<float, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
      if (e == cudaSuccess)
        e = cudaFuncSetAttribute(styled_tail_bwd_nhwc_kernel<__nv_bfloat16, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
      if (e != cudaSuccess) return cuda_fail(e, "styled_tail_backward_nhwc smem opt-in");
      configured.done();
    }
    if (smem > 100 * 1024) return fail(GG_ERR_UNSUPPORTED, "styled_tail_backward_nhwc: C too large for the reduction stage");
  }
  if (dtype == GG_F32) styled_tail_bwd_nhwc_kernel<float, false><<<static_cast<unsigned>(grid), kT, smem, st>>>(p);
  else styled_tail_bwd_nhwc_kernel<__nv_bfloat16, false><<<static_cast<unsigned>(grid), kT, smem, st>>>(p);
  GG_CHECK_LAUNCH("styled_tail_backward_nhwc launch");
  if (r > 0) {
    // partial is [N][K][r*C]: ONE finish launch writes every requested sum of a packed block; otherwise one launch per sum
    if (packed) {
      nhwc_finish_kernel<<<static_cast<unsigned>(N * ((r * C + 31) / 32)), dim3(32, 32), 0, st>>>(
          first, static_cast<const float*>(workspace), N, K, r * C, r * C);
    } else {
      auto finish_row = [&](float* dst, int row, int rows_n) {
        nhwc_finish_kernel<<<static_cast<unsigned>(N * ((rows_n * C + 31) / 32)), dim3(32, 32), 0, st>>>(
            dst, static_cast<const float*>(workspace) + static_cast<int64_t>(row) * C, N, K, rows_n * C, r * C);
      };
      if (d_s_next) finish_row(d_s_next, p.r_ds, 1);
      if (d_demod) finish_row(d_demod, p.r_dd, 1);
      if (d_wm) finish_row(d_wm, p.r_gw, 3);
    }
    GG_CHECK_LAUNCH("styled_tail_backward_nhwc finish launch");
  }
  return GG_OK;
}

int gg_styled_tail_backward_mask_nhwc(void* g_raw, const void* g_xs, const float* g_rgb, const void* mask,
                                      const float* s_next, const float* demod, const float* wm, int dtype, float alpha,
                                      float scale, int64_t N, int C, int64_t HW, void* stream) {
  if (N < 0 || C < 0 || HW < 0) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_mask_nhwc: negative size");
  if (dtype != GG_F32 && dtype != GG_BF16) return fail(GG_ERR_UNSUPPORTED, "styled_tail_backward_mask_nhwc: dtype %d not supported", dtype);
  if (N * HW * C == 0) return GG_OK;
  const int V = dtype == GG_BF16 ? 8 : 4;
  if (C % 32 != 0 || C / V > kT) return fail(GG_ERR_UNSUPPORTED, "styled_tail_backward_mask_nhwc: C must be a multiple of 32, <= %d", V * kT);
  if (!g_raw || !mask || (!g_xs && !g_rgb)) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_mask_nhwc: null tensor");
  if (g_xs && !s_next) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_mask_nhwc: g_xs needs s_next");
  if (g_rgb && !wm) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_mask_nhwc: g_rgb needs wm");
  const int64_t chunk64 = bwd_chunk(N, C / V, HW);
  if (chunk64 > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_mask_nhwc: plane too large");
  const int K = static_cast<int>((HW + chunk64 - 1) / chunk64);
  const int64_t grid = N * K;
  if (grid > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "styled_tail_backward_mask_nhwc: too many CTAs");
  TailBwdParams p;
  p.g_raw = g_raw; p.partial = nullptr; p.g_xs = g_xs; p.out = mask; p.raw = nullptr; p.s_next = s_next; p.demod = demod;
  p.g_rgb = g_rgb; p.wm = wm; p.alpha = alpha; p.gain = scale; p.C = C; p.hw = HW; p.chunk = static_cast<int>(chunk64);
  p.chunks_per_sample = K; p.r_ds = p.r_dd = p.r_gw = -1; p.n_red = 0;
  auto st = static_cast<cudaStream_t>(stream);
  if (dtype == GG_F32) styled_tail_bwd_nhwc_kernel<float, true><<<static_cast<unsigned>(grid), kT, 0, st>>>(p);
  else styled_tail_bwd_nhwc_kernel<__nv_bfloat16, true><<<static_cast<unsigned>(grid), kT, 0, st>>>(p);
  GG_CHECK_LAUNCH("styled_tail_backward_mask_nhwc launch");
  return GG_OK;
}

}  // extern "C"
