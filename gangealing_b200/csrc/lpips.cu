// lpips.cu -- the perceptual loss's front end on channels-last feature maps (sm_90a), SURVEY.md 8(f) rank 2.
//
// reference: models/losses/lpips.py:26-28 (`normalize_tensor`: f / (sqrt(sum_c f^2) + 1e-10)), :193-195
// (`diffs = (feats0 - feats1)**2`), :197-205 (`lins[kk](diffs)` = per-channel weights, or `.sum(dim=1)`), :226
// (`spatial_average` = mean over H, W).  The reference spends ~14 ATen passes per VGG layer forward (and ~25 backward)
// on five feature maps x two images every step; here ONE pass forward (reads both maps) and ONE pass backward
// (reads both maps, writes both gradients):
//     d[n] = 1/HW * sum_p sum_c w[c] * (a[n,p,c]/(|a[n,p,:]|+eps) - b[n,p,c]/(|b[n,p,:]|+eps))^2
// Feature maps are stored fp32 or bf16 (`dtype`; BASELINE config 3 runs the VGG in bf16); arithmetic and the result are fp32.
// A group of L = min(32, C/4) lanes owns one pixel: every lane keeps its channel quads of both maps in registers
// (<= 8 independent 128-bit loads in flight), the per-pixel sums are butterfly reductions inside the group, and the
// difference is formed from the normalised values themselves (no |a|^2 + |b|^2 - 2ab cancellation).
#include "common.cuh"

namespace gg {
namespace {

constexpr int kT = 256;
constexpr int kMaxTrips = 8;     // C <= 4 * 32 * 8 = 1024

// 4 consecutive channels of a feature map as fp32 (storage: fp32 -> one 16-byte access, bf16 -> one 8-byte access)
__device__ __forceinline__ float4 ld4(const float* base, int64_t quad) { return __ldcs(reinterpret_cast<const float4*>(base) + quad); }
__device__ __forceinline__ float4 ld4(const __nv_bfloat16* base, int64_t quad) {
  const uint2 u = __ldcs(reinterpret_cast<const uint2*>(base) + quad);
  return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                     __uint_as_float(u.y & 0xffff0000u));
}
__device__ __forceinline__ void st4(float* base, int64_t quad, const float4 v) { reinterpret_cast<float4*>(base)[quad] = v; }
__device__ __forceinline__ void st4(__nv_bfloat16* base, int64_t quad, const float4 v) {
  reinterpret_cast<uint2*>(base)[quad] = make_uint2(ChanVec<__nv_bfloat16>::pack2(v.x, v.y), ChanVec<__nv_bfloat16>::pack2(v.z, v.w));
}

template <int L>
__device__ __forceinline__ float group_sum(float v, unsigned mask) {
#pragma unroll
  for (int m = L / 2; m >= 1; m >>= 1) v += __shfl_xor_sync(mask, v, m);
  return v;
}

// TRIPS channel quads per lane (compile time): registers, no local memory.
template <typename T, int L, int TRIPS, bool BACKWARD>
__global__ void __launch_bounds__(kT)
feature_distance_kernel(float* __restrict__ partial, T* __restrict__ g0, T* __restrict__ g1,
                        const float* __restrict__ gout, const T* __restrict__ f0, const T* __restrict__ f1,
                        const float* __restrict__ w, int c4, int64_t hw, int chunk, int chunks_per_sample, float eps,
                        float inv_hw) {
  __shared__ float red[kT / 32];
  const int64_t n = blockIdx.x / chunks_per_sample;
  const int ck = blockIdx.x - n * chunks_per_sample;
  const int64_t p0 = static_cast<int64_t>(ck) * chunk, p1 = min(p0 + chunk, hw);
  constexpr int GROUPS = kT / L;                    // pixels in flight per CTA
  const int l = threadIdx.x % L, grp = threadIdx.x / L;
  const int lane = threadIdx.x & 31;
  const unsigned gmask = (L == 32) ? 0xffffffffu : (((1u << L) - 1u) << (lane / L * L));
  float4 wq[TRIPS];
#pragma unroll
  for (int t = 0; t < TRIPS; ++t)
    wq[t] = w ? __ldg(reinterpret_cast<const float4*>(w) + l + t * L) : make_float4(1.f, 1.f, 1.f, 1.f);
  const float gs = BACKWARD ? 2.f * __ldg(gout + n) * inv_hw : 0.f;
  float acc = 0.f;
  for (int64_t p = p0 + grp; p < p1; p += GROUPS) {
    const int64_t base = (n * hw + p) * c4;
    float4 a[TRIPS], b[TRIPS];
#pragma unroll
    for (int t = 0; t < TRIPS; ++t) a[t] = ld4(f0, base + l + t * L);
#pragma unroll
    for (int t = 0; t < TRIPS; ++t) b[t] = ld4(f1, base + l + t * L);
    float saa = 0.f, sbb = 0.f;
#pragma unroll
    for (int t = 0; t < TRIPS; ++t) {
      saa = fmaf(a[t].x, a[t].x, fmaf(a[t].y, a[t].y, fmaf(a[t].z, a[t].z, fmaf(a[t].w, a[t].w, saa))));
      sbb = fmaf(b[t].x, b[t].x, fmaf(b[t].y, b[t].y, fmaf(b[t].z, b[t].z, fmaf(b[t].w, b[t].w, sbb))));
    }
    saa = group_sum<L>(saa, gmask);
    sbb = group_sum<L>(sbb, gmask);
    const float ra = sqrtf(saa), rb = sqrtf(sbb);
    const float ia = 1.f / (ra + eps), ib = 1.f / (rb + eps);
    if (!BACKWARD) {
      float d = 0.f;
#pragma unroll
      for (int t = 0; t < TRIPS; ++t) {
        const float dx = a[t].x * ia - b[t].x * ib, dy = a[t].y * ia - b[t].y * ib;
        const float dz = a[t].z * ia - b[t].z * ib, dw = a[t].w * ia - b[t].w * ib;
        d = fmaf(wq[t].x * dx, dx, fmaf(wq[t].y * dy, dy, fmaf(wq[t].z * dz, dz, fmaf(wq[t].w * dw, dw, d))));
      }
      acc += d;                                     // lanes of a group hold partial sums; reduced once per CTA
    } else {
      // t_c = w_c (a^_c - b^_c);  Pa = sum t_c a_c;  Pb = sum t_c b_c
      float4 tq[TRIPS];
      float pa = 0.f, pb = 0.f;
#pragma unroll
      for (int t = 0; t < TRIPS; ++t) {
        tq[t].x = wq[t].x * (a[t].x * ia - b[t].x * ib); tq[t].y = wq[t].y * (a[t].y * ia - b[t].y * ib);
        tq[t].z = wq[t].z * (a[t].z * ia - b[t].z * ib); tq[t].w = wq[t].w * (a[t].w * ia - b[t].w * ib);
        pa = fmaf(tq[t].x, a[t].x, fmaf(tq[t].y, a[t].y, fmaf(tq[t].z, a[t].z, fmaf(tq[t].w, a[t].w, pa))));
        pb = fmaf(tq[t].x, b[t].x, fmaf(tq[t].y, b[t].y, fmaf(tq[t].z, b[t].z, fmaf(tq[t].w, b[t].w, pb))));
      }
      pa = group_sum<L>(pa, gmask);
      pb = group_sum<L>(pb, gmask);
      // d a^_c / d a_k = delta_ck * ia - a_c a_k * ia^2 / ra.  At an all-zero pixel the reference's autograd yields
      // nan (sqrt'(0) * 0 = inf * 0); the gradient of that pixel is DEFINED as 0 here (a dead pixel gets no signal).
      const float ka = ra > 0.f ? pa * ia * ia / ra : 0.f;
      const float kb = rb > 0.f ? pb * ib * ib / rb : 0.f;
      const float gsa = ra > 0.f ? gs : 0.f, gsb = rb > 0.f ? gs : 0.f;
#pragma unroll
      for (int t = 0; t < TRIPS; ++t) {
        float4 o;
        if (g0) {
          o.x = gsa * (tq[t].x * ia - a[t].x * ka); o.y = gsa * (tq[t].y * ia - a[t].y * ka);
          o.z = gsa * (tq[t].z * ia - a[t].z * ka); o.w = gsa * (tq[t].w * ia - a[t].w * ka);
          st4(g0, base + l + t * L, o);
        }
        if (g1) {
          o.x = -gsb * (tq[t].x * ib - b[t].x * kb); o.y = -gsb * (tq[t].y * ib - b[t].y * kb);
          o.z = -gsb * (tq[t].z * ib - b[t].z * kb); o.w = -gsb * (tq[t].w * ib - b[t].w * kb);
          st4(g1, base + l + t * L, o);
        }
      }
    }
  }
  if (!BACKWARD) {
    acc = warp_sum(acc);
    if (lane == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
#pragma unroll
      for (int i = 0; i < kT / 32; ++i) t += red[i];
      partial[blockIdx.x] = t * inv_hw;
    }
  }
}

__global__ void distance_finish_kernel(float* __restrict__ out, const float* __restrict__ partial, int64_t N, int K) {
  const int64_t n = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float t = 0.f;
  for (int k = 0; k < K; ++k) t += partial[n * K + k];
  out[n] = t;
}

int64_t distance_chunk(int64_t N, int64_t HW, int groups) {
  const int64_t target = 8LL * sm_count();
  int64_t k = (target + N - 1) / N;
  const int64_t kmax = (HW + 2 * groups - 1) / (2 * groups);
  if (k > kmax) k = kmax;
  if (k > 64) k = 64;                      // the finish kernel sums K partials serially
  if (k < 1) k = 1;
  return (HW + k - 1) / k;
}

template <typename T, bool BACKWARD>
int launch_distance(float* partial, T* g0, T* g1, const float* gout, const T* f0, const T* f1,
                    const float* w, int64_t N, int C, int64_t HW, float eps, cudaStream_t st, int* k_out) {
  const int c4 = C / 4;
  const int L = c4 >= 32 ? 32 : c4;         // c4 is a power of two here when < 32 (checked by the caller)
  const int trips = c4 / L;
  const int64_t chunk64 = distance_chunk(N, HW, kT / L);
  const int chunk = static_cast<int>(chunk64);
  const int K = static_cast<int>((HW + chunk - 1) / chunk);
  if (k_out) *k_out = K;
  const unsigned grid = static_cast<unsigned>(N * K);
  const float inv_hw = 1.f / static_cast<float>(HW);
#define GG_DIST(L_, T_)                                                                                          \
  feature_distance_kernel<T, L_, T_, BACKWARD><<<grid, kT, 0, st>>>(partial, g0, g1, gout, f0, f1, w, c4, HW, chunk, K, \
                                                                 eps, inv_hw)
  if (L == 32) {
    switch (trips) {
      case 1: GG_DIST(32, 1); break;
      case 2: GG_DIST(32, 2); break;
      case 3: GG_DIST(32, 3); break;
      case 4: GG_DIST(32, 4); break;
      case 6: GG_DIST(32, 6); break;
      case 8: GG_DIST(32, 8); break;
      default: return fail(GG_ERR_UNSUPPORTED, "feature_distance: C = %d is not a supported channel count", C);
    }
  } else if (L == 16) { GG_DIST(16, 1); }
  else if (L == 8) { GG_DIST(8, 1); }
  else if (L == 4) { GG_DIST(4, 1); }
  else if (L == 2) { GG_DIST(2, 1); }
  else { GG_DIST(1, 1); }
#undef GG_DIST
  return GG_OK;
}

int check_distance(const char* who, int64_t N, int C, int64_t HW, const float* weight) {
  if (N < 0 || C < 0 || HW < 0) return fail(GG_ERR_BAD_ARG, "%s: negative size", who);
  if (!aligned16(weight)) return fail(GG_ERR_BAD_ARG, "%s: weight must be 16-byte aligned", who);   // read as float4
  if (C % 4 != 0 || C > 4 * 32 * kMaxTrips) return fail(GG_ERR_UNSUPPORTED, "%s: C must be a multiple of 4, <= 1024", who);
  const int c4 = C / 4;
  if (c4 < 32 && (c4 & (c4 - 1)) != 0) return fail(GG_ERR_UNSUPPORTED, "%s: C < 128 must be a power of two", who);
  if (c4 >= 32 && c4 % 32 != 0) return fail(GG_ERR_UNSUPPORTED, "%s: C >= 128 must be a multiple of 128", who);
  if (N * HW > 0 && (HW + 0) > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "%s: plane too large", who);
  return GG_OK;
}

// ------------------------------------------------------------------------------------------------ VGG slice boundary
// Between two VGG16 slices the reference runs Conv2d (cuDNN) -> ReLU -> [tap for the distance] -> MaxPool2d(2, 2) -> Conv2d
// (lpips_backbones.py:106-121 = torchvision features 2-4, 7-9, 14-16, 21-23).  The tap feature map is the largest tensor
// of its slice and ATen walks it four more times: max_pool forward (read y, write pooled + an int64 index map), max_pool
// backward (zero-fill + scatter into a full-size gradient), the add of the two gradients that meet at the tap (distance +
// pool branch), and the ReLU backward.  Here:
//   forward   raw (conv output, no bias) -> y = relu(raw + bias) AND pooled = maxpool2x2(y), one read of raw
//   backward  g_raw = [y > 0] * (g_y + [this pixel is the window's FIRST maximum] * g_pooled)  -- the arg-max is recomputed
//             from the saved y with ATen's rule (scan the window row-major, replace on `>` or NaN: max_pool2d picks the first
//             maximum), so no index map exists; one pass: read y, g_y, g_pooled (1/4), write g_raw
// Thread = one 2x2 window x one 16-byte channel vector (4 fp32 / 8 bf16 channels); fp32 arithmetic.  HBM-bound:
// forward s*N*H*W*C*(1 + 1 + 1/4), backward s*N*H*W*C*(1 + 1 + 1/4 + 1).
// idx -> (channel vector, window x, window y, sample); 32-bit divisions whenever the tensor allows it (64-bit ones cost ~80
// instructions each)
__device__ __forceinline__ void decode_window(int64_t idx, int64_t total, int cv, int Wo, int Ho, int& cq, int& ox, int& oy,
                                              int64_t& n) {
  if (total <= 0xffffffffLL) {
    unsigned t = static_cast<unsigned>(idx);
    unsigned q = t / static_cast<unsigned>(cv);
    cq = static_cast<int>(t - q * static_cast<unsigned>(cv)); t = q;
    q = t / static_cast<unsigned>(Wo);
    ox = static_cast<int>(t - q * static_cast<unsigned>(Wo)); t = q;
    q = t / static_cast<unsigned>(Ho);
    oy = static_cast<int>(t - q * static_cast<unsigned>(Ho));
    n = q;
  } else {
    cq = static_cast<int>(idx % cv);
    int64_t t = idx / cv;
    ox = static_cast<int>(t % Wo); t /= Wo;
    oy = static_cast<int>(t % Ho);
    n = t / Ho;
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
bias_relu_pool_fwd_kernel(T* __restrict__ y, T* __restrict__ pooled, const T* __restrict__ raw, const float* __restrict__ bias,
                          int cv, int H, int W, int64_t total) {
  constexpr int V = ChanVec<T>::V;
  const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int Ho = H >> 1, Wo = W >> 1;
  int cq, ox, oy;
  int64_t n;
  decode_window(idx, total, cv, Wo, Ho, cq, ox, oy, n);
  const int64_t C = static_cast<int64_t>(cv) * V;
  const int64_t p00 = ((n * H + 2 * oy) * W + 2 * ox) * C + static_cast<int64_t>(cq) * V;
  const int64_t off[4] = {p00, p00 + C, p00 + W * C, p00 + W * C + C};
  uint4 in[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) in[j] = ldg_stream16(raw + off[j]);
  float b[V];
#pragma unroll
  for (int q = 0; q < V / 4; ++q) {
    const float4 bq = bias ? __ldg(reinterpret_cast<const float4*>(bias) + cq * (V / 4) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
    b[4 * q] = bq.x; b[4 * q + 1] = bq.y; b[4 * q + 2] = bq.z; b[4 * q + 3] = bq.w;
  }
  float m[V];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float x[V], o[V];
    ChanVec<T>::unpack(in[j], x);
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const float v = x[k] + b[k];
      o[k] = v > 0.f ? v : v * 0.f;          // relu; NaN stays NaN (torch.relu)
    }
    const uint4 packed = ChanVec<T>::pack(o);
    stg_stream16(y + off[j], packed);
    float r[V];
    ChanVec<T>::unpack(packed, r);            // pool the STORED (rounded) values: what a separate max_pool2d would read
#pragma unroll
    for (int k = 0; k < V; ++k) m[k] = (j == 0 || r[k] > m[k] || r[k] != r[k]) ? r[k] : m[k];
  }
  stg_stream16(pooled + ((n * Ho + oy) * Wo + ox) * C + static_cast<int64_t>(cq) * V, ChanVec<T>::pack(m));
}

template <typename T>
__global__ void __launch_bounds__(256)
bias_relu_pool_bwd_kernel(T* __restrict__ g_raw, const T* __restrict__ g_y, const T* __restrict__ g_pooled,
                          const T* __restrict__ y, int cv, int H, int W, int64_t total) {
  constexpr int V = ChanVec<T>::V;
  const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int Ho = H >> 1, Wo = W >> 1;
  int cq, ox, oy;
  int64_t n;
  decode_window(idx, total, cv, Wo, Ho, cq, ox, oy, n);
  const int64_t C = static_cast<int64_t>(cv) * V;
  const int64_t p00 = ((n * H + 2 * oy) * W + 2 * ox) * C + static_cast<int64_t>(cq) * V;
  const int64_t off[4] = {p00, p00 + C, p00 + W * C, p00 + W * C + C};
  uint4 yv[4], gv[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    yv[j] = ldg_stream16(y + off[j]);
    gv[j] = g_y ? ldg_stream16(g_y + off[j]) : make_uint4(0u, 0u, 0u, 0u);
  }
  float gp[V];
  if (g_pooled) ChanVec<T>::unpack(ldg_stream16(g_pooled + ((n * Ho + oy) * Wo + ox) * C + static_cast<int64_t>(cq) * V), gp);
  else {
#pragma unroll
    for (int k = 0; k < V; ++k) gp[k] = 0.f;
  }
  float yf[4][V];
#pragma unroll
  for (int j = 0; j < 4; ++j) ChanVec<T>::unpack(yv[j], yf[j]);
  int arg[V];
#pragma unroll
  for (int k = 0; k < V; ++k) {
    float m = yf[0][k];
    int a = 0;
#pragma unroll
    for (int j = 1; j < 4; ++j)
      if (yf[j][k] > m || yf[j][k] != yf[j][k]) { m = yf[j][k]; a = j; }
    arg[k] = a;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float g[V], o[V];
    ChanVec<T>::unpack(gv[j], g);
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const float tot = g[k] + (arg[k] == j ? gp[k] : 0.f);
      o[k] = yf[j][k] > 0.f ? tot : 0.f;      // threshold_backward
    }
    stg_stream16(g_raw + off[j], ChanVec<T>::pack(o));
  }
}

inline int check_pool(const char* who, int dtype, int64_t N, int C, int H, int W) {
  if (dtype != GG_F32 && dtype != GG_BF16) return fail(GG_ERR_UNSUPPORTED, "%s: dtype %d not supported (fp32 or bf16)", who, dtype);
  if (N < 0 || C < 0 || H < 0 || W < 0) return fail(GG_ERR_BAD_ARG, "%s: negative size", who);
  const int V = dtype == GG_F32 ? 4 : 8;
  if (C % V != 0) return fail(GG_ERR_UNSUPPORTED, "%s: C=%d must be a multiple of %d (16-byte channel vectors)", who, C, V);
  if ((H & 1) || (W & 1)) return fail(GG_ERR_UNSUPPORTED, "%s: H=%d, W=%d must be even (2x2 windows, stride 2, no padding)", who, H, W);
  return GG_OK;
}

}  // namespace
}  // namespace gg

using namespace gg;

extern "C" {

int64_t gg_feature_distance_workspace(int64_t N, int C, int64_t HW) {
  if (N <= 0 || C < 4 || HW <= 0) return 0;
  const int c4 = C / 4;
  const int L = c4 >= 32 ? 32 : c4;
  const int64_t chunk = distance_chunk(N, HW, kT / (L > 0 ? L : 1));
  return N * ((HW + chunk - 1) / chunk) * static_cast<int64_t>(sizeof(float));
}

int gg_feature_distance_forward(float* out, void* workspace, const void* f0, const void* f1, const float* weight,
                                int dtype, int64_t N, int C, int64_t HW, float eps, void* stream) {
  if (dtype != GG_F32 && dtype != GG_BF16) return fail(GG_ERR_UNSUPPORTED, "feature_distance: dtype %d not supported (fp32 or bf16)", dtype);
  int rc = check_distance("feature_distance", N, C, HW, weight);
  if (rc != GG_OK) return rc;
  if (N == 0) return GG_OK;
  if (!out) return fail(GG_ERR_BAD_ARG, "feature_distance: null output");
  auto st = static_cast<cudaStream_t>(stream);
  if (C == 0 || HW == 0) {   // mean over an empty set is undefined in the reference (nan); keep zeros
    cudaError_t e = cudaMemsetAsync(out, 0, N * sizeof(float), st);
    if (e != cudaSuccess) return cuda_fail(e, "feature_distance memset");
    return GG_OK;
  }
  if (!f0 || !f1 || !workspace) return fail(GG_ERR_BAD_ARG, "feature_distance: null tensor");
  int K = 1;
  if (dtype == GG_F32)
    rc = launch_distance<float, false>(static_cast<float*>(workspace), nullptr, nullptr, nullptr, static_cast<const float*>(f0),
                                       static_cast<const float*>(f1), weight, N, C, HW, eps, st, &K);
  else
    rc = launch_distance<__nv_bfloat16, false>(static_cast<float*>(workspace), nullptr, nullptr, nullptr,
                                               static_cast<const __nv_bfloat16*>(f0), static_cast<const __nv_bfloat16*>(f1),
                                               weight, N, C, HW, eps, st, &K);
  if (rc != GG_OK) return rc;
  GG_CHECK_LAUNCH("feature_distance forward launch");
  distance_finish_kernel<<<static_cast<unsigned>((N + 127) / 128), 128, 0, st>>>(out, static_cast<const float*>(workspace), N, K);
  GG_CHECK_LAUNCH("feature_distance finish launch");
  return GG_OK;
}

int gg_feature_distance_backward(void* g0, void* g1, const float* grad_out, const void* f0, const void* f1,
                                 const float* weight, int dtype, int64_t N, int C, int64_t HW, float eps, void* stream) {
  if (dtype != GG_F32 && dtype != GG_BF16) return fail(GG_ERR_UNSUPPORTED, "feature_distance backward: dtype %d not supported", dtype);
  int rc = check_distance("feature_distance backward", N, C, HW, weight);
  if (rc != GG_OK) return rc;
  if (N * HW == 0 || C == 0) return GG_OK;
  if (!grad_out || !f0 || !f1 || (!g0 && !g1)) return fail(GG_ERR_BAD_ARG, "feature_distance backward: null tensor");
  if (dtype == GG_F32)
    rc = launch_distance<float, true>(nullptr, static_cast<float*>(g0), static_cast<float*>(g1), grad_out, static_cast<const float*>(f0),
                                      static_cast<const float*>(f1), weight, N, C, HW, eps, static_cast<cudaStream_t>(stream), nullptr);
  else
    rc = launch_distance<__nv_bfloat16, true>(nullptr, static_cast<__nv_bfloat16*>(g0), static_cast<__nv_bfloat16*>(g1), grad_out,
                                              static_cast<const __nv_bfloat16*>(f0), static_cast<const __nv_bfloat16*>(f1), weight, N,
                                              C, HW, eps, static_cast<cudaStream_t>(stream), nullptr);
  if (rc != GG_OK) return rc;
  GG_CHECK_LAUNCH("feature_distance backward launch");
  return GG_OK;
}

int gg_bias_relu_pool_nhwc_forward(void* y, void* pooled, const void* raw, const float* bias, int dtype, int64_t N, int C, int H,
                                   int W, void* stream) {
  int rc = check_pool("bias_relu_pool", dtype, N, C, H, W);
  if (rc != GG_OK) return rc;
  const int V = dtype == GG_F32 ? 4 : 8;
  const int64_t total = N * (H / 2) * static_cast<int64_t>(W / 2) * (C / V);
  if (total == 0) return GG_OK;
  if (!y || !pooled || !raw) return fail(GG_ERR_BAD_ARG, "bias_relu_pool: null tensor");
  if (!aligned16(bias)) return fail(GG_ERR_BAD_ARG, "bias_relu_pool: bias must be 16-byte aligned");   // read as float4
  const int64_t grid = (total + 255) / 256;
  if (grid > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "bias_relu_pool: tensor too large");
  auto st = static_cast<cudaStream_t>(stream);
  if (dtype == GG_F32)
    bias_relu_pool_fwd_kernel<float><<<static_cast<unsigned>(grid), 256, 0, st>>>(
        static_cast<float*>(y), static_cast<float*>(pooled), static_cast<const float*>(raw), bias, C / V, H, W, total);
  else
    bias_relu_pool_fwd_kernel<__nv_bfloat16><<<static_cast<unsigned>(grid), 256, 0, st>>>(
        static_cast<__nv_bfloat16*>(y), static_cast<__nv_bfloat16*>(pooled), static_cast<const __nv_bfloat16*>(raw), bias, C / V, H,
        W, total);
  GG_CHECK_LAUNCH("bias_relu_pool forward launch");
  return GG_OK;
}

int gg_bias_relu_pool_nhwc_backward(void* grad_raw, const void* grad_y, const void* grad_pooled, const void* y, int dtype,
                                    int64_t N, int C, int H, int W, void* stream) {
  int rc = check_pool("bias_relu_pool backward", dtype, N, C, H, W);
  if (rc != GG_OK) return rc;
  const int V = dtype == GG_F32 ? 4 : 8;
  const int64_t total = N * (H / 2) * static_cast<int64_t>(W / 2) * (C / V);
  if (total == 0) return GG_OK;
  if (!grad_raw || !y) return fail(GG_ERR_BAD_ARG, "bias_relu_pool backward: null tensor");
  const int64_t grid = (total + 255) / 256;
  if (grid > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "bias_relu_pool backward: tensor too large");
  auto st = static_cast<cudaStream_t>(stream);
  if (dtype == GG_F32)
    bias_relu_pool_bwd_kernel<float><<<static_cast<unsigned>(grid), 256, 0, st>>>(
        static_cast<float*>(grad_raw), static_cast<const float*>(grad_y), static_cast<const float*>(grad_pooled),
        static_cast<const float*>(y), C / V, H, W, total);
  else
    bias_relu_pool_bwd_kernel<__nv_bfloat16><<<static_cast<unsigned>(grid), 256, 0, st>>>(
        static_cast<__nv_bfloat16*>(grad_raw), static_cast<const __nv_bfloat16*>(grad_y),
        static_cast<const __nv_bfloat16*>(grad_pooled), static_cast<const __nv_bfloat16*>(y), C / V, H, W, total);
  GG_CHECK_LAUNCH("bias_relu_pool backward launch");
  return GG_OK;
}

}  // extern "C"
