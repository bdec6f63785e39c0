// bias_act.cu -- bias + (noise) + leaky-ReLU + gain family, forward and backward (sm_90a).
//
// Replaces reference models/stylegan2/op/fused_bias_act_kernel.cu:18-99 (one scalar element per
// thread-iteration, 128-thread blocks, int div/mod per element) with 128-bit streaming accesses,
// four independent vectors in flight per thread and one channel lookup per vector.  HBM-bound:
// algorithmic bytes = s*(2*numel) forward, s*(3*numel) backward (s = bytes/element).
#include "common.cuh"

namespace gg {
namespace {

constexpr int kThreads = 256;
constexpr int kUnroll = 4;

__device__ __forceinline__ float act_apply(float x, float ref, int act, int grad, float alpha) {
  // table of fused_bias_act_kernel.cu:28-47 (act*10+grad)
  if (grad == 2) return 0.f;
  if (act == 3) {
    const float gate = (grad == 0) ? x : ref;
    return gate > 0.f ? x : x * alpha;
  }
  return x;
}

// Flat kernel, exact reference semantics: bias index = (i / step_b) % size_b.
// VEC elements per access (16 bytes when VEC = 16/sizeof(T), or VEC = 1 scalar fallback).
template <typename T, int VEC, typename Index>
__global__ void __launch_bounds__(kThreads)
bias_act_flat_kernel(T* __restrict__ out, const T* __restrict__ x, const T* __restrict__ bias,
                     const T* __restrict__ ref, int act, int grad, float alpha, float scale,
                     Index n_vec, Index step_b, Index size_b) {
  const Index base = (static_cast<Index>(blockIdx.x) * kUnroll) * kThreads + threadIdx.x;
  if constexpr (VEC > 1) {
    Vec16<T> xv[kUnroll], rv[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const Index v = base + static_cast<Index>(u) * kThreads;
      if (v < n_vec) {
        xv[u] = ld_vec_stream(x + v * VEC);
        if (ref) rv[u] = ld_vec_stream(ref + v * VEC);
      }
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const Index v = base + static_cast<Index>(u) * kThreads;
      if (v < n_vec) {
        float b = 0.f;
        if (bias) b = Cvt<T>::to_f(bias[((v * VEC) / step_b) % size_b]);
        Vec16<T> o;
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
          const float r = ref ? Cvt<T>::to_f(rv[u].v[k]) : 0.f;
          o.v[k] = Cvt<T>::from_f(act_apply(Cvt<T>::to_f(xv[u].v[k]) + b, r, act, grad, alpha) * scale);
        }
        st_vec_stream(out + v * VEC, o);
      }
    }
  } else {
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const Index i = base + static_cast<Index>(u) * kThreads;
      if (i < n_vec) {
        float b = 0.f;
        if (bias) b = Cvt<T>::to_f(bias[(i / step_b) % size_b]);
        const float r = ref ? Cvt<T>::to_f(ref[i]) : 0.f;
        out[i] = Cvt<T>::from_f(act_apply(Cvt<T>::to_f(x[i]) + b, r, act, grad, alpha) * scale);
      }
    }
  }
}

// (N, C, HW) kernel with per-sample noise plane: out = lrelu(x + nw*noise[n,p] + bias[c]) * scale.
template <typename T, int VEC>
__global__ void __launch_bounds__(kThreads)
noise_bias_act_kernel(T* __restrict__ out, const T* __restrict__ x, const T* __restrict__ noise,
                      const float* __restrict__ noise_weight, const float* __restrict__ bias,
                      const float* __restrict__ row_scale, float alpha, float scale, int64_t n_vec, int64_t C,
                      int64_t HW) {
  const float nw = noise ? (noise_weight ? __ldg(noise_weight) : 1.f) : 0.f;
  const int64_t base = (static_cast<int64_t>(blockIdx.x) * kUnroll) * kThreads + threadIdx.x;
  Vec16<T> xv[kUnroll], nv[kUnroll];
  float bv[kUnroll], rv[kUnroll];
#pragma unroll
  for (int u = 0; u < kUnroll; ++u) {
    const int64_t v = base + static_cast<int64_t>(u) * kThreads;
    if (v < n_vec) {
      const int64_t i = v * VEC;
      xv[u] = ld_vec_stream(x + i);
      const int64_t row = i / HW;  // n*C + c
      const int64_t p = i - row * HW;
      const int64_t n = row / C;
      const int64_t c = row - n * C;
      bv[u] = bias ? __ldg(bias + c) : 0.f;
      rv[u] = row_scale ? __ldg(row_scale + row) : 1.f;
      if (noise) nv[u] = *reinterpret_cast<const Vec16<T>*>(noise + n * HW + p);  // re-read per channel: keep in L1/L2
    }
  }
#pragma unroll
  for (int u = 0; u < kUnroll; ++u) {
    const int64_t v = base + static_cast<int64_t>(u) * kThreads;
    if (v < n_vec) {
      Vec16<T> o;
#pragma unroll
      for (int k = 0; k < VEC; ++k) {
        float t = fmaf(Cvt<T>::to_f(xv[u].v[k]), rv[u], bv[u]);
        if (noise) t = fmaf(nw, Cvt<T>::to_f(nv[u].v[k]), t);
        o.v[k] = Cvt<T>::from_f((t > 0.f ? t : t * alpha) * scale);
      }
      st_vec_stream(out + v * VEC, o);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
noise_bias_act_scalar_kernel(T* __restrict__ out, const T* __restrict__ x, const T* __restrict__ noise,
                             const float* __restrict__ noise_weight, const float* __restrict__ bias,
                             const float* __restrict__ row_scale, float alpha, float scale, int64_t numel, int64_t C,
                             int64_t HW) {
  const float nw = noise ? (noise_weight ? __ldg(noise_weight) : 1.f) : 0.f;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x; i < numel;
       i += static_cast<int64_t>(gridDim.x) * kThreads) {
    const int64_t row = i / HW, p = i - row * HW, n = row / C, c = row - n * C;
    float t = Cvt<T>::to_f(x[i]) * (row_scale ? __ldg(row_scale + row) : 1.f) + (bias ? __ldg(bias + c) : 0.f);
    if (noise) t = fmaf(nw, Cvt<T>::to_f(noise[n * HW + p]), t);
    out[i] = Cvt<T>::from_f((t > 0.f ? t : t * alpha) * scale);
  }
}

// Row-wise kernels over (rows, HW) planes, a row being one (n, c) plane, with one fp32 sum per row:
//   MODE 0  channel scale       out = x*s[row]; with y, sum x*y   (modulating the INPUT of a weight-shared convolution,
//                               networks.py:236/253 rewritten as conv(W, x*s); the sum is the gradient w.r.t. s)
//   MODE 1  bias-act backward   out = (y > 0 ? x : alpha*x)*gain, y = the saved forward output; sum of out as stored,
//                               as the reference's grad_input.sum() sums the stored gradient
// Sums are finished by bias_grad_finish_kernel / row_finish_kernel in a fixed order -> bit-reproducible (the reference's
// grad_input.sum() is not).
template <typename T, int MODE>
__device__ __forceinline__ void rowwise_op(float x, T y, bool has_y, float sv, float alpha, float gain, T& out,
                                           float& acc) {
  if constexpr (MODE == 0) {
    out = Cvt<T>::from_f(x * sv);
    if (has_y) acc = fmaf(x, Cvt<T>::to_f(y), acc);
  } else {
    const T r = Cvt<T>::from_f((Cvt<T>::to_f(y) > 0.f ? x : x * alpha) * gain);
    out = r;
    acc += Cvt<T>::to_f(r);
  }
}

// One CTA owns `chunk` consecutive elements of one row and writes their sum to partial[blockIdx.x]
// (blockIdx.x = row * chunks_per_row + chunk index).  VEC elements per access: 16 bytes (VEC = 16/sizeof(T)), or VEC = 1
// scalar fallback.
template <typename T, int VEC, int MODE>
__global__ void __launch_bounds__(kThreads)
rowwise_nchw_kernel(T* __restrict__ out, float* __restrict__ partial, const T* __restrict__ x, const T* __restrict__ y,
                    const float* __restrict__ s, float alpha, float gain, int64_t HW, int64_t chunk, int chunks_per_row) {
  const int64_t row = blockIdx.x / chunks_per_row;
  const int ck = blockIdx.x - row * chunks_per_row;
  const int64_t p0 = static_cast<int64_t>(ck) * chunk;
  const int64_t p1 = min(p0 + chunk, HW);
  const int64_t off = row * HW;
  const float sv = MODE == 0 ? __ldg(s + row) : 1.f;
  const bool has_y = MODE == 1 || y != nullptr;
  float acc = 0.f;
  if constexpr (VEC > 1) {
    const int64_t nv = (p1 - p0) / VEC;  // chunk and HW are multiples of VEC on this path
    for (int64_t v0 = 0; v0 < nv; v0 += static_cast<int64_t>(kThreads) * kUnroll) {
      Vec16<T> xv[kUnroll], yv[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const int64_t v = v0 + u * kThreads + threadIdx.x;
        if (v < nv) {
          xv[u] = ld_vec_stream(x + off + p0 + v * VEC);
          if (has_y) yv[u] = ld_vec_stream(y + off + p0 + v * VEC);
        }
      }
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const int64_t v = v0 + u * kThreads + threadIdx.x;
        if (v < nv) {
          Vec16<T> r;
#pragma unroll
          for (int k = 0; k < VEC; ++k)
            rowwise_op<T, MODE>(Cvt<T>::to_f(xv[u].v[k]), yv[u].v[k], has_y, sv, alpha, gain, r.v[k], acc);
          st_vec_stream(out + off + p0 + v * VEC, r);
        }
      }
    }
  } else {
    for (int64_t p = p0 + threadIdx.x; p < p1; p += kThreads)
      rowwise_op<T, MODE>(Cvt<T>::to_f(x[off + p]), has_y ? y[off + p] : T{}, has_y, sv, alpha, gain, out[off + p],
                        acc);
  }
  if (partial) {
    __shared__ float wsum[kThreads / 32];
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < kThreads / 32; ++w) t += wsum[w];
      partial[blockIdx.x] = t;
    }
  }
}

// Small rows (HW < 1024): one warp per row, 8 rows per CTA; the row's sum goes to partial[row].
template <typename T, int MODE>
__global__ void __launch_bounds__(kThreads)
rowwise_nchw_rows_kernel(T* __restrict__ out, float* __restrict__ partial, const T* __restrict__ x,
                         const T* __restrict__ y, const float* __restrict__ s, float alpha, float gain, int64_t rows,
                         int64_t HW) {
  const int64_t row = static_cast<int64_t>(blockIdx.x) * (kThreads / 32) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int64_t off = row * HW;
  const float sv = MODE == 0 ? __ldg(s + row) : 1.f;
  const bool has_y = MODE == 1 || y != nullptr;
  float acc = 0.f;
  for (int64_t p = lane; p < HW; p += 32)
    rowwise_op<T, MODE>(Cvt<T>::to_f(x[off + p]), has_y ? y[off + p] : T{}, has_y, sv, alpha, gain, out[off + p],
                        acc);
  if (partial) {
    acc = warp_sum(acc);
    if (lane == 0) partial[row] = acc;
  }
}

// grad_bias[c] = sum_n sum_k partial[(n*C + c)*K + k]   (fixed order; one warp per channel)
__global__ void bias_grad_finish_kernel(float* __restrict__ grad_bias, const float* __restrict__ partial,
                                        int64_t N, int64_t C, int K) {
  const int64_t c = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= C) return;
  const int lane = threadIdx.x & 31;
  float acc = 0.f;
  const int64_t total = N * K;
  for (int64_t j = lane; j < total; j += 32) {
    const int64_t n = j / K;
    const int k = static_cast<int>(j - n * K);
    acc += partial[(n * C + c) * K + k];
  }
  acc = warp_sum(acc);
  if (lane == 0) grad_bias[c] = acc;
}

// row_dot[row] = sum_k partial[row*K + k]
__global__ void row_finish_kernel(float* __restrict__ row_dot, const float* __restrict__ partial, int64_t rows, int K) {
  const int64_t r = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  float acc = 0.f;
  for (int k = 0; k < K; ++k) acc += partial[r * K + k];
  row_dot[r] = acc;
}

template <typename T>
int launch_flat(void* out, const void* x, const void* bias, const void* ref, int act, int grad,
                float alpha, float scale, int64_t size_x, int64_t step_b, int64_t size_b,
                cudaStream_t st) {
  constexpr int V = 16 / sizeof(T);
  const bool vec = (step_b % V == 0 || bias == nullptr) && (size_x % V == 0) && aligned16(out) &&
                   aligned16(x) && (ref == nullptr || aligned16(ref));
  const int64_t n_vec = vec ? size_x / V : size_x;
  const int64_t per_cta = static_cast<int64_t>(kThreads) * kUnroll;
  const int64_t grid = (n_vec + per_cta - 1) / per_cta;
  if (grid > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "fused_bias_act: tensor too large");
  const bool small = size_x < (1LL << 31);
  auto* o = static_cast<T*>(out);
  auto* xi = static_cast<const T*>(x);
  auto* b = static_cast<const T*>(bias);
  auto* r = static_cast<const T*>(ref);
  if (size_b == 0) size_b = 1;
  if (step_b == 0) step_b = 1;
#define GG_LAUNCH(VEC_, IDX_)                                                                      \
  bias_act_flat_kernel<T, VEC_, IDX_><<<static_cast<unsigned>(grid), kThreads, 0, st>>>(           \
      o, xi, b, r, act, grad, alpha, scale, static_cast<IDX_>(n_vec), static_cast<IDX_>(step_b),   \
      static_cast<IDX_>(size_b))
  if (vec) {
    if (small) GG_LAUNCH(V, uint32_t); else GG_LAUNCH(V, int64_t);
  } else {
    if (small) GG_LAUNCH(1, uint32_t); else GG_LAUNCH(1, int64_t);
  }
#undef GG_LAUNCH
  GG_CHECK_LAUNCH("fused_bias_act launch");
  return GG_OK;
}

template <typename T>
int launch_noise(void* out, const void* x, const void* noise, const float* nw, const float* bias,
                 const float* row_scale, float alpha, float scale, int64_t N, int64_t C, int64_t HW, cudaStream_t st) {
  constexpr int V = 16 / sizeof(T);
  const int64_t numel = N * C * HW;
  const bool vec = (HW % V == 0) && aligned16(out) && aligned16(x) && (!noise || aligned16(noise));
  if (vec) {
    const int64_t n_vec = numel / V;
    const int64_t per_cta = static_cast<int64_t>(kThreads) * kUnroll;
    const int64_t grid = (n_vec + per_cta - 1) / per_cta;
    if (grid > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "noise_bias_act: tensor too large");
    noise_bias_act_kernel<T, V><<<static_cast<unsigned>(grid), kThreads, 0, st>>>(
        static_cast<T*>(out), static_cast<const T*>(x), static_cast<const T*>(noise), nw, bias, row_scale, alpha,
        scale, n_vec, C, HW);
  } else {
    int64_t grid = (numel + kThreads - 1) / kThreads;
    if (grid > static_cast<int64_t>(sm_count()) * 16) grid = static_cast<int64_t>(sm_count()) * 16;
    noise_bias_act_scalar_kernel<T><<<static_cast<unsigned>(grid), kThreads, 0, st>>>(
        static_cast<T*>(out), static_cast<const T*>(x), static_cast<const T*>(noise), nw, bias, row_scale, alpha,
        scale, numel, C, HW);
  }
  GG_CHECK_LAUNCH("noise_bias_act launch");
  return GG_OK;
}

// Geometry of the row-wise launch, shared by the workspace queries and the launch.  Each mode keeps its own chunk: a
// different chunk regroups the partial sums, and so changes the bits of the reductions.
struct RowGeom {
  bool small_rows;      // one warp per row
  int64_t chunk;        // elements per CTA within a row
  int chunks_per_row;   // K partial sums per row
};
inline RowGeom row_geom(int mode, int64_t HW) {
  RowGeom g;
  g.small_rows = HW < 1024;
  if (g.small_rows) {
    g.chunk = HW;
    g.chunks_per_row = 1;
  } else {
    g.chunk = mode == 0 ? 16384 : 8192;  // 64 KB / 32 KB of fp32 per stream per CTA
    g.chunks_per_row = static_cast<int>((HW + g.chunk - 1) / g.chunk);
  }
  return g;
}

// The row-wise kernel and its finishing reduction over N*C rows.  MODE 0: dst = row_dot[N*C] (gg_channel_scale passes
// its rows as N, C = 1); MODE 1: dst = grad_bias[C].  `who` names the entry point in error messages.
template <typename T, int MODE>
int launch_rowwise(const char* who, void* out, float* dst, void* workspace, const void* x, const void* y, const float* s,
                   float alpha, float gain, int64_t N, int64_t C, int64_t HW, cudaStream_t st) {
  constexpr int V = 16 / sizeof(T);
  const int64_t rows = N * C;
  const RowGeom geo = row_geom(MODE, HW);
  // MODE 0's one-warp-per-row kernel writes row_dot itself; every other sum goes through the workspace
  float* partial = !dst ? nullptr : (MODE == 0 && geo.small_rows) ? dst : static_cast<float*>(workspace);
  auto* o = static_cast<T*>(out);
  auto* xi = static_cast<const T*>(x);
  auto* yi = static_cast<const T*>(y);
  if (geo.small_rows) {
    const int64_t grid = (rows + (kThreads / 32) - 1) / (kThreads / 32);
    if (grid > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "%s: too many rows", who);
    rowwise_nchw_rows_kernel<T, MODE><<<static_cast<unsigned>(grid), kThreads, 0, st>>>(o, partial, xi, yi, s, alpha,
                                                                                         gain, rows, HW);
  } else {
    const int64_t grid = rows * geo.chunks_per_row;
    if (grid > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "%s: too many rows", who);
    const bool vec = (HW % V == 0) && (geo.chunk % V == 0) && aligned16(out) && aligned16(x) && (!y || aligned16(y));
    if (vec)
      rowwise_nchw_kernel<T, V, MODE><<<static_cast<unsigned>(grid), kThreads, 0, st>>>(
          o, partial, xi, yi, s, alpha, gain, HW, geo.chunk, geo.chunks_per_row);
    else
      rowwise_nchw_kernel<T, 1, MODE><<<static_cast<unsigned>(grid), kThreads, 0, st>>>(
          o, partial, xi, yi, s, alpha, gain, HW, geo.chunk, geo.chunks_per_row);
  }
  GG_CHECK_LAUNCH("rowwise_nchw launch");
  if (dst && MODE == 1) {
    const int warps = 4;
    bias_grad_finish_kernel<<<static_cast<unsigned>((C + warps - 1) / warps), warps * 32, 0, st>>>(dst, partial, N, C,
                                                                                                  geo.chunks_per_row);
    GG_CHECK_LAUNCH("bias_grad_finish launch");
  } else if (dst && !geo.small_rows) {
    row_finish_kernel<<<static_cast<unsigned>((rows + 255) / 256), 256, 0, st>>>(dst, partial, rows, geo.chunks_per_row);
    GG_CHECK_LAUNCH("row_finish launch");
  }
  return GG_OK;
}

}  // namespace
}  // namespace gg

using namespace gg;

extern "C" {

int gg_fused_bias_act(void* out, const void* x, const void* bias, const void* ref, int dtype, int act,
                      int grad, float alpha, float scale, int64_t size_x, int64_t step_b,
                      int64_t size_b, void* stream) {
  if (size_x < 0 || step_b < 0 || size_b < 0) return fail(GG_ERR_BAD_ARG, "fused_bias_act: negative size");
  if (size_x == 0) return GG_OK;
  if (!out || !x) return fail(GG_ERR_BAD_ARG, "fused_bias_act: null tensor");
  if (act != 1 && act != 3) return fail(GG_ERR_UNSUPPORTED, "fused_bias_act: act must be 1 (linear) or 3 (lrelu)");
  if (grad < 0 || grad > 2) return fail(GG_ERR_BAD_ARG, "fused_bias_act: grad must be 0, 1 or 2");
  if (bias && (size_b <= 0 || step_b <= 0)) return fail(GG_ERR_BAD_ARG, "fused_bias_act: bias given with size_b/step_b <= 0");
  GG_DISPATCH_T16(dtype, "fused_bias_act",
                  return launch_flat<T_>(out, x, bias, ref, act, grad, alpha, scale, size_x, step_b, size_b,
                                         static_cast<cudaStream_t>(stream)));
  return GG_OK;
}

int gg_noise_bias_act(void* out, const void* x, const void* noise, const float* noise_weight,
                      const float* bias, const float* row_scale, int dtype, float alpha, float scale, int64_t N,
                      int64_t C, int64_t HW, void* stream) {
  if (N < 0 || C < 0 || HW < 0) return fail(GG_ERR_BAD_ARG, "noise_bias_act: negative size");
  if (N * C * HW == 0) return GG_OK;
  if (!out || !x) return fail(GG_ERR_BAD_ARG, "noise_bias_act: null tensor");
  GG_DISPATCH_T16(dtype, "noise_bias_act",
                  return launch_noise<T_>(out, x, noise, noise_weight, bias, row_scale, alpha, scale, N, C, HW,
                                          static_cast<cudaStream_t>(stream)));
  return GG_OK;
}

int64_t gg_channel_scale_workspace(int64_t rows, int64_t HW) {
  if (rows <= 0 || HW <= 0) return 0;
  return rows * row_geom(0, HW).chunks_per_row * static_cast<int64_t>(sizeof(float));
}

int gg_channel_scale(void* out, float* row_dot, void* workspace, const void* x, const void* y, const float* s, int dtype,
                     int64_t rows, int64_t HW, void* stream) {
  if (rows < 0 || HW < 0) return fail(GG_ERR_BAD_ARG, "channel_scale: negative size");
  if (rows * HW == 0) {
    if (row_dot && rows > 0) {   // the sum over an empty plane is 0
      cudaError_t e = cudaMemsetAsync(row_dot, 0, rows * sizeof(float), static_cast<cudaStream_t>(stream));
      if (e != cudaSuccess) return cuda_fail(e, "channel_scale memset");
    }
    return GG_OK;
  }
  if (!out || !x || !s) return fail(GG_ERR_BAD_ARG, "channel_scale: null tensor");
  if (row_dot && (!y || !workspace)) return fail(GG_ERR_BAD_ARG, "channel_scale: row_dot needs y and a workspace");
  // this entry point's limit is rows x chunks, also for small rows where a CTA takes 8 rows (launch_rowwise counts CTAs)
  if (rows * row_geom(0, HW).chunks_per_row > 0x7fffffffLL) return fail(GG_ERR_BAD_ARG, "channel_scale: too many rows");
  GG_DISPATCH_T16(dtype, "channel_scale",
                  return launch_rowwise<T_, 0>("channel_scale", out, row_dot, workspace, x, row_dot ? y : nullptr, s,
                                               0.f, 1.f, rows, 1, HW, static_cast<cudaStream_t>(stream)));
  return GG_OK;
}

int64_t gg_bias_act_backward_workspace(int64_t N, int64_t C, int64_t HW) {
  if (N <= 0 || C <= 0 || HW <= 0) return 0;
  return N * C * row_geom(1, HW).chunks_per_row * static_cast<int64_t>(sizeof(float));
}

int gg_bias_act_backward(void* gx, float* grad_bias, void* workspace, const void* g, const void* out,
                         int dtype, float alpha, float scale, int64_t N, int64_t C, int64_t HW,
                         void* stream) {
  if (N < 0 || C < 0 || HW < 0) return fail(GG_ERR_BAD_ARG, "bias_act_backward: negative size");
  auto st = static_cast<cudaStream_t>(stream);
  if (N * C * HW == 0) {
    if (grad_bias && C > 0) {
      cudaError_t e = cudaMemsetAsync(grad_bias, 0, C * sizeof(float), st);
      if (e != cudaSuccess) return cuda_fail(e, "bias_act_backward memset");
    }
    return GG_OK;
  }
  if (!gx || !g || !out) return fail(GG_ERR_BAD_ARG, "bias_act_backward: null tensor");
  if (grad_bias && !workspace) return fail(GG_ERR_BAD_ARG, "bias_act_backward: grad_bias needs a workspace");
  GG_DISPATCH_T16(dtype, "bias_act_backward",
                  return launch_rowwise<T_, 1>("bias_act_backward", gx, grad_bias, workspace, g, out, nullptr, alpha,
                                               scale, N, C, HW, st));
  return GG_OK;
}

}  // extern "C"
