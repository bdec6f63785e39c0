// optim.cu -- the per-iteration bookkeeping of the training loop as fused kernels (sm_90a), SURVEY.md 8(f) rank 3.
//
//   gg_adam_ema_step   reference train.py:126-134: `t_optim.step()`, `ll_optim.step()` (torch.optim.Adam, betas (0.9, 0.999),
//                      eps 1e-8) and `accumulate(t_ema, t_module)` (models/__init__.py:19-24: a `mul_` + `add_` PAIR PER
//                      PARAMETER TENSOR) as ONE multi-tensor pass over every parameter of both optimisers:
//                          m = m + (1-b1)(g - m);  v = b2 v + (1-b2) g^2
//                          p -= lr/(1-b1^t) * m / (sqrt(v)/sqrt(1-b2^t) + eps)           (torch's default Adam arithmetic)
//                          ema = decay*ema + (1-decay)*p                                   (tensors that have an EMA twin)
//                      36 B per parameter with EMA (read p, g, m, v, ema; write p, m, v, ema) instead of 28 B (fused Adam) +
//                      20 B (the two EMA passes); learning rates and the step counter live in device memory, so the step is
//                      CUDA-graph capturable and one captured graph serves the whole lr schedule.
//   gg_tv_loss_*       reference models/losses/loss.py:4-12 `total_variation_loss(delta_flow)`: Huber-penalised finite
//                      differences of the (N, H, W, 2) residual flow, mean over each difference tensor -- ~15 ATen launches
//                      forward and ~25 backward on a 4 MB tensor; here one reduction kernel forward (+ finish) and one
//                      gather-form (atomic-free, deterministic) kernel backward.
#include "common.cuh"
#include "tv.cuh"

namespace gg {
namespace {

struct AdamTensor {          // one row of the device-resident table (7 x 8 bytes)
  float* p; const float* g; float* m; float* v; float* ema;
  int64_t numel;
  const float* lr;           // device scalar of this tensor's parameter group
};

__global__ void adam_tick_kernel(float* __restrict__ state, double beta1, double beta2) {
  // state[0] = step (as float, exact up to 2^24), state[1] = 1 - b1^t, state[2] = sqrt(1 - b2^t)
  const float t = state[0] + 1.f;
  state[0] = t;
  state[1] = static_cast<float>(1.0 - pow(beta1, static_cast<double>(t)));
  state[2] = static_cast<float>(sqrt(1.0 - pow(beta2, static_cast<double>(t))));
}

constexpr int kAdamThreads = 256;

__global__ void __launch_bounds__(kAdamThreads)
adam_ema_kernel(const AdamTensor* __restrict__ table, const int* __restrict__ block_tensor,
                const int* __restrict__ block_chunk, const float* __restrict__ state, float omb1, float beta2, float omb2,
                float eps, float decay, float omd, int chunk) {
  // omb1 = 1 - beta1, omb2 = 1 - beta2, omd = 1 - decay are formed in double precision on the host (1 - 0.999f in fp32
  // would be off by 5e-5 relative)
  const AdamTensor t = table[block_tensor[blockIdx.x]];
  const int64_t e0 = static_cast<int64_t>(block_chunk[blockIdx.x]) * chunk;
  const int64_t e1 = min(e0 + static_cast<int64_t>(chunk), t.numel);
  const float lr = __ldg(t.lr);
  const float step_size = lr / state[1];
  const float inv_bc2 = 1.f / state[2];
  const bool vec = ((reinterpret_cast<uintptr_t>(t.p) | reinterpret_cast<uintptr_t>(t.g) | reinterpret_cast<uintptr_t>(t.m) |
                     reinterpret_cast<uintptr_t>(t.v) | reinterpret_cast<uintptr_t>(t.ema)) & 15) == 0 && (e0 & 3) == 0;
  auto upd = [&](float& p, float g, float& m, float& v, float& e) {
    m = fmaf(omb1, g - m, m);
    v = fmaf(omb2 * g, g, beta2 * v);
    const float denom = sqrtf(v) * inv_bc2 + eps;
    p -= step_size * (m / denom);
    e = fmaf(decay, e, omd * p);
  };
  if (vec) {
    const int64_t n4 = (e1 - e0) >> 2;
    for (int64_t i = threadIdx.x; i < n4; i += kAdamThreads) {
      const int64_t o = e0 + i * 4;
      float4 p = *reinterpret_cast<const float4*>(t.p + o), g = __ldcs(reinterpret_cast<const float4*>(t.g + o));
      float4 m = *reinterpret_cast<const float4*>(t.m + o), v = *reinterpret_cast<const float4*>(t.v + o);
      float4 e = t.ema ? *reinterpret_cast<const float4*>(t.ema + o) : make_float4(0.f, 0.f, 0.f, 0.f);
      upd(p.x, g.x, m.x, v.x, e.x); upd(p.y, g.y, m.y, v.y, e.y); upd(p.z, g.z, m.z, v.z, e.z); upd(p.w, g.w, m.w, v.w, e.w);
      *reinterpret_cast<float4*>(t.p + o) = p;
      *reinterpret_cast<float4*>(t.m + o) = m;
      *reinterpret_cast<float4*>(t.v + o) = v;
      if (t.ema) *reinterpret_cast<float4*>(t.ema + o) = e;
    }
    for (int64_t o = e0 + n4 * 4 + threadIdx.x; o < e1; o += kAdamThreads) {
      float p = t.p[o], m = t.m[o], v = t.v[o], e = t.ema ? t.ema[o] : 0.f;
      upd(p, t.g[o], m, v, e);
      t.p[o] = p; t.m[o] = m; t.v[o] = v;
      if (t.ema) t.ema[o] = e;
    }
  } else {
    for (int64_t o = e0 + threadIdx.x; o < e1; o += kAdamThreads) {
      float p = t.p[o], m = t.m[o], v = t.v[o], e = t.ema ? t.ema[o] : 0.f;
      upd(p, t.g[o], m, v, e);
      t.p[o] = p; t.m[o] = m; t.v[o] = v;
      if (t.ema) t.ema[o] = e;
    }
  }
}

// ------------------------------------------------------------------------------------------------ equalised-lr weights
// gg_scale_cast_multi   reference networks.py:121-127,146-149 (`self.weight * self.scale` inside EVERY EqualConv2d /
//                       EqualLinear forward): one ATen multiply per layer forward and one per layer backward -- 124
//                       parameter-sized launches per step at ~3.6 us each, plus a cast each way with bf16 activations.
//                       Here: dst[i] = (dst type) (src[i] * scale) for a whole TABLE of tensors in one launch; used forward
//                       (fp32 master weight -> scaled weight in the convolution's dtype) and backward (gradient of the scaled
//                       weight, fp32 or bf16 -> fp32 gradient of the master weight) by op/scaled_weights.py.
struct ScaleTensor {          // one row of the device-resident table (4 x 8 bytes)
  const void* src; void* dst;
  int64_t numel;
  float scale;
  int dtypes;                 // src dtype | dst dtype << 8   (GG_F32 / GG_BF16)
};

__device__ __forceinline__ float ld_as_float(const void* p, int dt, int64_t i) {
  return dt == GG_F32 ? static_cast<const float*>(p)[i] : __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i]);
}
__device__ __forceinline__ void st_from_float(void* p, int dt, int64_t i, float v) {
  if (dt == GG_F32) static_cast<float*>(p)[i] = v;
  else static_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v);
}

__global__ void __launch_bounds__(kAdamThreads)
scale_cast_multi_kernel(const ScaleTensor* __restrict__ table, const int* __restrict__ block_tensor,
                        const int* __restrict__ block_chunk, int chunk) {
  const ScaleTensor t = table[block_tensor[blockIdx.x]];
  const int64_t e0 = static_cast<int64_t>(block_chunk[blockIdx.x]) * chunk;
  const int64_t e1 = min(e0 + static_cast<int64_t>(chunk), t.numel);
  const int sdt = t.dtypes & 0xff, ddt = (t.dtypes >> 8) & 0xff;
  const bool vec = ((reinterpret_cast<uintptr_t>(t.src) | reinterpret_cast<uintptr_t>(t.dst)) & 15) == 0 && (e0 & 3) == 0;
  int64_t done = e0;
  if (vec) {
    const int64_t n4 = (e1 - e0) >> 2;
    for (int64_t i = threadIdx.x; i < n4; i += kAdamThreads) {
      const int64_t o = e0 + i * 4;
      float v[4];
      if (sdt == GG_F32) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(static_cast<const float*>(t.src) + o));
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
      } else {
        const uint2 a = __ldg(reinterpret_cast<const uint2*>(static_cast<const __nv_bfloat16*>(t.src) + o));
        v[0] = __uint_as_float(a.x << 16); v[1] = __uint_as_float(a.x & 0xffff0000u);
        v[2] = __uint_as_float(a.y << 16); v[3] = __uint_as_float(a.y & 0xffff0000u);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] *= t.scale;
      if (ddt == GG_F32) {
        *reinterpret_cast<float4*>(static_cast<float*>(t.dst) + o) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
        const __nv_bfloat162 lo = __floats2bfloat162_rn(v[0], v[1]), hi = __floats2bfloat162_rn(v[2], v[3]);
        *reinterpret_cast<uint2*>(static_cast<__nv_bfloat16*>(t.dst) + o) =
            make_uint2(*reinterpret_cast<const uint32_t*>(&lo), *reinterpret_cast<const uint32_t*>(&hi));
      }
    }
    done = e0 + n4 * 4;
  }
  for (int64_t o = done + threadIdx.x; o < e1; o += kAdamThreads) st_from_float(t.dst, ddt, o, ld_as_float(t.src, sdt, o) * t.scale);
}

// ------------------------------------------------------------------------------------------------ total variation
constexpr int kTvThreads = 256;

// partial[block] = sum over the block's elements of huber(dy)*inv_y + huber(dx)*inv_x
__global__ void __launch_bounds__(kTvThreads)
tv_fwd_kernel(float* __restrict__ partial, const float* __restrict__ f, int64_t total, int H, int W, float inv_y, float inv_x) {
  __shared__ float red[kTvThreads / 32];
  float acc = 0.f;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kTvThreads + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * kTvThreads) {
    const int64_t pix = i >> 1;
    const int x = static_cast<int>(pix % W);
    const int y = static_cast<int>((pix / W) % H);
    const float c = f[i];
    if (y + 1 < H) acc = fmaf(huber(c - f[i + 2 * W]), inv_y, acc);
    if (x + 1 < W) acc = fmaf(huber(c - f[i + 2]), inv_x, acc);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < kTvThreads / 32; ++i) t += red[i];
    partial[blockIdx.x] = t;
  }
}

__global__ void tv_finish_kernel(float* __restrict__ out, const float* __restrict__ partial, int n) {
  __shared__ float red[32];
  float acc = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += partial[i];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (blockDim.x + 31) / 32; ++i) t += red[i];
    out[0] = t;
  }
}

// grad[i] = go * ( h'(f[i]-f[i+dy])*inv_y - h'(f[i-dy]-f[i])*inv_y + the same along x )
__global__ void __launch_bounds__(kTvThreads)
tv_bwd_kernel(float* __restrict__ grad, const float* __restrict__ gout, const float* __restrict__ f, int64_t total, int H,
              int W, float inv_y, float inv_x) {
  const float go = __ldg(gout);
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kTvThreads + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * kTvThreads) {
    const int64_t pix = i >> 1;
    const int x = static_cast<int>(pix % W);
    const int y = static_cast<int>((pix / W) % H);
    const float c = f[i];
    float g = 0.f;
    if (y + 1 < H) g = fmaf(huber_grad(c - f[i + 2 * W]), inv_y, g);
    if (y > 0) g = fmaf(-huber_grad(f[i - 2 * W] - c), inv_y, g);
    if (x + 1 < W) g = fmaf(huber_grad(c - f[i + 2]), inv_x, g);
    if (x > 0) g = fmaf(-huber_grad(f[i - 2] - c), inv_x, g);
    grad[i] = go * g;
  }
}

inline int tv_blocks(int64_t total) {
  int64_t b = (total + kTvThreads - 1) / kTvThreads;
  const int64_t cap = 4LL * sm_count();
  return static_cast<int>(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace
}  // namespace gg

using namespace gg;

extern "C" {

int gg_scale_cast_multi(const void* table, const int* block_tensor, const int* block_chunk, int blocks, int chunk,
                        void* stream) {
  if (blocks < 0 || chunk < 4 || (chunk & 3)) return fail(GG_ERR_BAD_ARG, "scale_cast_multi: bad geometry (chunk must be a multiple of 4)");
  if (blocks == 0) return GG_OK;
  if (!table || !block_tensor || !block_chunk) return fail(GG_ERR_BAD_ARG, "scale_cast_multi: null table");
  scale_cast_multi_kernel<<<static_cast<unsigned>(blocks), kAdamThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const ScaleTensor*>(table), block_tensor, block_chunk, chunk);
  GG_CHECK_LAUNCH("scale_cast_multi launch");
  return GG_OK;
}

int gg_adam_ema_step(const void* table, const int* block_tensor, const int* block_chunk, int blocks, int chunk,
                     float* state, double beta1, double beta2, double eps, double ema_decay, void* stream) {
  if (blocks < 0 || chunk < 1) return fail(GG_ERR_BAD_ARG, "adam_ema_step: bad geometry");
  if (!state) return fail(GG_ERR_BAD_ARG, "adam_ema_step: null state");
  if (!(beta1 >= 0.0 && beta1 < 1.0 && beta2 >= 0.0 && beta2 < 1.0 && eps >= 0.0)) return fail(GG_ERR_BAD_ARG, "adam_ema_step: bad hyper-parameters");
  auto st = static_cast<cudaStream_t>(stream);
  adam_tick_kernel<<<1, 1, 0, st>>>(state, beta1, beta2);
  GG_CHECK_LAUNCH("adam_tick launch");
  if (blocks == 0) return GG_OK;
  if (!table || !block_tensor || !block_chunk) return fail(GG_ERR_BAD_ARG, "adam_ema_step: null table");
  adam_ema_kernel<<<static_cast<unsigned>(blocks), kAdamThreads, 0, st>>>(static_cast<const AdamTensor*>(table), block_tensor,
                                                                         block_chunk, state, static_cast<float>(1.0 - beta1),
                                                                         static_cast<float>(beta2), static_cast<float>(1.0 - beta2),
                                                                         static_cast<float>(eps), static_cast<float>(ema_decay),
                                                                         static_cast<float>(1.0 - ema_decay), chunk);
  GG_CHECK_LAUNCH("adam_ema launch");
  return GG_OK;
}

int64_t gg_tv_loss_workspace(int64_t N, int H, int W) {
  if (N <= 0 || H <= 0 || W <= 0) return 0;
  return static_cast<int64_t>(tv_blocks(N * H * static_cast<int64_t>(W) * 2)) * static_cast<int64_t>(sizeof(float));
}

int gg_tv_loss_forward(float* out, void* workspace, const float* flow, int64_t N, int H, int W, void* stream) {
  if (N < 0 || H < 0 || W < 0) return fail(GG_ERR_BAD_ARG, "tv_loss: negative size");
  if (!out) return fail(GG_ERR_BAD_ARG, "tv_loss: null output");
  auto st = static_cast<cudaStream_t>(stream);
  const int64_t total = N * H * static_cast<int64_t>(W) * 2;
  if (total == 0 || H < 2 || W < 2) return fail(GG_ERR_BAD_ARG, "tv_loss: the flow needs at least 2 x 2 pixels (the reference's mean of an empty difference is nan)");
  if (!flow || !workspace) return fail(GG_ERR_BAD_ARG, "tv_loss: null tensor");
  const float inv_y = 1.f / (static_cast<float>(N) * (H - 1) * W * 2), inv_x = 1.f / (static_cast<float>(N) * H * (W - 1) * 2);
  const int blocks = tv_blocks(total);
  tv_fwd_kernel<<<blocks, kTvThreads, 0, st>>>(static_cast<float*>(workspace), flow, total, H, W, inv_y, inv_x);
  GG_CHECK_LAUNCH("tv_fwd launch");
  tv_finish_kernel<<<1, 256, 0, st>>>(out, static_cast<const float*>(workspace), blocks);
  GG_CHECK_LAUNCH("tv_finish launch");
  return GG_OK;
}

int gg_tv_loss_backward(float* grad_flow, const float* grad_out, const float* flow, int64_t N, int H, int W, void* stream) {
  if (N < 0 || H < 0 || W < 0) return fail(GG_ERR_BAD_ARG, "tv_loss backward: negative size");
  const int64_t total = N * H * static_cast<int64_t>(W) * 2;
  if (total == 0) return GG_OK;
  if (H < 2 || W < 2) return fail(GG_ERR_BAD_ARG, "tv_loss backward: the flow needs at least 2 x 2 pixels");
  if (!grad_flow || !grad_out || !flow) return fail(GG_ERR_BAD_ARG, "tv_loss backward: null tensor");
  const float inv_y = 1.f / (static_cast<float>(N) * (H - 1) * W * 2), inv_x = 1.f / (static_cast<float>(N) * H * (W - 1) * 2);
  tv_bwd_kernel<<<tv_blocks(total) * 4, kTvThreads, 0, static_cast<cudaStream_t>(stream)>>>(grad_flow, grad_out, flow, total, H, W,
                                                                                          inv_y, inv_x);
  GG_CHECK_LAUNCH("tv_bwd launch");
  return GG_OK;
}

}  // extern "C"
