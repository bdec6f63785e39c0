// blend.cu -- Laplacian pyramid blending (sm_90a), reference utils/laplacian_blending.py:56-107.
//
// The reference builds Laplacian stacks of img0 / img1 and a Gaussian stack of the mask with a depthwise 2-D F.conv2d per
// level (replicate padding, the same width k + a at every level, sigma s * m^l), then
//     out = sum_{l<L-1} lerp(A_l - A_{l+1}, B_l - B_{l+1}, M_l) + lerp(A_{L-1}, B_{L-1}, M_{L-1}),   G_{l+1} = T_l G_l.
// With clamped indices the 2-D blur T_l separates EXACTLY into a horizontal and a vertical 1-D pass, so one launch per level
// does, for every (2C+1)-plane sample and a TH x TW output tile:
//   1. stage the input tile plus a (P-1)-wide halo in shared memory, with clamped (replicate) addressing;
//   2. horizontal pass over all TH+P-1 halo rows into a second shared buffer (8 outputs per thread, taps in registers);
//   3. vertical pass from shared memory (8 rows per thread), then the level's epilogue.
// P is the tap count rounded up to a multiple of 8 (compile-time, so both passes fully unroll); the padding taps are 0.
// With the 45-tap preset the work is fp32-FMA-bound: (1 + (TH+P-1)/TH) * P FMA per pixel and plane vs ~6 B of HBM traffic.
//
// Backward (gather form, no atomics): a forward sweep keeps the mask stack M_1..M_{L-1} and the mask's direct gradient
//   d_l = sum_c g_c ((B_l - B_{l+1}) - (A_l - A_{l+1})),  d_{L-1} = sum_c g_c (B_{L-1} - A_{L-1})
// in the workspace, then Horner's rule runs down the chain: U_{L-1} = g c_{L-1}, U_l = g c_l + T_l^T U_{l+1} with
//   c^A_0 = 1 - M_0, c^A_l = M_{l-1} - M_l;  c^B_0 = M_0, c^B_l = M_l - M_{l-1};  U^M_{L-1} = d_{L-1}, U^M_l = d_l + T_l^T U^M_{l+1}.
// T_l^T is the same tiled kernel on zero-padded input (the taps are symmetric), except that the first and last row/column
// gather the taps that clamped onto them in the forward pass (the "border fold", prefix sums of the taps).
#include "common.cuh"

namespace gg {
namespace {

constexpr int kBlendThreads = 256;
constexpr int kTW = 32;            // tile width  (one warp of columns in the vertical pass)
constexpr int kTH = 64;            // tile height (8 warps x 8 rows)
constexpr int kMaxWidth = 63;      // taps per level; P = 64 at most

enum { BL_FWD = 0, BL_BWD_SWEEP = 1, BL_ADJ = 2 };

struct LevelArgs {
  const float* a_in; const float* b_in; const float* m_in;   // level-l planes (ADJ: U_{l+1})
  float* a_out; float* b_out; float* m_out;                  // level-(l+1) planes (ADJ: U_l)
  float* acc;            // FWD: out;  BWD_SWEEP: d_l
  float* acc_last;       // BWD_SWEEP, last level: d_{L-1}
  const float* g;        // BWD_SWEEP / ADJ: upstream gradient (N, C, H, W)
  const float* m_prev;   // ADJ: M_{l-1} (l >= 1)
  const float* m_cur;    // ADJ: M_l
  const float* d;        // ADJ: d_l (may alias m_out: read then overwritten by the same thread)
  const float* taps;     // this level's `width` taps
  int width, C, H, W;
  int first, last;       // FWD / BWD_SWEEP: l == 0, l == L-2;  ADJ: first = (l == 0)
};

// torch.lerp's formula (ATen lerp: weight < 0.5 ? a + w (b - a) : b - (b - a)(1 - w)), single-rounded products
__device__ __forceinline__ float lerp_ref(float a, float b, float w) {
  return fabsf(w) < 0.5f ? fmaf(w, b - a, a) : fmaf(-(b - a), 1.f - w, b);
}

// value of the tap-prefix fold at a border: sum over i < =min(r, n-1) of src(i) * cum[r - i]  (cum[m] = sum_{t<=m} w[t])
__device__ __forceinline__ float fold(const float* src, int stride, int r, int n, const float* cum) {
  const int lim = min(r, n - 1);
  float s = 0.f;
  for (int i = 0; i <= lim; ++i) s = fmaf(src[i * stride], cum[r - i], s);
  return s;
}

template <int NC, int MODE>
__global__ void __launch_bounds__(kBlendThreads, 2)   // 2 CTAs/SM: <= 128 registers, no spills at any P
blend_level_kernel(const LevelArgs p) {
  constexpr int P = 8 * NC;
  constexpr int HROWS = kTH + P - 1;      // rows the vertical pass reads
  constexpr int SWI = kTW + P;            // staged row stride (columns read: < kTW + P - 1)
  extern __shared__ __align__(16) float smem[];
  float* s_in = smem;                     // HROWS x SWI
  float* s_h = s_in + HROWS * SWI;        // HROWS x kTW
  float* s_cum = s_h + HROWS * kTW;       // P (ADJ: tap prefix sums)

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int H = p.H, W = p.W, C = p.C, r = p.width >> 1;
  const int x0 = blockIdx.x * kTW, y0 = blockIdx.y * kTH;
  const int64_t n = blockIdx.z, HW = static_cast<int64_t>(H) * W;

  float w[P];
#pragma unroll
  for (int j = 0; j < P; ++j) w[j] = j < p.width ? __ldg(p.taps + j) : 0.f;
  float wsum = 0.f;
  if (MODE == BL_ADJ) {
    if (tid == 0) {
      double c = 0.0;
      for (int j = 0; j < p.width; ++j) { c += static_cast<double>(p.taps[j]); s_cum[j] = static_cast<float>(c); }
    }
    __syncthreads();
    wsum = s_cum[p.width - 1];
  }

  // this thread's vertical-pass outputs: column x, rows y .. y+7
  const int vx = lane, vy = warp * 8;
  const int gx = x0 + vx;

  for (int plane = 0; plane < 2 * C + 1; ++plane) {
    // plane 0 = mask; then A_c, B_c alternating
    const int c = (plane - 1) >> 1;
    const bool is_mask = plane == 0, is_a = !is_mask && ((plane - 1) & 1) == 0;
    const float* src = is_mask ? p.m_in + n * HW : (is_a ? p.a_in : p.b_in) + (n * C + c) * HW;

    // 1. stage: clamped (FWD / BWD_SWEEP) or zero-padded (ADJ) input rows y0-r .. y0-r+HROWS-1, cols x0-r .. x0-r+SWI-1
    for (int q = warp; q < HROWS; q += kBlendThreads / 32) {
      const int sy = y0 - r + q;
      const bool row_in = sy >= 0 && sy < H;
      const float* row = src + static_cast<int64_t>(min(max(sy, 0), H - 1)) * W;
      for (int cc = lane; cc < SWI; cc += 32) {
        const int sx = x0 - r + cc;
        float v;
        if (MODE == BL_ADJ) v = (row_in && sx >= 0 && sx < W) ? __ldg(row + sx) : 0.f;
        else v = __ldg(row + min(max(sx, 0), W - 1));
        s_in[q * SWI + cc] = v;
      }
    }
    __syncthreads();

    // 2. horizontal pass: h[q][xx] = sum_j w[j] s_in[q][xx + j]
    for (int it = tid; it < HROWS * (kTW / 8); it += kBlendThreads) {
      const int q = it / (kTW / 8), xg = (it % (kTW / 8)) * 8;
      const float* s = s_in + q * SWI + xg;
      float acc[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] = 0.f;
#pragma unroll
      for (int i = 0; i < P + 8; i += 4) {
        const float4 v4 = *reinterpret_cast<const float4*>(s + i);
        const float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const int j = i + u - k;
            if (j >= 0 && j < P) acc[k] = fmaf(w[j], v[u], acc[k]);
          }
      }
      if (MODE == BL_ADJ && (x0 + xg == 0 || x0 + xg + 8 > W - 1)) {   // border fold (first / last column)
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int x = x0 + xg + k;
          const float* rowp = s_in + q * SWI;
          if (W == 1 && x == 0) acc[k] = rowp[r] * wsum;
          else if (x == 0) acc[k] = fold(rowp + r, 1, r, W, s_cum);                    // col of image x=i: r + i
          else if (x == W - 1) acc[k] = fold(rowp + (W - 1 - x0) + r, -1, r, W, s_cum); // col of x=W-1-i
        }
      }
      float4* o = reinterpret_cast<float4*>(s_h + q * kTW + xg);
      o[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
      o[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
    __syncthreads();

    // 3. vertical pass: v[yy][x] = sum_j w[j] h[yy + j][x], rows vy .. vy+7
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
#pragma unroll
    for (int i = 0; i < P + 7; ++i) {
      const float v = s_h[(vy + i) * kTW + vx];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int j = i - k;
        if (j >= 0 && j < P) acc[k] = fmaf(w[j], v, acc[k]);
      }
    }
    if (MODE == BL_ADJ && (y0 + vy == 0 || y0 + vy + 8 > H - 1)) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int y = y0 + vy + k;
        const float* colp = s_h + vx;
        if (H == 1 && y == 0) acc[k] = colp[r * kTW] * wsum;
        else if (y == 0) acc[k] = fold(colp + r * kTW, kTW, r, H, s_cum);
        else if (y == H - 1) acc[k] = fold(colp + ((H - 1 - y0) + r) * kTW, -kTW, r, H, s_cum);
      }
    }

    // epilogue
    if (gx < W) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int y = y0 + vy + k;
        if (y >= H) break;
        const int64_t pix = static_cast<int64_t>(y) * W + gx;
        const float v1 = acc[k];
        if (MODE != BL_ADJ) {
          const float v0 = s_in[(vy + k + r) * SWI + vx + r];
          if (is_mask) { p.m_out[n * HW + pix] = v1; continue; }
          const int64_t off = (n * C + c) * HW + pix;
          if (is_a) { p.a_out[off] = v1; continue; }
          p.b_out[off] = v1;
          const float a0 = p.a_in[off], a1 = p.a_out[off];   // a_out: written above by this thread
          if (MODE == BL_FWD) {
            const float m0 = p.m_in[n * HW + pix], m1 = p.m_out[n * HW + pix];
            float t = lerp_ref(a0 - a1, v0 - v1, m0);
            float o = p.first ? t : p.acc[off] + t;
            if (p.last) o = o + lerp_ref(a1, v1, m1);
            p.acc[off] = o;
          } else {
            const float g = p.g[off];
            const float dt = g * ((v0 - v1) - (a0 - a1));
            p.acc[n * HW + pix] = c == 0 ? dt : p.acc[n * HW + pix] + dt;
            if (p.last) {
              const float dl = g * (v1 - a1);
              p.acc_last[n * HW + pix] = c == 0 ? dl : p.acc_last[n * HW + pix] + dl;
            }
          }
        } else {
          if (is_mask) { p.m_out[n * HW + pix] = p.d[n * HW + pix] + v1; continue; }
          const int64_t off = (n * C + c) * HW + pix;
          const float mc = p.m_cur[n * HW + pix];
          const float ca = p.first ? 1.f - mc : p.m_prev[n * HW + pix] - mc;     // c^A_l
          const float cb = p.first ? mc : mc - p.m_prev[n * HW + pix];           // c^B_l
          (is_a ? p.a_out : p.b_out)[off] = fmaf(p.g[off], is_a ? ca : cb, v1);
        }
      }
    }
    __syncthreads();
  }
}

// U_{L-1} = g c_{L-1}: c^A = M_{L-2} - M_{L-1}, c^B = -c^A  (L >= 2)
__global__ void blend_adj_init_kernel(float* __restrict__ ua, float* __restrict__ ub, const float* __restrict__ g,
                                      const float* __restrict__ m_prev, const float* __restrict__ m_last, int C,
                                      int64_t HW, int64_t total) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int64_t n = i / (C * HW), pix = i % HW;
  const float ca = m_prev[n * HW + pix] - m_last[n * HW + pix];
  ua[i] = g[i] * ca;
  ub[i] = g[i] * -ca;
}

// L == 1: out = lerp(img0, img1, mask)
__global__ void blend_lerp_kernel(float* __restrict__ out, const float* __restrict__ a, const float* __restrict__ b,
                                  const float* __restrict__ m, int C, int64_t HW, int64_t total) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int64_t n = i / (C * HW), pix = i % HW;
  out[i] = lerp_ref(a[i], b[i], m[n * HW + pix]);
}

// L == 1 backward: g0 = g (1 - M), g1 = g M, gm = sum_c g (B - A)
__global__ void blend_lerp_bwd_kernel(float* __restrict__ ga, float* __restrict__ gb, float* __restrict__ gm,
                                      const float* __restrict__ g, const float* __restrict__ a, const float* __restrict__ b,
                                      const float* __restrict__ m, int C, int64_t HW, int64_t total) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;   // over N * HW
  if (i >= total) return;
  const int64_t n = i / HW, pix = i % HW;
  const float mv = m[i];
  float s = 0.f;
  for (int c = 0; c < C; ++c) {
    const int64_t off = (n * C + c) * HW + pix;
    ga[off] = g[off] * (1.f - mv);
    gb[off] = g[off] * mv;
    s = c == 0 ? g[off] * (b[off] - a[off]) : s + g[off] * (b[off] - a[off]);
  }
  gm[i] = s;
}

size_t level_smem_bytes(int nc) {
  const int P = 8 * nc, hrows = kTH + P - 1;
  return sizeof(float) * (static_cast<size_t>(hrows) * (kTW + P) + static_cast<size_t>(hrows) * kTW + P);
}

template <int NC, int MODE>
int launch_level_t(const LevelArgs& a, int64_t N, cudaStream_t st) {
  static DeviceOnce once;
  const size_t smem = level_smem_bytes(NC);
  if (once.needed()) {
    cudaError_t e = cudaFuncSetAttribute(blend_level_kernel<NC, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(smem));
    if (e != cudaSuccess) return cuda_fail(e, "laplacian_blend: smem attribute");
    once.done();
  }
  const dim3 grid((a.W + kTW - 1) / kTW, (a.H + kTH - 1) / kTH, static_cast<unsigned>(N));
  blend_level_kernel<NC, MODE><<<grid, kBlendThreads, smem, st>>>(a);
  GG_CHECK_LAUNCH("laplacian_blend level launch");
  return GG_OK;
}

template <int MODE>
int launch_level(const LevelArgs& a, int64_t N, cudaStream_t st) {
  switch ((a.width + 7) / 8) {
    case 1: return launch_level_t<1, MODE>(a, N, st);
    case 2: return launch_level_t<2, MODE>(a, N, st);
    case 3: return launch_level_t<3, MODE>(a, N, st);
    case 4: return launch_level_t<4, MODE>(a, N, st);
    case 5: return launch_level_t<5, MODE>(a, N, st);
    case 6: return launch_level_t<6, MODE>(a, N, st);
    case 7: return launch_level_t<7, MODE>(a, N, st);
    default: return launch_level_t<8, MODE>(a, N, st);
  }
}

int check_args(int64_t N, int C, int H, int W, int levels, int width, const float* taps, const char* what) {
  if (N <= 0 || C <= 0 || H <= 0 || W <= 0) return fail(GG_ERR_BAD_ARG, "%s: sizes must be positive", what);
  if (levels < 1) return fail(GG_ERR_BAD_ARG, "%s: levels must be >= 1 (got %d)", what, levels);
  if (N > 65535) return fail(GG_ERR_UNSUPPORTED, "%s: batch > 65535", what);
  if (levels > 1) {
    if (H > 65535 * kTH) return fail(GG_ERR_UNSUPPORTED, "%s: height > %d (65535 row tiles of %d)", what, 65535 * kTH, kTH);
    if (!taps) return fail(GG_ERR_BAD_ARG, "%s: null taps", what);
    if (width < 1 || width % 2 == 0) return fail(GG_ERR_BAD_ARG, "%s: tap width must be odd and positive (got %d)", what, width);
    if (width > kMaxWidth) return fail(GG_ERR_UNSUPPORTED, "%s: tap width %d exceeds the cap of %d", what, width, kMaxWidth);
  }
  return GG_OK;
}

}  // namespace
}  // namespace gg

using namespace gg;

extern "C" {

int64_t gg_laplacian_blend_workspace(int64_t N, int C, int H, int W, int levels, int backward) {
  if (N <= 0 || C <= 0 || H <= 0 || W <= 0 || levels <= 1) return 0;
  const int64_t plane = N * static_cast<int64_t>(H) * W;
  if (!backward) return 4 * 2 * (2 * C + 1) * plane;                 // ping-pong A, B, M
  return 4 * (4 * C * plane + (2 * static_cast<int64_t>(levels) - 1) * plane);   // A/B ping-pong, M_1..M_{L-1}, d_0..d_{L-1}
}

int gg_laplacian_blend_forward(float* out, void* workspace, const float* img0, const float* img1, const float* mask,
                               const float* taps, int64_t N, int C, int H, int W, int levels, int width, void* stream) {
  int rc = check_args(N, C, H, W, levels, width, taps, "laplacian_blend_forward");
  if (rc) return rc;
  if (!out || !img0 || !img1 || !mask || (levels > 1 && !workspace))
    return fail(GG_ERR_BAD_ARG, "laplacian_blend_forward: null tensor");
  auto st = static_cast<cudaStream_t>(stream);
  const int64_t HW = static_cast<int64_t>(H) * W, total = N * C * HW;
  if (levels == 1) {
    blend_lerp_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(out, img0, img1, mask, C, HW, total);
    GG_CHECK_LAUNCH("laplacian_blend lerp launch");
    return GG_OK;
  }
  float* ws = static_cast<float*>(workspace);
  float* pa[2] = {ws, ws + total};
  float* pb[2] = {ws + 2 * total, ws + 3 * total};
  float* pm[2] = {ws + 4 * total, ws + 4 * total + N * HW};
  for (int l = 0; l < levels - 1; ++l) {
    LevelArgs a{};
    a.a_in = l ? pa[(l - 1) & 1] : img0;
    a.b_in = l ? pb[(l - 1) & 1] : img1;
    a.m_in = l ? pm[(l - 1) & 1] : mask;
    a.a_out = pa[l & 1]; a.b_out = pb[l & 1]; a.m_out = pm[l & 1];
    a.acc = out;
    a.taps = taps + static_cast<int64_t>(l) * width;
    a.width = width; a.C = C; a.H = H; a.W = W;
    a.first = l == 0; a.last = l == levels - 2;
    if ((rc = launch_level<BL_FWD>(a, N, st))) return rc;
  }
  return GG_OK;
}

int gg_laplacian_blend_backward(float* grad_img0, float* grad_img1, float* grad_mask, void* workspace,
                                const float* grad_out, const float* img0, const float* img1, const float* mask,
                                const float* taps, int64_t N, int C, int H, int W, int levels, int width, void* stream) {
  int rc = check_args(N, C, H, W, levels, width, taps, "laplacian_blend_backward");
  if (rc) return rc;
  if (!grad_img0 || !grad_img1 || !grad_mask || !grad_out || !img0 || !img1 || !mask || (levels > 1 && !workspace))
    return fail(GG_ERR_BAD_ARG, "laplacian_blend_backward: null tensor");
  auto st = static_cast<cudaStream_t>(stream);
  const int64_t HW = static_cast<int64_t>(H) * W, plane = N * HW, total = N * C * HW;
  if (levels == 1) {
    blend_lerp_bwd_kernel<<<static_cast<unsigned>((plane + 255) / 256), 256, 0, st>>>(
        grad_img0, grad_img1, grad_mask, grad_out, img0, img1, mask, C, HW, plane);
    GG_CHECK_LAUNCH("laplacian_blend lerp backward launch");
    return GG_OK;
  }
  float* ws = static_cast<float*>(workspace);
  float* pa[2] = {ws, ws + total};
  float* pb[2] = {ws + 2 * total, ws + 3 * total};
  float* mstack = ws + 4 * total;                          // M_l at mstack + (l-1) * plane, l = 1 .. L-1
  float* dstack = mstack + static_cast<int64_t>(levels - 1) * plane;   // d_l at dstack + l * plane, l = 0 .. L-1
  auto M = [&](int l) -> const float* { return l ? mstack + (l - 1) * plane : mask; };
  // forward sweep: mask stack and the mask's direct gradient per level
  for (int l = 0; l < levels - 1; ++l) {
    LevelArgs a{};
    a.a_in = l ? pa[(l - 1) & 1] : img0;
    a.b_in = l ? pb[(l - 1) & 1] : img1;
    a.m_in = M(l);
    a.a_out = pa[l & 1]; a.b_out = pb[l & 1]; a.m_out = mstack + static_cast<int64_t>(l) * plane;
    a.acc = dstack + static_cast<int64_t>(l) * plane;
    a.acc_last = dstack + static_cast<int64_t>(levels - 1) * plane;
    a.g = grad_out;
    a.taps = taps + static_cast<int64_t>(l) * width;
    a.width = width; a.C = C; a.H = H; a.W = W;
    a.first = l == 0; a.last = l == levels - 2;
    if ((rc = launch_level<BL_BWD_SWEEP>(a, N, st))) return rc;
  }
  // reverse Horner sweep
  blend_adj_init_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(
      pa[0], pb[0], grad_out, M(levels - 2), M(levels - 1), C, HW, total);
  GG_CHECK_LAUNCH("laplacian_blend adjoint init launch");
  int cur = 0;
  for (int l = levels - 2; l >= 0; --l) {
    LevelArgs a{};
    a.a_in = pa[cur]; a.b_in = pb[cur];
    a.m_in = dstack + static_cast<int64_t>(l + 1) * plane;     // U^M_{l+1} (d_{L-1} itself for the first step)
    float* um = l ? dstack + static_cast<int64_t>(l) * plane : grad_mask;   // U^M_l overwrites d_l in place
    a.a_out = l ? pa[cur ^ 1] : grad_img0;
    a.b_out = l ? pb[cur ^ 1] : grad_img1;
    a.m_out = um;
    a.d = dstack + static_cast<int64_t>(l) * plane;
    a.g = grad_out;
    a.m_prev = l ? M(l - 1) : nullptr;
    a.m_cur = M(l);
    a.taps = taps + static_cast<int64_t>(l) * width;
    a.width = width; a.C = C; a.H = H; a.W = W;
    a.first = l == 0;
    if ((rc = launch_level<BL_ADJ>(a, N, st))) return rc;
    cur ^= 1;
  }
  return GG_OK;
}

}  // extern "C"
