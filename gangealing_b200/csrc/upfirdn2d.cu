// upfirdn2d.cu -- FIR resampling (upsample / pad / filter / decimate) for sm_90a.
//
// Two kernels:
//  * fir4_band_kernel: up = down = 1, filter <= 4x4 (every Blur on GANgealing's hot path,
//    reference upfirdn2d_kernel.cu "mode 1/2", :250-262).  A persistent CTA walks (plane, row-band)
//    work items; the input rows of a band are ONE contiguous span of global memory (full-width rows
//    of a dense plane), which a single elected thread moves with a 1-D bulk-TMA copy
//    (cp.async.bulk, SASS UBLKCP) into a 3-stage shared-memory ring signalled by mbarriers.  Rows of
//    these tensors are (2H+1)*4 bytes long, i.e. never 16-byte aligned, so the copy moves the
//    16-byte-aligned superset of the span and the consumers index through the residual shift.
//    Consumers keep a 4x4 register window per output column and slide it down the band, so every
//    input element is read from shared memory 4x (not 16x) and from HBM once (+3 halo rows/band).
//    The epilogue optionally fuses NoiseInjection + bias + leaky-ReLU + gain (+ per-plane scale):
//    the "fused upfirdn2d+bias-act path" -- one read and one write of the activation instead of
//    three of each (blur, noise add, bias-act) in the reference.
//    Algorithmic bytes/launch = s*M*(Hin*Win + Hout*Wout) [+ s*N*Hout*Wout noise + 4*(C+1+16)].
//  * upfirdn2d_generic_kernel: any up/down/pad/filter size (RGB skip up x2, its backward down x2,
//    5x5 test filters ...): one thread per output, polyphase tap walk, fp32 accumulate.
#include <algorithm>
#include <utility>

#include "common.cuh"

namespace gg {
namespace {

// ------------------------------------------------------------------------------------------------
// generic gather kernel
// ------------------------------------------------------------------------------------------------
struct GenericParams {
  int in_h, in_w, out_h, out_w;
  int kh, kw;
  int up_x, up_y, down_x, down_y;
  int pad_x0, pad_y0;
};

struct Epilogue {          // optional fused tail: lrelu(row_scale*t + nw*noise + bias) * scale
  const void* noise;       // (N, out_h, out_w), element type of the tensor, or null
  const float* noise_weight;
  const float* bias;       // (C)
  const float* row_scale;  // (N*C)
  int C;
  int act;
  float alpha, scale;
};

__device__ __forceinline__ int floordiv(int a, int b) {  // b > 0
  int q = a / b;
  return (q * b > a) ? q - 1 : q;
}
__device__ __forceinline__ int ceildiv_s(int a, int b) { return -floordiv(-a, b); }

// UPC / DNC: compile-time up / down factors (0 = runtime): the two resamplers of the hot path -- the to-RGB skip's x2
// up-sampling and its backward (x2 decimation), networks.py:28-46 -- divide by a constant (shifts instead of 4 integer
// divisions per output).
template <typename T, bool FUSED, int UPC = 0, int DNC = 0>
__global__ void __launch_bounds__(256)
upfirdn2d_generic_kernel(T* __restrict__ out, const T* __restrict__ in, const float* __restrict__ taps,
                         GenericParams p, Epilogue ep, int64_t total) {
  if (UPC) { p.up_x = UPC; p.up_y = UPC; }
  if (DNC) { p.down_x = DNC; p.down_y = DNC; }
  float nw = 0.f;
  if (FUSED) nw = ep.noise ? (ep.noise_weight ? __ldg(ep.noise_weight) : 1.f) : 0.f;
  // out[m, oy, ox] = sum_{ky,kx} U[oy*dy + ky, ox*dx + kx] * taps[kh-1-ky][kw-1-kx]
  // U = zero-inserted, padded input: U[y, x] = in[(y-pad_y0)/up_y, (x-pad_x0)/up_x] when divisible & in range.
  const bool small = total <= 0x7fffffffLL;     // 32-bit index arithmetic (a 64-bit div/mod pair costs more than the taps)
  for (int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    int ox, oy;
    int64_t m;
    if (small) {
      const unsigned i32 = static_cast<unsigned>(idx), t32 = i32 / static_cast<unsigned>(p.out_w);
      ox = static_cast<int>(i32 - t32 * static_cast<unsigned>(p.out_w));
      const unsigned m32 = t32 / static_cast<unsigned>(p.out_h);
      oy = static_cast<int>(t32 - m32 * static_cast<unsigned>(p.out_h));
      m = m32;
    } else {
      ox = static_cast<int>(idx % p.out_w);
      const int64_t t = idx / p.out_w;
      oy = static_cast<int>(t % p.out_h);
      m = t / p.out_h;
    }
    const int y0 = oy * p.down_y - p.pad_y0;  // U-row of ky = 0, in input*up coordinates
    const int x0 = ox * p.down_x - p.pad_x0;
    const int iy_lo = max(ceildiv_s(y0, p.up_y), 0);
    const int iy_hi = min(floordiv(y0 + p.kh - 1, p.up_y), p.in_h - 1);
    const int ix_lo = max(ceildiv_s(x0, p.up_x), 0);
    const int ix_hi = min(floordiv(x0 + p.kw - 1, p.up_x), p.in_w - 1);
    const T* plane = in + m * p.in_h * static_cast<int64_t>(p.in_w);
    float acc = 0.f;
    for (int iy = iy_lo; iy <= iy_hi; ++iy) {
      const int ky = iy * p.up_y - y0;
      const float* trow = taps + (p.kh - 1 - ky) * p.kw;
      const T* irow = plane + static_cast<int64_t>(iy) * p.in_w;
      for (int ix = ix_lo; ix <= ix_hi; ++ix) {
        const int kx = ix * p.up_x - x0;
        acc = fmaf(Cvt<T>::to_f(irow[ix]), __ldg(trow + (p.kw - 1 - kx)), acc);
      }
    }
    if (FUSED) {
      const int64_t n = m / ep.C;
      const int c = static_cast<int>(m - n * ep.C);
      float t = acc * (ep.row_scale ? __ldg(ep.row_scale + m) : 1.f) + (ep.bias ? __ldg(ep.bias + c) : 0.f);
      if (ep.noise)
        t = fmaf(nw, Cvt<T>::to_f(static_cast<const T*>(ep.noise)[(n * p.out_h + oy) * static_cast<int64_t>(p.out_w) + ox]), t);
      acc = t * ((ep.act == 3 && t < 0.f) ? ep.alpha * ep.scale : ep.scale);
    }
    out[idx] = Cvt<T>::from_f(acc);
  }
}

// ------------------------------------------------------------------------------------------------
// polyphase x2 resamplers (4x4 taps, fp32): the to-RGB skip's `Upsample` (up 2, pad (2,1): networks.py:28-46) and its
// backward (down 2, pad (1,1): upfirdn2d.py:111-116).  Of the 16 taps only a 2x2 phase touches a non-zero sample of the
// zero-inserted signal, so the up-sampler does 4 FMAs per output; a thread owns 2 input columns x 1 input row ->
// 2 rows x 4 columns of output (two 16-byte stores); the decimator owns 2 adjacent outputs (one 16-byte + 2 scalar
// loads per input row, one 8-byte store).  HBM-bound: 4*M*(5*H*W) bytes; neighbours are L1/L2 hits.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
up2_k4_kernel(float* __restrict__ out, const float* __restrict__ in, const float* __restrict__ taps, int64_t planes,
              int H, int W) {
  float f[4][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) f[i >> 2][i & 3] = __ldg(taps + i);
  const int wp = W >> 1;
  const int64_t total = planes * H * wp;
  for (int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int t = static_cast<int>(idx % wp);
    const int64_t q = idx / wp;
    const int j = static_cast<int>(q % H);
    const int64_t m = q / H;
    const float* p = in + (m * H + j) * static_cast<int64_t>(W) + 2 * t;
    float v[3][4];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int iy = j - 1 + r;
      const bool ok = iy >= 0 && iy < H;
      const float* row = p + (r - 1) * W;
      const float2 c = ok ? __ldg(reinterpret_cast<const float2*>(row)) : make_float2(0.f, 0.f);
      v[r][1] = c.x;
      v[r][2] = c.y;
      v[r][0] = (ok && t > 0) ? __ldg(row - 1) : 0.f;
      v[r][3] = (ok && 2 * t + 2 < W) ? __ldg(row + 2) : 0.f;
    }
    float* o = out + ((m * 2 * H + 2 * j) * static_cast<int64_t>(2 * W)) + 4 * t;
#pragma unroll
    for (int a = 0; a < 2; ++a) {        // output row 2j+a: input rows j-1+a+d' with tap row 3-a-2d'
      float r4[4];
#pragma unroll
      for (int ox = 0; ox < 4; ++ox) {   // output col 4t+ox: phase b = ox&1, first input col index (ox+1)>>1
        const int b = ox & 1, c0 = (ox + 1) >> 1;
        float acc = v[a][c0] * f[3 - a][3 - b];
        acc = fmaf(v[a][c0 + 1], f[3 - a][1 - b], acc);
        acc = fmaf(v[a + 1][c0], f[1 - a][3 - b], acc);
        acc = fmaf(v[a + 1][c0 + 1], f[1 - a][1 - b], acc);
        r4[ox] = acc;
      }
      __stcs(reinterpret_cast<float4*>(o + a * 2 * W), make_float4(r4[0], r4[1], r4[2], r4[3]));
    }
  }
}

__global__ void __launch_bounds__(256)
down2_k4_kernel(float* __restrict__ out, const float* __restrict__ in, const float* __restrict__ taps, int64_t planes,
                int Hi, int Wi) {
  float f[4][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) f[i >> 2][i & 3] = __ldg(taps + i);
  const int Ho = Hi >> 1, Wo = Wi >> 1, wp = Wo >> 1;
  const int64_t total = planes * Ho * wp;
  for (int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int t = static_cast<int>(idx % wp);
    const int64_t q = idx / wp;
    const int oy = static_cast<int>(q % Ho);
    const int64_t m = q / Ho;
    float o0 = 0.f, o1 = 0.f;
#pragma unroll
    for (int ky = 0; ky < 4; ++ky) {     // input row 2oy-1+ky, tap row 3-ky; cols 4t-1 .. 4t+4
      const int iy = 2 * oy - 1 + ky;
      if (iy < 0 || iy >= Hi) continue;
      const float* row = in + (m * Hi + iy) * static_cast<int64_t>(Wi) + 4 * t;
      const float4 c = __ldg(reinterpret_cast<const float4*>(row));
      const float l = t > 0 ? __ldg(row - 1) : 0.f;
      const float r = 4 * t + 4 < Wi ? __ldg(row + 4) : 0.f;
      const float* fr = f[3 - ky];
      o0 = fmaf(l, fr[3], fmaf(c.x, fr[2], fmaf(c.y, fr[1], fmaf(c.z, fr[0], o0))));
      o1 = fmaf(c.y, fr[3], fmaf(c.z, fr[2], fmaf(c.w, fr[1], fmaf(r, fr[0], o1))));
    }
    *reinterpret_cast<float2*>(out + (m * Ho + oy) * static_cast<int64_t>(Wo) + 2 * t) = make_float2(o0, o1);
  }
}

// ------------------------------------------------------------------------------------------------
// band kernel (up = down = 1, <= 4x4 taps)
// ------------------------------------------------------------------------------------------------
constexpr int kBandThreads = 256;
constexpr int kBandWarps = kBandThreads / 32;
constexpr int kStages = 3;
constexpr int kRS = 8;   // output rows per lane (the register window slides over kRS + 3 input rows)
constexpr int kCO = 4;   // adjacent output columns per lane (one 16-byte store for fp32)
constexpr int kGuard = 16;  // bytes in front of every slot, so columns -1..-3 of its first row are addressable

// A work item is `planes_per_item` consecutive planes x one band of output rows.  Each plane of the item owns a
// SLOT of the stage that holds the band's VIRTUAL input rows vy0 .. vy0 + vrows - 1 (vy0 = oy0 - pad_y0, vrows =
// band rows + 3) back to back at pitch in_w: the real rows arrive by one bulk-TMA copy of the 16-byte-aligned
// superset of their contiguous global span; rows outside the image (zero padding above/below) and the few foreign
// elements the aligned superset drags in are zero-filled by the CTA once the copy has landed.  Consumers therefore
// never test row validity: every input of every output is a plain shared-memory read.
struct BandParams {
  int64_t planes;        // M = N*C
  int in_h, in_w, out_h, out_w;
  int pad_x0, pad_y0;
  int band_rows;         // R: output rows per work item
  int bands;             // ceil(out_h / R)
  int planes_per_item;   // P (> 1 only when bands == 1)
  int slot_elems;        // elements per plane slot (multiple of 16 B)
  int stage_elems;       // P * slot_elems
  int lx_log2;           // lanes across a strip = 1 << lx_log2 (strip = 4*lanes columns)
  int vec_io;            // 1: out (and noise) rows are 16-byte aligned -> vector store / load
  // fused epilogue
  int C;                 // channels (plane m -> n = m / C, c = m % C)
  int act;               // 1 linear, 3 lrelu
  float alpha, scale;
};

constexpr int kMaxPlanesPerItem = 32;

struct Item {            // geometry shared by all planes of a work item
  int64_t m0;            // first plane
  int n_planes;
  int oy0, rows;         // output rows of the band
  int vy0, vrows;        // virtual input rows held by a slot
  int lo, nreal;         // real input rows [lo, lo + nreal) (nreal <= 0: the band sees only padding)
  int d0;                // element offset of the copy destination inside a slot (multiple of 16 B)
};

struct ItemS {           // what the producer thread publishes per stage (shared memory)
  Item it;
  int v0[kMaxPlanesPerItem];   // slot position of (virtual row vy0, column 0), per plane
};

__device__ __forceinline__ Item item_geom(const BandParams& p, int64_t item, int elem_size) {
  Item it;
  if (p.bands == 1) {
    it.m0 = item * p.planes_per_item;
    it.n_planes = static_cast<int>(min(static_cast<int64_t>(p.planes_per_item), p.planes - it.m0));
    it.oy0 = 0;
    it.rows = p.out_h;
  } else {
    it.m0 = item / p.bands;
    it.n_planes = 1;
    it.oy0 = static_cast<int>(item - it.m0 * p.bands) * p.band_rows;
    it.rows = min(p.band_rows, p.out_h - it.oy0);
  }
  it.vy0 = it.oy0 - p.pad_y0;
  it.vrows = it.rows + 3;
  it.lo = max(it.vy0, 0);
  const int hi = min(it.vy0 + it.vrows - 1, p.in_h - 1);
  it.nreal = hi - it.lo + 1;
  const int per16 = 16 / elem_size;
  const int n_top = (it.nreal > 0 ? it.lo : it.vy0 + it.vrows) - it.vy0;   // zero rows above the first real row
  it.d0 = (kGuard / elem_size + n_top * p.in_w + per16 - 1) / per16 * per16;
  return it;
}

template <typename T>
struct PlaneCopy {       // bulk copy of one plane's real rows
  const T* src;          // 16-byte aligned
  uint32_t bytes;        // multiple of 16
  int shift;             // elements between src and the first real element
};

template <typename T>
__device__ __forceinline__ PlaneCopy<T> plane_copy(const T* in, const BandParams& p, const Item& it, int pl) {
  PlaneCopy<T> c;
  const T* first = in + ((it.m0 + pl) * p.in_h + it.lo) * static_cast<int64_t>(p.in_w);
  const T* last = first + static_cast<int64_t>(it.nreal) * p.in_w;  // one past
  const uintptr_t a0 = reinterpret_cast<uintptr_t>(first) & ~static_cast<uintptr_t>(15);
  const uintptr_t a1 = (reinterpret_cast<uintptr_t>(last) + 15) & ~static_cast<uintptr_t>(15);
  c.src = reinterpret_cast<const T*>(a0);
  c.bytes = static_cast<uint32_t>(a1 - a0);
  c.shift = static_cast<int>((reinterpret_cast<uintptr_t>(first) - a0) / sizeof(T));
  return c;
}

// issued by one thread: publish the item's geometry, arm the barrier with the item's total bytes, then one
// bulk copy per plane
template <typename T>
__device__ __forceinline__ void issue_item(const T* in, const BandParams& p, int64_t item, T* stage, uint64_t* bar,
                                           ItemS* pub) {
  const Item it = item_geom(p, item, sizeof(T));
  pub->it = it;
  if (it.nreal <= 0) {
    for (int pl = 0; pl < it.n_planes; ++pl) pub->v0[pl] = it.d0 - it.vrows * p.in_w;
    return;
  }
  uint32_t total = 0;
  for (int pl = 0; pl < it.n_planes; ++pl) {
    const PlaneCopy<T> c = plane_copy(in, p, it, pl);
    total += c.bytes;
    pub->v0[pl] = it.d0 + c.shift - (it.lo - it.vy0) * p.in_w;
  }
  // the stage was last touched through the generic proxy (zero-fill stores, reads): order them before the
  // async-proxy writes of the copies
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  mbar_expect_tx(bar, total);
  for (int pl = 0; pl < it.n_planes; ++pl) {
    const PlaneCopy<T> c = plane_copy(in, p, it, pl);
    tma_bulk_g2s(stage + static_cast<int64_t>(pl) * p.slot_elems + it.d0, c.src, c.bytes, bar);
  }
}

template <typename T> struct Vec4 { T v[4]; };

// Generic-type lane (any T, separable or full 16-tap filter): 4 adjacent output columns x up to kRS rows with a
// register window sliding down.  `vrow0` points at virtual row vy0, column 0 of this plane's slot.
template <typename T, bool SEP, bool FUSED>
__device__ __forceinline__ void lane_strip(T* __restrict__ out_plane, const T* __restrict__ vrow0, int vy0,
                                           const T* __restrict__ noise_plane, const BandParams& p,
                                           const float (&kf)[4][4], const float (&ku)[4], const float (&kv)[4],
                                           int oys, int nrow, int x0, float rs, float bc, float nw) {
  const int colbase = x0 - p.pad_x0;
  int cidx[kCO + 3];
  uint32_t cmask[kCO + 3];
#pragma unroll
  for (int i = 0; i < kCO + 3; ++i) {
    const int c = colbase + i;
    cidx[i] = min(max(c, 0), p.in_w - 1);
    cmask[i] = (c >= 0 && c < p.in_w) ? 0xffffffffu : 0u;
  }
  const int iys = oys - p.pad_y0;
  float win[4][SEP ? kCO : kCO + 3];
#pragma unroll
  for (int r = 0; r < kRS + 3; ++r) {
    if (r < nrow + 3) {
      const T* trow = vrow0 + static_cast<int64_t>(iys + r - vy0) * p.in_w;
      float raw[kCO + 3];
#pragma unroll
      for (int i = 0; i < kCO + 3; ++i)
        raw[i] = __uint_as_float(__float_as_uint(Cvt<T>::to_f(trow[cidx[i]])) & cmask[i]);
      if (SEP) {
#pragma unroll
        for (int j = 0; j < kCO; ++j)
          win[r & 3][j] = fmaf(kv[3], raw[j + 3], fmaf(kv[2], raw[j + 2], fmaf(kv[1], raw[j + 1], kv[0] * raw[j])));
      } else {
#pragma unroll
        for (int i = 0; i < kCO + 3; ++i) win[r & 3][i] = raw[i];
      }
      if (r >= 3) {
        const int ro = r - 3;
        float acc[kCO];
#pragma unroll
        for (int j = 0; j < kCO; ++j) {
          if (SEP) {
            acc[j] = fmaf(ku[3], win[(ro + 3) & 3][j],
                          fmaf(ku[2], win[(ro + 2) & 3][j], fmaf(ku[1], win[(ro + 1) & 3][j], ku[0] * win[ro & 3][j])));
          } else {
            float a_ = 0.f;
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
              for (int b = 0; b < 4; ++b) a_ = fmaf(win[(ro + a) & 3][j + b], kf[a][b], a_);
            acc[j] = a_;
          }
          if (FUSED) {
            float t = fmaf(acc[j], rs, bc);
            if (noise_plane && x0 + j < p.out_w)
              t = fmaf(nw, Cvt<T>::to_f(noise_plane[static_cast<int64_t>(oys + ro) * p.out_w + x0 + j]), t);
            const float g = (p.act == 3 && t < 0.f) ? p.alpha * p.scale : p.scale;
            acc[j] = t * g;
          }
        }
        T* op = out_plane + static_cast<int64_t>(oys + ro) * p.out_w + x0;
        if (p.vec_io) {
          Vec4<T> o;
#pragma unroll
          for (int j = 0; j < kCO; ++j) o.v[j] = Cvt<T>::from_f(acc[j]);
          *reinterpret_cast<Vec4<T>*>(op) = o;
        } else {
#pragma unroll
          for (int j = 0; j < kCO; ++j)
            if (x0 + j < p.out_w) op[j] = Cvt<T>::from_f(acc[j]);
        }
      }
    }
  }
}

// fp32 + separable filter fast path.  A slot holds its virtual rows as one flat array, so element (row, col) sits
// at flat position pos = row*in_w + col + const, whose 16-byte alignment rotates from row to row (in_w is odd on
// the hot path).  Each lane reads the 16-byte-aligned quads covering its 7 inputs (LDS.128, consecutive lanes ->
// consecutive quads: conflict-free).  Which registers feed the horizontal pass depends on pos mod 4, which is
// WARP-UNIFORM and, given the alignment S0 of the strip's first row and IW4 = in_w mod 4, a compile-time
// constant per unrolled row: the kernel is instantiated per IW4 and branches once per task on S0, so the inner
// loop is straight-line FMA code: no row/column tests, shuffles, selects or per-value address arithmetic.
// Out-of-range columns are handled by folding a 0/1 mask into per-lane horizontal weights, so the elements they
// touch must be finite: plan_band admits only pads whose stored outputs read columns -3 .. in_w + 2, i.e. real
// neighbours in the flat slot or the 3 zero-filled elements in front of the first / behind the last virtual row.
template <int IW4, int S0, bool FUSED, bool VEC>
struct StripF32 {
  float* __restrict__ out_ptr;        // &out[plane][oys][x0]
  const float* __restrict__ row_ptr;  // slot element (row oys - pad_y0, column x0 - pad_x0), NOT aligned
  const BandParams& p;
  const float (&ku)[4];
  float wgt[kCO][4];
  float4 nz[kRS];
  float hw[4][kCO];
  int nrow, x0;
  float rs, bc, nw, gpos, gdiff;
  bool has_noise;

  template <int R>
  __device__ __forceinline__ void step() {
    constexpr int SH = (S0 + R * IW4) & 3;       // alignment of this row's first input (compile-time)
    const float4* qp = reinterpret_cast<const float4*>(row_ptr + R * p.in_w - SH);
    const float4 q0 = qp[0], q1 = qp[1];
    float4 q2 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (SH >= 2) q2 = qp[2];                     // inputs SH .. SH+6 reach the third quad only when SH >= 2
    const float Q[12] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w};
#pragma unroll
    for (int j = 0; j < kCO; ++j)
      hw[R & 3][j] = fmaf(wgt[j][3], Q[SH + j + 3],
                          fmaf(wgt[j][2], Q[SH + j + 2], fmaf(wgt[j][1], Q[SH + j + 1], wgt[j][0] * Q[SH + j])));
    if (R >= 3) {
      constexpr int RO = R >= 3 ? R - 3 : 0;
      float acc[kCO];
#pragma unroll
      for (int j = 0; j < kCO; ++j) {
        acc[j] = fmaf(ku[3], hw[(RO + 3) & 3][j],
                      fmaf(ku[2], hw[(RO + 2) & 3][j], fmaf(ku[1], hw[(RO + 1) & 3][j], ku[0] * hw[RO & 3][j])));
        if (FUSED) {
          float t = fmaf(acc[j], rs, bc);
          if (has_noise) {
            const float4 nv4 = nz[RO < kRS ? RO : 0];
            const float nv = j == 0 ? nv4.x : (j == 1 ? nv4.y : (j == 2 ? nv4.z : nv4.w));
            t = fmaf(nw, nv, t);
          }
          // lrelu(t)*scale = scale*t + (alpha*scale - scale)*min(t, 0): one ALU op + two FMA-pipe ops
          acc[j] = fmaf(gdiff, fminf(t, 0.f), gpos * t);
        }
      }
      if (RO < nrow) {
        float* op = out_ptr + static_cast<int64_t>(RO) * p.out_w;
        if (VEC) {
          *reinterpret_cast<float4*>(op) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        } else {
#pragma unroll
          for (int j = 0; j < kCO; ++j)
            if (x0 + j < p.out_w) op[j] = acc[j];
        }
      }
    }
  }

  template <int... Rs>
  __device__ __forceinline__ void run(std::integer_sequence<int, Rs...>) {
    (step<Rs>(), ...);
  }
};

template <int IW4, int S0, bool FUSED, bool VEC>
__device__ __forceinline__ void lane_strip_f32(float* __restrict__ out_plane, const float* __restrict__ row_ptr,
                                               const float* __restrict__ noise_plane, const BandParams& p,
                                               const float (&ku)[4], const float (&kv)[4], int oys, int nrow, int x0,
                                               float rs, float bc, float nw) {
  StripF32<IW4, S0, FUSED, VEC> st{out_plane + static_cast<int64_t>(oys) * p.out_w + x0, row_ptr, p, ku};
  st.nrow = nrow; st.x0 = x0;
  st.rs = rs; st.bc = bc; st.nw = nw; st.has_noise = FUSED && noise_plane != nullptr;
  st.gpos = p.scale; st.gdiff = (p.act == 3) ? p.alpha * p.scale - p.scale : 0.f;
  const int colbase = x0 - p.pad_x0;
#pragma unroll
  for (int j = 0; j < kCO; ++j)
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int c = colbase + j + b;
      st.wgt[j][b] = (c >= 0 && c < p.in_w) ? kv[b] : 0.f;
    }
  if (FUSED && noise_plane) {
#pragma unroll
    for (int r = 0; r < kRS; ++r) {
      st.nz[r] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < nrow) {
        const float* np_ = noise_plane + static_cast<int64_t>(oys + r) * p.out_w + x0;
        if (VEC) {
          st.nz[r] = __ldg(reinterpret_cast<const float4*>(np_));
        } else {
          if (x0 + 0 < p.out_w) st.nz[r].x = __ldg(np_ + 0);
          if (x0 + 1 < p.out_w) st.nz[r].y = __ldg(np_ + 1);
          if (x0 + 2 < p.out_w) st.nz[r].z = __ldg(np_ + 2);
          if (x0 + 3 < p.out_w) st.nz[r].w = __ldg(np_ + 3);
        }
      }
    }
  }
  st.run(std::make_integer_sequence<int, kRS + 3>{});
}

template <typename T, int IW4, bool FUSED>
__global__ void __launch_bounds__(kBandThreads, 2)
fir4_band_kernel(T* __restrict__ out, const T* __restrict__ in, const float* __restrict__ filt, int kh,
                 int kw, const T* __restrict__ noise, const float* __restrict__ noise_weight,
                 const float* __restrict__ bias, const float* __restrict__ row_scale,
                 const __grid_constant__ BandParams p, int64_t n_items) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ uint64_t full_bar[kStages];
  __shared__ ItemS pub[kStages];
  T* stage_base = reinterpret_cast<T*>(smem_raw);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) mbar_init(&full_bar[s], 1);
    mbar_fence_init();
  }
  __syncthreads();

  const int64_t stride = gridDim.x;
  // prologue: fill kStages-1 stages (issued before the tap set-up below so the copies fly meanwhile)
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < kStages - 1; ++s) {
      const int64_t it = blockIdx.x + s * stride;
      if (it < n_items) issue_item(in, p, it, stage_base + static_cast<int64_t>(s) * p.stage_elems, &full_bar[s], &pub[s]);
    }
  }

  // flipped 4x4 taps in registers: kf[a][b] multiplies input (oy + a - pad_y0, ox + b - pad_x0)
  float kf[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
      kf[a][b] = (a < kh && b < kw) ? __ldg(filt + (kh - 1 - a) * kw + (kw - 1 - b)) : 0.f;  // flipped: true convolution
  // rank-1 test: kf == ku (x) kv within 1e-6 of the largest tap -> separable fast path (every Blur in
  // GANgealing: [1,3,3,1] (x) [1,3,3,1], exactly representable)
  float ku[4], kv[4];
  bool sep;
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
    float dev = 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) dev = fmaxf(dev, fabsf(kf[a][b] - ku[a] * kv[b]));
    sep = dev <= 1e-6f * big;
  }

  float nw = 0.f;
  if (FUSED) nw = noise ? (noise_weight ? __ldg(noise_weight) : 1.f) : 0.f;
  __syncthreads();  // the prologue's published item geometry is visible to every thread

  // strip geometry: `full_x` strips of lx lanes x 4 columns, plus one narrower tail strip whose lanes
  // are folded down the rows instead (so 129- or 65-wide outputs do not pay for a second full strip)
  const int lx_main = 1 << p.lx_log2;
  const int full_x = p.out_w / (lx_main * kCO);
  const int tail_w = p.out_w - full_x * lx_main * kCO;
  int lt_log2 = 0;
  while ((1 << lt_log2) * kCO < tail_w) ++lt_log2;

  uint32_t phase_bits = 0;  // bit s: parity the next wait on stage s must observe
  int k = 0;                // local iteration counter
  for (int64_t item = blockIdx.x; item < n_items; item += stride, ++k) {
    const int stage = k % kStages;
    // prefetch the item kStages-1 ahead into the stage freed by the previous iteration
    if (tid == 0) {
      const int64_t nxt = item + (kStages - 1) * stride;
      if (nxt < n_items) {
        const int ns = (k + kStages - 1) % kStages;
        issue_item(in, p, nxt, stage_base + static_cast<int64_t>(ns) * p.stage_elems, &full_bar[ns], &pub[ns]);
      }
    }
    // geometry published by the producer (visible: written before the previous iteration's / the prologue's barrier)
    const Item& it = pub[stage].it;
    if (it.nreal > 0) {  // a padding-only band issues no transfer, so its stage's phase does not advance
      mbar_wait(&full_bar[stage], (phase_bits >> stage) & 1u);
      phase_bits ^= 1u << stage;
    }
    T* stage_ptr = stage_base + static_cast<int64_t>(stage) * p.stage_elems;   // 16-byte aligned
    // zero padding rows above / below the image (first / last band of a plane only)
    const int n_top = it.nreal > 0 ? it.lo - it.vy0 : it.vrows;
    const int n_bot = it.nreal > 0 ? it.vrows - n_top - it.nreal : 0;
    if (n_top > 0 || n_bot > 0) {
      for (int pl = 0; pl < it.n_planes; ++pl) {
        T* slot = stage_ptr + static_cast<int64_t>(pl) * p.slot_elems;
        const int v0 = pub[stage].v0[pl];
        const int first_real = v0 + n_top * p.in_w;
        const int after_real = first_real + max(it.nreal, 0) * p.in_w;
        for (int e = v0 + tid; e < first_real; e += kBandThreads) slot[e] = Cvt<T>::from_f(0.f);
        for (int e = after_real + tid; e < v0 + it.vrows * p.in_w; e += kBandThreads) slot[e] = Cvt<T>::from_f(0.f);
      }
      __syncthreads();
    }

    const int sy_main = (it.rows + (32 >> p.lx_log2) * kRS - 1) / ((32 >> p.lx_log2) * kRS);
    const int main_tasks = full_x * sy_main;
    const int tail_tasks = tail_w > 0 ? (it.rows + (32 >> lt_log2) * kRS - 1) / ((32 >> lt_log2) * kRS) : 0;
    const int tasks_per_plane = main_tasks + tail_tasks;
    const int n_tasks = tasks_per_plane * it.n_planes;
    for (int task = warp; task < n_tasks; task += kBandWarps) {
      const int pl = task / tasks_per_plane;
      const int rem = task - pl * tasks_per_plane;
      int sy, xs, lg;  // strip row, first column of the strip, log2(lanes across)
      if (rem < main_tasks) {
        sy = rem / full_x;
        xs = (rem - sy * full_x) * lx_main * kCO;
        lg = p.lx_log2;
      } else {
        sy = rem - main_tasks;
        xs = full_x * lx_main * kCO;
        lg = lt_log2;
      }
      const int lane_x = lane & ((1 << lg) - 1);
      const int lane_y = lane >> lg;
      const int64_t m = it.m0 + pl;
      const int oys = it.oy0 + (sy * (32 >> lg) + lane_y) * kRS;
      const int nrow = min(kRS, it.oy0 + it.rows - oys);
      const int x0 = xs + lane_x * kCO;
      if (nrow <= 0 || x0 >= p.out_w) continue;
      float rs = 1.f, bc = 0.f;
      const T* noise_plane = nullptr;
      if (FUSED) {
        const int64_t n = m / p.C;
        const int c = static_cast<int>(m - n * p.C);
        if (row_scale) rs = __ldg(row_scale + m);
        if (bias) bc = __ldg(bias + c);
        if (noise) noise_plane = noise + n * p.out_h * static_cast<int64_t>(p.out_w);
      }
      T* out_plane = out + m * p.out_h * static_cast<int64_t>(p.out_w);
      T* slot = stage_ptr + static_cast<int64_t>(pl) * p.slot_elems;
      const int v0 = pub[stage].v0[pl];
      // The 3 elements in front of the first virtual row and behind the last one are foreign (alignment
      // prefix / suffix of the copy, or never written): only the lanes below ever touch them (with zero
      // weight), so those lanes make them finite zeros themselves -- no extra barrier.
      if (x0 == 0 && oys == it.oy0) {
#pragma unroll
        for (int e = 1; e <= 3; ++e) slot[v0 - e] = Cvt<T>::from_f(0.f);
      }
      if (x0 + kCO + 3 - p.pad_x0 > p.in_w && oys + kRS >= it.oy0 + it.rows) {
        const int vend = v0 + it.vrows * p.in_w;
#pragma unroll
        for (int e = 0; e < 3; ++e) slot[vend + e] = Cvt<T>::from_f(0.f);
      }
      if constexpr (sizeof(T) == 4 && IW4 >= 0) {
        if (sep) {
          const int pos0 = v0 + (oys - p.pad_y0 - it.vy0) * p.in_w + (x0 - p.pad_x0);
          const float* row_ptr = reinterpret_cast<const float*>(slot) + pos0;
#define GG_STRIP(S0_, V_)                                                                                    \
  lane_strip_f32<IW4, S0_, FUSED, V_>(reinterpret_cast<float*>(out_plane), row_ptr,                             \
                                      reinterpret_cast<const float*>(noise_plane), p, ku, kv, oys, nrow, x0, rs, \
                                      bc, nw)
          if (p.vec_io) {
            switch (pos0 & 3) {   // warp-uniform: lanes differ by multiples of 4 columns / 8 rows
              case 0: GG_STRIP(0, true); break;
              case 1: GG_STRIP(1, true); break;
              case 2: GG_STRIP(2, true); break;
              default: GG_STRIP(3, true); break;
            }
          } else {
            switch (pos0 & 3) {
              case 0: GG_STRIP(0, false); break;
              case 1: GG_STRIP(1, false); break;
              case 2: GG_STRIP(2, false); break;
              default: GG_STRIP(3, false); break;
            }
          }
#undef GG_STRIP
          continue;
        }
      }
      if (sep)
        lane_strip<T, true, FUSED>(out_plane, slot + v0, it.vy0, noise_plane, p, kf, ku, kv, oys, nrow, x0, rs, bc, nw);
      else
        lane_strip<T, false, FUSED>(out_plane, slot + v0, it.vy0, noise_plane, p, kf, ku, kv, oys, nrow, x0, rs, bc, nw);
    }
    __syncthreads();  // every warp is done with `stage` (and its published geometry) before it is refilled
  }
}

inline int dtype_size(int dtype) { return dtype == GG_F32 ? 4 : 2; }

// host-side geometry for the band kernel; returns false when the shape is better served by the generic kernel
struct BandPlan {
  BandParams p;
  size_t smem_bytes;
  int64_t n_items;
  int grid;
};

inline bool plan_band(int dtype, int64_t planes, int in_h, int in_w, int out_h, int out_w, int pad_x0,
                      int pad_y0, const void* out, const void* noise, BandPlan* plan) {
  if (out_w < 24 || out_h < 8) return false;  // tiny planes: launch-bound, one thread per output is as good
  // A stored output column ox reads input columns ox - pad_x0 .. ox - pad_x0 + 3 (zero taps included).  The fp32
  // separable path weights out-of-range columns by zero instead of masking them, so each must be a real neighbour
  // or one of the 3 zero-filled elements in front of / behind a slot's virtual rows: columns -3 .. in_w + 2.
  // Wider pads (pad_x0 > 3, or pad_x1 + 4 - kernel_w > 3) go to the generic kernel.
  if (pad_x0 > 3 || out_w - pad_x0 > in_w) return false;
  const int es = dtype_size(dtype);
  const int per16 = 16 / es;
  int lx_log2 = 5;
  while (lx_log2 > 0 && (1 << (lx_log2 - 1)) * kCO >= out_w) --lx_log2;
  const int lx = 1 << lx_log2, ly = 32 >> lx_log2;
  const int strip_w = lx * kCO, strip_h = ly * kRS;
  const int strips_x = out_w / strip_w > 0 ? out_w / strip_w : 1;  // full strips (the tail strip folds down the rows)
  const int64_t budget = 36 * 1024;  // bytes per stage (3 stages x 2 CTAs per SM)
  auto slot_elems_for = [&](int rows) {   // guard + virtual rows + alignment slack + trailing guard, 16-byte multiple
    // a partial last strip still walks kRS + 3 input rows (its surplus outputs are never stored): round rows up
    const int rows8 = (rows + kRS - 1) / kRS * kRS;
    const int64_t e = kGuard / es + static_cast<int64_t>(rows8 + 3) * in_w + 2 * per16 + 4;
    return (e + per16 - 1) / per16 * per16;
  };
  BandParams& p = plan->p;
  int r, bands, ppi = 1;
  if (slot_elems_for(out_h) * es <= budget) {           // whole planes per item, several when small
    r = out_h; bands = 1;
    const int strips_y = (out_h + strip_h - 1) / strip_h;
    const int tasks = strips_x * strips_y;
    ppi = (kBandWarps + tasks - 1) / tasks;
    const int64_t fit = budget / (slot_elems_for(out_h) * es);
    if (ppi > fit) ppi = static_cast<int>(fit);
    if (ppi < 1) ppi = 1;
    if (ppi > planes) ppi = static_cast<int>(planes);
    if (ppi > kMaxPlanesPerItem) ppi = kMaxPlanesPerItem;
  } else {
    // warp tasks per band: strips_x * R/strip_h; aim for >= 8 tasks within the budget
    r = strip_h * ((kBandWarps + strips_x - 1) / strips_x);
    while (r > strip_h && slot_elems_for(r) * es > budget) r -= strip_h;
    if (slot_elems_for(r) * es > 64 * 1024) return false;  // rows too wide for the ring
    if (r >= out_h) return false;
    bands = (out_h + r - 1) / r;
  }
  const int64_t slot_elems = slot_elems_for(r);
  const size_t smem = static_cast<size_t>(slot_elems) * ppi * es * kStages;
  if (smem > 200 * 1024) return false;
  p.planes = planes; p.in_h = in_h; p.in_w = in_w; p.out_h = out_h; p.out_w = out_w;
  p.pad_x0 = pad_x0; p.pad_y0 = pad_y0;
  p.band_rows = r; p.bands = bands; p.planes_per_item = ppi;
  p.slot_elems = static_cast<int>(slot_elems);
  p.stage_elems = static_cast<int>(slot_elems * ppi);
  p.lx_log2 = lx_log2;
  const uintptr_t align = static_cast<uintptr_t>(4 * es);
  p.vec_io = (out_w % 4 == 0) && (reinterpret_cast<uintptr_t>(out) % align == 0) &&
             (noise == nullptr || reinterpret_cast<uintptr_t>(noise) % align == 0);
  p.C = 1; p.act = 1; p.alpha = 0.f; p.scale = 1.f;
  plan->smem_bytes = smem;
  plan->n_items = (bands == 1) ? (planes + ppi - 1) / ppi : planes * bands;
  const int ctas_per_sm = smem * 2 <= 220 * 1024 ? 2 : 1;
  const int64_t max_grid = static_cast<int64_t>(sm_count()) * ctas_per_sm;
  int64_t grid = plan->n_items < max_grid ? plan->n_items : max_grid;
  // The fp32 fast path has one code variant per 16-byte alignment class of a plane's rows.  A persistent CTA strides
  // over items by gridDim.x; rounding the grid down so that the stride is a whole number of 4 planes keeps every CTA
  // on ONE alignment class, i.e. one hot code variant in its instruction cache instead of a rotation of four.
  const int64_t unit = static_cast<int64_t>(bands) * 4;
  if (grid >= 2 * unit) grid = grid / unit * unit;
  plan->grid = static_cast<int>(grid);
  return true;
}

template <typename T, int IW4, bool FUSED>
int launch_band_t(const BandPlan& pl, void* out, const void* in, const float* filt, int kh, int kw, const void* noise,
                  const float* nw, const float* bias, const float* row_scale, cudaStream_t st) {
  auto kern = fir4_band_kernel<T, IW4, FUSED>;
  static DeviceOnce configured;
  if (configured.needed()) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(200 * 1024));
    if (e != cudaSuccess) return cuda_fail(e, "fir4_band smem opt-in");
    configured.done();
  }
  kern<<<pl.grid, kBandThreads, pl.smem_bytes, st>>>(
      static_cast<T*>(out), static_cast<const T*>(in), filt, kh, kw, static_cast<const T*>(noise), nw, bias,
      row_scale, pl.p, pl.n_items);
  GG_CHECK_LAUNCH("fir4_band launch");
  return GG_OK;
}

template <bool FUSED>
int launch_band(int dtype, const BandPlan& pl, void* out, const void* in, const float* filt, int kh, int kw,
                const void* noise, const float* nw, const float* bias, const float* row_scale,
                cudaStream_t st) {
  switch (dtype) {
    case GG_F32:
      switch (pl.p.in_w & 3) {  // row-to-row alignment rotation is a template parameter of the fp32 fast path
        case 0: return launch_band_t<float, 0, FUSED>(pl, out, in, filt, kh, kw, noise, nw, bias, row_scale, st);
        case 1: return launch_band_t<float, 1, FUSED>(pl, out, in, filt, kh, kw, noise, nw, bias, row_scale, st);
        case 2: return launch_band_t<float, 2, FUSED>(pl, out, in, filt, kh, kw, noise, nw, bias, row_scale, st);
        default: return launch_band_t<float, 3, FUSED>(pl, out, in, filt, kh, kw, noise, nw, bias, row_scale, st);
      }
    case GG_F16: return launch_band_t<__half, -1, FUSED>(pl, out, in, filt, kh, kw, noise, nw, bias, row_scale, st);
    case GG_BF16: return launch_band_t<__nv_bfloat16, -1, FUSED>(pl, out, in, filt, kh, kw, noise, nw, bias, row_scale, st);
    default: return fail(GG_ERR_UNSUPPORTED, "upfirdn2d: dtype %d not supported (f32/f16/bf16)", dtype);
  }
}

template <typename T>
int launch_generic_t(void* out, const void* in, const float* filt, const GenericParams& gp, const Epilogue* ep,
                     int64_t total, cudaStream_t st) {
  int64_t grid = (total + 255) / 256;
  const int64_t cap = static_cast<int64_t>(sm_count()) * 32;
  if (grid > cap) grid = cap;
  if (ep)
    upfirdn2d_generic_kernel<T, true><<<static_cast<unsigned>(grid), 256, 0, st>>>(
        static_cast<T*>(out), static_cast<const T*>(in), filt, gp, *ep, total);
  else if (gp.up_x == 2 && gp.up_y == 2 && gp.down_x == 1 && gp.down_y == 1)
    upfirdn2d_generic_kernel<T, false, 2, 1><<<static_cast<unsigned>(grid), 256, 0, st>>>(
        static_cast<T*>(out), static_cast<const T*>(in), filt, gp, Epilogue{}, total);
  else if (gp.up_x == 1 && gp.up_y == 1 && gp.down_x == 2 && gp.down_y == 2)
    upfirdn2d_generic_kernel<T, false, 1, 2><<<static_cast<unsigned>(grid), 256, 0, st>>>(
        static_cast<T*>(out), static_cast<const T*>(in), filt, gp, Epilogue{}, total);
  else
    upfirdn2d_generic_kernel<T, false><<<static_cast<unsigned>(grid), 256, 0, st>>>(
        static_cast<T*>(out), static_cast<const T*>(in), filt, gp, Epilogue{}, total);
  GG_CHECK_LAUNCH("upfirdn2d_generic launch");
  return GG_OK;
}

inline int launch_generic(int dtype, void* out, const void* in, const float* filt, const GenericParams& gp,
                          const Epilogue* ep, int64_t total, cudaStream_t st) {
  switch (dtype) {
    case GG_F32: return launch_generic_t<float>(out, in, filt, gp, ep, total, st);
    case GG_F16: return launch_generic_t<__half>(out, in, filt, gp, ep, total, st);
    default: return launch_generic_t<__nv_bfloat16>(out, in, filt, gp, ep, total, st);
  }
}

inline int check_common(const char* who, const void* out, const void* in, const float* kernel, int dtype,
                        int64_t major, int in_h, int in_w, int kh, int kw, int up_x, int up_y, int down_x,
                        int down_y, int out_h, int out_w) {
  if (major < 0 || in_h < 0 || in_w < 0) return fail(GG_ERR_BAD_ARG, "%s: negative size", who);
  if (kh < 1 || kw < 1) return fail(GG_ERR_BAD_ARG, "%s: empty filter", who);
  if (up_x < 1 || up_y < 1 || down_x < 1 || down_y < 1) return fail(GG_ERR_BAD_ARG, "%s: up/down must be >= 1", who);
  if (out_h < 1 || out_w < 1) return fail(GG_ERR_BAD_ARG, "%s: output would be empty (%d x %d)", who, out_h, out_w);
  if (dtype != GG_F32 && dtype != GG_F16 && dtype != GG_BF16)
    return fail(GG_ERR_UNSUPPORTED, "%s: dtype %d not supported (f32/f16/bf16)", who, dtype);
  if (major > 0 && (!out || !in || !kernel)) return fail(GG_ERR_BAD_ARG, "%s: null tensor", who);
  return GG_OK;
}

}  // namespace
}  // namespace gg

using namespace gg;

extern "C" {

int gg_upfirdn2d(void* out, const void* in, const float* kernel, int dtype, int64_t major, int in_h,
                 int in_w, int kernel_h, int kernel_w, int up_x, int up_y, int down_x, int down_y,
                 int pad_x0, int pad_x1, int pad_y0, int pad_y1, void* stream) {
  // out size: reference upfirdn2d.py:103-104 / upfirdn2d_kernel.cu:236-239
  const int out_h = (up_y >= 1 && down_y >= 1 && kernel_h >= 1) ? (in_h * up_y + pad_y0 + pad_y1 - kernel_h) / down_y + 1 : 0;
  const int out_w = (up_x >= 1 && down_x >= 1 && kernel_w >= 1) ? (in_w * up_x + pad_x0 + pad_x1 - kernel_w) / down_x + 1 : 0;
  if (in_h * up_y + pad_y0 + pad_y1 - kernel_h < 0 || in_w * up_x + pad_x0 + pad_x1 - kernel_w < 0)
    return fail(GG_ERR_BAD_ARG, "upfirdn2d: filter larger than padded input");
  int rc = check_common("upfirdn2d", out, in, kernel, dtype, major, in_h, in_w, kernel_h, kernel_w, up_x, up_y,
                        down_x, down_y, out_h, out_w);
  if (rc != GG_OK) return rc;
  if (major == 0) return GG_OK;
  auto st = static_cast<cudaStream_t>(stream);
  if (up_x == 1 && up_y == 1 && down_x == 1 && down_y == 1 && kernel_h <= 4 && kernel_w <= 4 && in_h > 0 &&
      in_w > 0) {
    BandPlan pl;
    if (plan_band(dtype, major, in_h, in_w, out_h, out_w, pad_x0, pad_y0, out, nullptr, &pl))
      return launch_band<false>(dtype, pl, out, in, kernel, kernel_h, kernel_w, nullptr, nullptr, nullptr,
                                nullptr, st);
  }
  // polyphase fast paths of the to-RGB skip (fp32 planes, 4x4 taps): x2 up with pad (2,1), x2 down with pad (1,1)
  const bool aligned16 = ((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(in)) & 15) == 0;
  if (dtype == GG_F32 && kernel_h == 4 && kernel_w == 4 && aligned16 && in_h > 0 && in_w > 0) {
    const int cap = sm_count() * 16;
    if (up_x == 2 && up_y == 2 && down_x == 1 && down_y == 1 && pad_x0 == 2 && pad_y0 == 2 && pad_x1 == 1 && pad_y1 == 1 &&
        (in_w & 1) == 0) {
      const int64_t work = major * in_h * (in_w >> 1);
      const int grid = static_cast<int>(std::min<int64_t>((work + 255) / 256, cap));
      up2_k4_kernel<<<grid, 256, 0, st>>>(static_cast<float*>(out), static_cast<const float*>(in), kernel, major, in_h, in_w);
      GG_CHECK_LAUNCH("upfirdn2d x2 up-sampler launch");
      return GG_OK;
    }
    if (up_x == 1 && up_y == 1 && down_x == 2 && down_y == 2 && pad_x0 == 1 && pad_y0 == 1 && pad_x1 == 1 && pad_y1 == 1 &&
        (in_w & 3) == 0 && (in_h & 1) == 0) {
      const int64_t work = major * (in_h >> 1) * (in_w >> 2);
      const int grid = static_cast<int>(std::min<int64_t>((work + 255) / 256, cap));
      down2_k4_kernel<<<grid, 256, 0, st>>>(static_cast<float*>(out), static_cast<const float*>(in), kernel, major, in_h, in_w);
      GG_CHECK_LAUNCH("upfirdn2d x2 decimator launch");
      return GG_OK;
    }
  }
  GenericParams gp{in_h, in_w, out_h, out_w, kernel_h, kernel_w, up_x, up_y, down_x, down_y, pad_x0, pad_y0};
  const int64_t total = major * out_h * static_cast<int64_t>(out_w);
  return launch_generic(dtype, out, in, kernel, gp, nullptr, total, st);
}

int gg_blur_noise_bias_act(void* out, const void* in, const float* kernel, const void* noise,
                           const float* noise_weight, const float* bias, const float* row_scale,
                           int dtype, int64_t N, int64_t C, int in_h, int in_w, int kernel_h,
                           int kernel_w, int pad_x0, int pad_x1, int pad_y0, int pad_y1, int act,
                           float alpha, float scale, void* stream) {
  if (N < 0 || C < 0) return fail(GG_ERR_BAD_ARG, "blur_noise_bias_act: negative size");
  if (act != 1 && act != 3) return fail(GG_ERR_UNSUPPORTED, "blur_noise_bias_act: act must be 1 or 3");
  if (kernel_h > 4 || kernel_w > 4) return fail(GG_ERR_UNSUPPORTED, "blur_noise_bias_act: filter larger than 4x4");
  const int out_h = in_h + pad_y0 + pad_y1 - kernel_h + 1;
  const int out_w = in_w + pad_x0 + pad_x1 - kernel_w + 1;
  const int64_t major = N * C;
  int rc = check_common("blur_noise_bias_act", out, in, kernel, dtype, major, in_h, in_w, kernel_h, kernel_w,
                        1, 1, 1, 1, out_h, out_w);
  if (rc != GG_OK) return rc;
  if (major == 0) return GG_OK;
  if (in_h == 0 || in_w == 0) return fail(GG_ERR_BAD_ARG, "blur_noise_bias_act: empty input plane");
  BandPlan pl;
  if (!plan_band(dtype, major, in_h, in_w, out_h, out_w, pad_x0, pad_y0, out, noise, &pl)) {
    // tiny or very wide planes: generic gather kernel with the same fused epilogue
    GenericParams gp{in_h, in_w, out_h, out_w, kernel_h, kernel_w, 1, 1, 1, 1, pad_x0, pad_y0};
    Epilogue ep{noise, noise_weight, bias, row_scale, static_cast<int>(C), act, alpha, scale};
    return launch_generic(dtype, out, in, kernel, gp, &ep, major * out_h * static_cast<int64_t>(out_w),
                          static_cast<cudaStream_t>(stream));
  }
  pl.p.C = static_cast<int>(C);
  pl.p.act = act;
  pl.p.alpha = alpha;
  pl.p.scale = scale;
  return launch_band<true>(dtype, pl, out, in, kernel, kernel_h, kernel_w, noise, noise_weight, bias,
                           row_scale, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
