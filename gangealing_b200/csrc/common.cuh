// common.cuh -- shared device/host helpers for libgg_b200 (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdarg>
#include <cstdio>

#include "../../include/gg_b200.h"

namespace gg {

// ---------------------------------------------------------------- errors (thread-local message)
inline char* err_buf() {
  static thread_local char buf[512] = {0};
  return buf;
}
inline int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(err_buf(), 512, fmt, ap);
  va_end(ap);
  return code;
}
inline int cuda_fail(cudaError_t e, const char* what) {
  return fail(GG_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
}
// Check the launch only (cudaPeekAtLastError does not clear sticky state and does not sync).
#define GG_CHECK_LAUNCH(what)                               \
  do {                                                      \
    cudaError_t e__ = cudaPeekAtLastError();                \
    if (e__ != cudaSuccess) {                               \
      (void)cudaGetLastError();                             \
      return ::gg::cuda_fail(e__, what);                    \
    }                                                       \
  } while (0)

// Storage-type dispatch: runs the statement(s) with T_ bound to the C type of `dtype_`; any other code returns
// GG_ERR_UNSUPPORTED from the enclosing function.  GG_DISPATCH_T takes fp32 and bf16 (the channels-last kernels),
// GG_DISPATCH_T16 fp16 as well.
#define GG_DISPATCH_CASE_(code_, type_, ...) \
  case code_: { using T_ = type_; __VA_ARGS__; break; }
#define GG_DISPATCH_T(dtype_, who_, ...)                                                                             \
  switch (dtype_) {                                                                                                  \
    GG_DISPATCH_CASE_(GG_F32, float, __VA_ARGS__)                                                                    \
    GG_DISPATCH_CASE_(GG_BF16, __nv_bfloat16, __VA_ARGS__)                                                           \
    default: return ::gg::fail(GG_ERR_UNSUPPORTED, "%s: dtype %d not supported (fp32 or bf16)", who_, dtype_);       \
  }
#define GG_DISPATCH_T16(dtype_, who_, ...)                                                                           \
  switch (dtype_) {                                                                                                  \
    GG_DISPATCH_CASE_(GG_F32, float, __VA_ARGS__)                                                                    \
    GG_DISPATCH_CASE_(GG_F16, __half, __VA_ARGS__)                                                                   \
    GG_DISPATCH_CASE_(GG_BF16, __nv_bfloat16, __VA_ARGS__)                                                           \
    default: return ::gg::fail(GG_ERR_UNSUPPORTED, "%s: dtype %d not supported (fp32, fp16 or bf16)", who_, dtype_); \
  }

int sm_count();  // defined in api.cu

// True when `p` may be read as float4 / uint4.  Entry points whose kernels read a caller's pointer 16 bytes at a time
// refuse a misaligned one (GG_ERR_BAD_ARG) before any launch; a null pointer passes.
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// One-time per-DEVICE configuration guard (cudaFuncSetAttribute is a per-device attribute, so a process that drives a
// second GPU must opt in there too).  Usage:  static DeviceOnce once;  if (once.needed()) { ...; once.done(); }
struct DeviceOnce {
  unsigned long long mask[2] = {0ull, 0ull};   // up to 128 device ordinals; benign race: configuring twice is harmless
  int dev = 0;
  bool needed() {
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 128) return true;
    return ((__atomic_load_n(&mask[dev >> 6], __ATOMIC_ACQUIRE) >> (dev & 63)) & 1ull) == 0ull;
  }
  void done() {
    if (dev >= 0 && dev < 128) __atomic_fetch_or(&mask[dev >> 6], 1ull << (dev & 63), __ATOMIC_RELEASE);
  }
};

// ---------------------------------------------------------------- dtype traits (fp32 math)
template <typename T> struct Cvt;
template <> struct Cvt<float> {
  static __device__ __forceinline__ float to_f(float v) { return v; }
  static __device__ __forceinline__ float from_f(float v) { return v; }
};
template <> struct Cvt<__half> {
  static __device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
  static __device__ __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
};
template <> struct Cvt<__nv_bfloat16> {
  static __device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};

// 16-byte vector of T
template <typename T> struct alignas(16) Vec16 {
  static constexpr int N = 16 / sizeof(T);
  T v[N];
};

template <typename T>
__device__ __forceinline__ Vec16<T> ld_vec_stream(const T* p) {  // streaming 128-bit load
  Vec16<T> r;
  uint4 u;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w)
               : "l"(p));
  *reinterpret_cast<uint4*>(&r) = u;
  return r;
}
template <typename T>
__device__ __forceinline__ void st_vec_stream(T* p, const Vec16<T>& r) {
  const uint4 u = *reinterpret_cast<const uint4*>(&r);
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(u.x), "r"(u.y),
               "r"(u.z), "r"(u.w)
               : "memory");
}

// ---------------------------------------------------------------- 16-byte channel vectors as fp32 lanes
// A channels-last activation is read / written 16 bytes at a time: V = 4 channels of fp32 or 8 channels of bf16.
// Arithmetic is always fp32 (bf16 is a storage format here: BASELINE config 3 "bf16 activations, fp32 accumulate").
template <typename T> struct ChanVec;
template <> struct ChanVec<float> {
  static constexpr int V = 4;
  static __device__ __forceinline__ void unpack(const uint4& u, float (&f)[4]) {
    f[0] = __uint_as_float(u.x); f[1] = __uint_as_float(u.y); f[2] = __uint_as_float(u.z); f[3] = __uint_as_float(u.w);
  }
  static __device__ __forceinline__ uint4 pack(const float (&f)[4]) {
    return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
  }
};
template <> struct ChanVec<__nv_bfloat16> {
  static constexpr int V = 8;
  static __device__ __forceinline__ void unpack(const uint4& u, float (&f)[8]) {   // bf16 -> fp32 is a 16-bit shift
    f[0] = __uint_as_float(u.x << 16); f[1] = __uint_as_float(u.x & 0xffff0000u);
    f[2] = __uint_as_float(u.y << 16); f[3] = __uint_as_float(u.y & 0xffff0000u);
    f[4] = __uint_as_float(u.z << 16); f[5] = __uint_as_float(u.z & 0xffff0000u);
    f[6] = __uint_as_float(u.w << 16); f[7] = __uint_as_float(u.w & 0xffff0000u);
  }
  static __device__ __forceinline__ uint32_t pack2(float lo, float hi) {           // cvt.rn.bf16x2.f32
    const __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
  }
  static __device__ __forceinline__ uint4 pack(const float (&f)[8]) {
    return make_uint4(pack2(f[0], f[1]), pack2(f[2], f[3]), pack2(f[4], f[5]), pack2(f[6], f[7]));
  }
};
__device__ __forceinline__ uint4 ldg_stream16(const void* p) {       // read-once activation data: bypass L1
  uint4 u;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(p));
  return u;
}
__device__ __forceinline__ void stg_stream16(void* p, const uint4& u) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(u.x), "r"(u.y), "r"(u.z), "r"(u.w) : "memory");
}

// ---------------------------------------------------------------- sign mask of a channels-last activation
// One bit per element, `stored value > 0` (what lrelu' tests in the backward kernels), packed along the channels: word w of
// a pixel holds channels 32w .. 32w+31, bit = channel & 31; the tensor is (N, H, W, C/32) uint32.  A backward pass that
// needs no reduction over the activation reads the mask (1/32 or 1/16 of the bytes) instead of the activation.
// SignFloor<T>::v: the largest fp32 value whose STORED form is not positive.  bf16 rounds (0, 2^-134] to zero.
template <typename T> struct SignFloor { static constexpr float v = 0.f; };
template <> struct SignFloor<__nv_bfloat16> { static constexpr float v = 0x1p-134f; };

template <typename T, int V>
__device__ __forceinline__ uint32_t sign_bits(const float (&o)[V]) {
  uint32_t m = 0u;
#pragma unroll
  for (int k = 0; k < V; ++k) m |= (o[k] > SignFloor<T>::v ? 1u : 0u) << k;
  return m;
}
// The 32 / V adjacent lanes that own one word's channels (lane `cq` owns channels cq*V ..) combine their bits; every lane of
// `lanes` must call.  The word is complete in all of them; the lane with (cq*V) % 32 == 0 stores it.
template <int V>
__device__ __forceinline__ uint32_t sign_word(uint32_t bits, int cq, unsigned lanes) {
  constexpr int L = 32 / V;
  uint32_t w = bits << (V * (cq & (L - 1)));
#pragma unroll
  for (int m = L / 2; m >= 1; m >>= 1) w |= __shfl_xor_sync(lanes, w, m);
  return w;
}
// the V bits of channel vector `cq` (channels cq*V ..) of a pixel whose mask words start at `px`
template <int V>
__device__ __forceinline__ uint32_t sign_load(const uint32_t* px, int cq) {
  return __ldg(px + (cq * V >> 5)) >> (cq * V & 31);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------- mbarrier + bulk-TMA (cp.async.bulk)
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
// Bounded: a transfer that never completes (a bad tensor map, a faulted copy) traps after ~2^28 polls instead of
// hanging the GPU until the watchdog fires.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  uint32_t spins = 0;
  do {
    if (++spins == (1u << 28)) __trap();
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!done);
}
// 1-D bulk copy global -> shared, completion signalled on `bar` (SASS: UBLKCP).
// dst, src 16-byte aligned; bytes a multiple of 16.
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                             uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

}  // namespace gg
