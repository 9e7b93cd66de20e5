// Weight-freeze and calibration kernels: the step BEFORE the quantized-linear hot path (SURVEY.md 8f rank 1 and 2).
//
//   quantize_affine            -- quanto::quantize_affine, optimum/quanto/library/quantize.py:58-78 (3-5 ATen launches)
//   pack                       -- pack_weights, optimum/quanto/tensor/packed.py:24-69 (python loop of shift+or launches)
//   quantize_qbits_max         -- MaxOptimizer (tensor/optimizers/max_optimizer.py:26-37, affine_optimizer.py:52-63)
//                                 + quantize_affine + pack_weights for an axis-0 grouped weight as ONE launch:
//                                 reads the float weight once (2 B/weight), writes 0.5 B/weight + scale/shift
//   absmax                     -- calibrate.py:37-61 absmax_scale, per-tensor reduction
//   absmax_update              -- absmax_scale + the Calibration scale update (calibrate.py:31-34), in place, one launch
//   quantize_qbytes_absmax     -- AbsmaxOptimizer (tensor/optimizers/absmax_optimizer.py:29-36) + quantize_symmetric
//                                 (library/quantize.py:51-55) for an axis-0 8-bit weight as ONE launch
//
// All bit-exact with the reference's CPU arithmetic (see quantize_math.cuh); HBM-bound; launched on the caller's stream.
#include "../../include/quanto_b200.h"

#include "host_common.cuh"
#include "quantize_math.cuh"

namespace qb {

constexpr int kFzThreads = 256;

// ---------------------------------------------------------------------------------------------------------------
// quantize_affine (unfused): base viewed as [outer, inner] (already grouped); scale/shift index = row (axis_mode 1),
// column (axis_mode 2) or 0 (axis_mode 0).  shift: T, or uint8 zero-points when ZP.
// ---------------------------------------------------------------------------------------------------------------
template <typename T, bool ZP, int VEC>
__global__ void __launch_bounds__(kFzThreads)
    quantize_affine_kernel(const T* __restrict__ base, const T* __restrict__ scale, const void* __restrict__ shift,
                           uint8_t* __restrict__ out, int64_t numel, int64_t inner, int axis_mode, float qmax,
                           int zp_signed) {
  const int64_t n_items = (numel + VEC - 1) / VEC;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  // zero-points: the reference adds the VALUE of the integer tensor (library/quantize.py:74-76), so an int8 tensor may
  // carry negative zero-points (a group whose minimum is positive) and a uint8 tensor values up to 255
  auto load_z = [&](int64_t i) -> float {
    if constexpr (ZP) {
      const uint8_t b = static_cast<const uint8_t*>(shift)[i];
      return zp_signed ? static_cast<float>(static_cast<int8_t>(b)) : static_cast<float>(b);
    } else {
      return to_float<T>(static_cast<const T*>(shift)[i]);
    }
  };
  for (int64_t it = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; it < n_items; it += stride) {
    const int64_t e0 = it * VEC;
    float f[VEC];
    if constexpr (VEC == 8) load8_stream<T>(base + e0, f);  // host guarantees inner % 8 == 0: one row per vector
    else f[0] = to_float<T>(base[e0]);
    const int64_t i0 = (axis_mode == 1) ? (e0 / inner) : ((axis_mode == 2) ? (e0 % inner) : 0);
    float s = to_float<T>(scale[i0]);
    float z = load_z(i0);
    alignas(8) uint8_t q[VEC];
    bool done = false;
    if constexpr (VEC == 8) {
      if (axis_mode != 2) {  // one scale / shift for the whole vector
        uint32_t b8[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
        if (rcp_is_safe<T>(s)) affine_quantize8<T, ZP, true>(f, s, __frcp_rn(s), z, static_cast<int>(qmax), 0, b8);
        else affine_quantize8<T, ZP, false>(f, s, 0.f, z, static_cast<int>(qmax), 0, b8);
#pragma unroll
        for (int j = 0; j < 8; ++j) q[j] = static_cast<uint8_t>(b8[j]);
        done = true;
      }
    }
    if (!done) {
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        if (axis_mode == 2 && j > 0) {
          s = to_float<T>(scale[i0 + j]);
          z = load_z(i0 + j);
        }
        q[j] = static_cast<uint8_t>(affine_quantize_one<T, ZP>(f[j], s, z, qmax));
      }
    }
    if constexpr (VEC == 8) __stcs(reinterpret_cast<uint2*>(out + e0), *reinterpret_cast<uint2*>(q));
    else out[e0] = q[0];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// pack: out[i] = OR_p (in[p * plane + i] << bits*p) truncated to a byte, i < plane = R * cols, R = ceil(rows / planes);
// source bytes beyond rows*cols count as zero (the reference ORs a shorter last slice, packed.py:64-67).
// No masking of the inputs: like the reference, out-of-range values spill into the higher planes.
// ---------------------------------------------------------------------------------------------------------------
template <int BITS>
__global__ void __launch_bounds__(kFzThreads)
    pack_vec_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, int64_t plane_vecs, int64_t total_vecs) {
  constexpr int PLANES = 8 / BITS;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < plane_vecs; i += stride) {
    uint4 v[PLANES];
#pragma unroll
    for (int p = 0; p < PLANES; ++p) {
      const int64_t idx = static_cast<int64_t>(p) * plane_vecs + i;
      v[p] = (idx < total_vecs) ? __ldcs(in + idx) : make_uint4(0u, 0u, 0u, 0u);
    }
    uint4 acc = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (int p = 0; p < PLANES; ++p) {
      const uint32_t keep = ((0xFFu << (BITS * p)) & 0xFFu) * 0x01010101u;  // per-byte wrap of the uint8 shift
      acc.x |= (v[p].x << (BITS * p)) & keep;
      acc.y |= (v[p].y << (BITS * p)) & keep;
      acc.z |= (v[p].z << (BITS * p)) & keep;
      acc.w |= (v[p].w << (BITS * p)) & keep;
    }
    __stcs(out + i, acc);
  }
}

template <int BITS>
__global__ void __launch_bounds__(kFzThreads)
    pack_scalar_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int64_t plane, int64_t total) {
  constexpr int PLANES = 8 / BITS;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < plane; i += stride) {
    uint32_t acc = 0;
#pragma unroll
    for (int p = 0; p < PLANES; ++p) {
      const int64_t idx = static_cast<int64_t>(p) * plane + i;
      if (idx < total) acc |= (static_cast<uint32_t>(in[idx]) << (BITS * p)) & 0xFFu;
    }
    out[i] = static_cast<uint8_t>(acc);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// quantize_qbits_max: fused MaxOptimizer + quantize_affine + pack_weights, axis 0.
// The weight [N, K] viewed as grouped rows [rows = N*K/G, G] (tensor/grouped.py:17-30: a pure reshape for axis 0).
// Packed row pr holds grouped rows pr + p * packed_rows, p < 8/BITS, in its bit planes (tensor/packed.py:45-69).
// A team of TL lanes owns one packed row: each lane takes 8 consecutive columns of every plane's row (16-byte loads),
// the team reduces min / max with xor shuffles, every lane derives the row's scale / shift redundantly, quantises its
// 8 columns of each plane and stores 8 packed bytes.  TL = the power of two >= G/8 (lanes past G/8 idle).
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
struct Raw8 {  // 8 elements of T as loaded: one 16-byte vector (fp16/bf16) or two (fp32)
  uint4 v[sizeof(T) == 2 ? 1 : 2];
};

template <typename T>
__device__ __forceinline__ Raw8<T> load_raw8(const T* __restrict__ p) {
  Raw8<T> r;
  r.v[0] = __ldcs(reinterpret_cast<const uint4*>(p));
  if constexpr (sizeof(T) == 4) r.v[1] = __ldcs(reinterpret_cast<const uint4*>(p) + 1);
  return r;
}

template <typename T>
__device__ __forceinline__ void widen8(const Raw8<T>& r, float (&f)[8]) {
  if constexpr (sizeof(T) == 2) {
    const T* e = reinterpret_cast<const T*>(&r.v[0]);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = to_float<T>(e[j]);
  } else {
    f[0] = __uint_as_float(r.v[0].x); f[1] = __uint_as_float(r.v[0].y); f[2] = __uint_as_float(r.v[0].z);
    f[3] = __uint_as_float(r.v[0].w); f[4] = __uint_as_float(r.v[1].x); f[5] = __uint_as_float(r.v[1].y);
    f[6] = __uint_as_float(r.v[1].z); f[7] = __uint_as_float(r.v[1].w);
  }
}

template <typename T, int BITS, bool ZP, int TL>
__global__ void __launch_bounds__(kFzThreads, BITS == 4 ? 4 : 2)
    quantize_qbits_max_kernel(const T* __restrict__ base, uint8_t* __restrict__ packed, T* __restrict__ scale,
                              void* __restrict__ shift, int64_t rows, int64_t packed_rows, int group) {
  constexpr int PLANES = 8 / BITS;
  constexpr float QMAX = static_cast<float>((1 << BITS) - 1);
  constexpr int TEAMS_PER_WARP = 32 / TL;
  const int lane = threadIdx.x & 31;
  const int team_in_warp = lane / TL;
  const int col0 = (lane % TL) * 8;
  const bool lane_active = col0 < group;
  const int64_t warp_global = static_cast<int64_t>(blockIdx.x) * (kFzThreads / 32) + (threadIdx.x >> 5);
  const int64_t step = static_cast<int64_t>(gridDim.x) * (kFzThreads / 32) * TEAMS_PER_WARP;

  // the rows of packed row `pr` this lane reads (zeros where the row does not exist)
  auto fetch = [&](int64_t pr, Raw8<T> (&raw)[PLANES]) {
#pragma unroll
    for (int p = 0; p < PLANES; ++p) {
      const int64_t row = pr + static_cast<int64_t>(p) * packed_rows;
      if (pr < packed_rows && row < rows && lane_active) {
        raw[p] = load_raw8<T>(base + row * group + col0);
      } else {
        raw[p].v[0] = make_uint4(0u, 0u, 0u, 0u);
        if constexpr (sizeof(T) == 4) raw[p].v[1] = make_uint4(0u, 0u, 0u, 0u);
      }
    }
  };

  // the loop bound is uniform per warp (full-mask shuffles inside); the next packed row's loads are issued before
  // the current one is processed so that each thread keeps 2 x PLANES x 16 B in flight
  int64_t p0 = warp_global * TEAMS_PER_WARP;
  Raw8<T> cur[PLANES];
  if (p0 < packed_rows) fetch(p0 + team_in_warp, cur);
  for (; p0 < packed_rows; p0 += step) {
    const int64_t pr = p0 + team_in_warp;
    const bool team_valid = pr < packed_rows;
    Raw8<T> nxt[PLANES];
    if (p0 + step < packed_rows) fetch(pr + step, nxt);
    constexpr bool PACKED_BF16 = std::is_same<T, __nv_bfloat16>::value;
    uint32_t bytes[8];    // generic path: one quantised value per element, planes or-ed in
    uint32_t acc[4];      // bf16 path: elements (2i, 2i+1) in bytes 0 and 2 of acc[i]
#pragma unroll
    for (int j = 0; j < 8; ++j) bytes[j] = 0u;
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] = 0u;
#pragma unroll
    for (int p = 0; p < PLANES; ++p) {
      const int64_t row = pr + static_cast<int64_t>(p) * packed_rows;
      const bool row_valid = team_valid && row < rows;
      float lo = __int_as_float(0x7f800000), hi = __int_as_float(0xff800000);  // +inf / -inf
      float f[8];
      if constexpr (PACKED_BF16) {
        // (min, -max) of the lane's 8 values in ONE bf16x2 register: the team reduction is then one shuffle and one
        // packed min per round instead of two of each (max(x) = -min(-x), exact)
        uint32_t red = 0x7F807F80u;  // (+inf, +inf): neutral for inactive lanes / missing rows
        if (row_valid && lane_active) {
          const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&cur[p].v[0]);
          const __nv_bfloat162 mn = __hmin2(__hmin2(h[0], h[1]), __hmin2(h[2], h[3]));
          const __nv_bfloat162 nx = __hneg2(__hmax2(__hmax2(h[0], h[1]), __hmax2(h[2], h[3])));
          const __nv_bfloat162 both = __hmin2(__halves2bfloat162(__low2bfloat16(mn), __low2bfloat16(nx)),
                                              __halves2bfloat162(__high2bfloat16(mn), __high2bfloat16(nx)));
          red = *reinterpret_cast<const uint32_t*>(&both);
        }
#pragma unroll
        for (int off = TL / 2; off > 0; off >>= 1) {
          const uint32_t other = __shfl_xor_sync(0xffffffffu, red, off);
          const __nv_bfloat162 m = __hmin2(*reinterpret_cast<const __nv_bfloat162*>(&red),
                                           *reinterpret_cast<const __nv_bfloat162*>(&other));
          red = *reinterpret_cast<const uint32_t*>(&m);
        }
        lo = __uint_as_float(red << 16);
        hi = -__uint_as_float(red & 0xFFFF0000u);
      } else {
        widen8<T>(cur[p], f);
        if (row_valid && lane_active) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            lo = fminf(lo, f[j]);
            hi = fmaxf(hi, f[j]);
          }
        }
#pragma unroll
        for (int off = TL / 2; off > 0; off >>= 1) {
          lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, off));
          hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, off));
        }
      }
      // scale = rnd(rnd(hi - lo) / (2^bits - 1)), shift = -lo          (max_optimizer.py:31-36)
      // bf16: rnd(d * rcp(qmax)) == rnd(d / qmax) for every normal quotient (checked exhaustively over all bf16 d for
      // qmax = 15 and 3; the general argument is in quantize_math.cuh), so the IEEE division runs only for tiny ranges
      const float d = rnd<T>(__fsub_rn(hi, lo));
      float s;
      if (PACKED_BF16 && d > 1e-30f) s = rnd<T>(__fmul_rn(d, 1.0f / QMAX));
      else s = rnd<T>(__fdiv_rn(d, QMAX));
      const bool fast = rcp_is_safe<T>(s);
      const float r = fast ? __frcp_rn(s) : 0.f;
      float z = -lo;
      if constexpr (ZP) {
        // shift = clamp(round(shift / scale), 0, 2^bits - 1) as uint8    (affine_optimizer.py:59-62); NaN -> 0
        const float zq = fast ? rnd<T>(__fmul_rn(z, r)) : rnd<T>(__fdiv_rn(z, s));
        z = fminf(fmaxf(rintf(zq), 0.f), QMAX);
      }
      if (row_valid) {
        if (lane_active) {
          if constexpr (PACKED_BF16) {
            if (fast) {
              // All in packed bf16 except the product with the fp32 reciprocal (quantize_math.cuh explains why each step
              // equals the reference's fp32-then-round sequence): b + z is one exact-then-rounded bf16 add; the quotient
              // is widened, multiplied, rounded back as a pair; clamp o rint = rint o clamp (integer bounds; max before
              // min so that NaN -> lower bound -> 0 like the reference's cast); rint rides on one bf16 add of 192: in
              // [128, 256) the bf16 ulp is 1, so the sum's 7 mantissa bits are 64 + rint(t).  The zero-point is added to
              // that integer afterwards (folding it into the 192 would flip half-to-even ties when zp is odd); both
              // 16-bit lanes at once: every lane holds 64 + n >= 64 - zp, so the subtraction never borrows.
              const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&cur[p].v[0]);
              const __nv_bfloat162 zadd = __float2bfloat162_rn(ZP ? 0.f : z);
              const __nv_bfloat162 cl_lo = __float2bfloat162_rn(ZP ? -z : 0.f);
              const __nv_bfloat162 cl_hi = __float2bfloat162_rn(ZP ? QMAX - z : QMAX);
              const __nv_bfloat162 magic = __float2bfloat162_rn(192.f);
              const uint32_t bias2 = (64u - (ZP ? static_cast<uint32_t>(z) : 0u)) * 0x00010001u;
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                __nv_bfloat162 a = h[i];
                if constexpr (!ZP) a = __hadd2_rn(a, zadd);
                const __nv_bfloat162 t = __floats2bfloat162_rn(__fmul_rn(__low2float(a), r), __fmul_rn(__high2float(a), r));
                const __nv_bfloat162 m = __hadd2_rn(__hmin2(__hmax2(t, cl_lo), cl_hi), magic);
                acc[i] |= ((*reinterpret_cast<const uint32_t*>(&m) & 0x007F007Fu) - bias2) << (BITS * p);
              }
            } else {
              uint32_t tmp[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
              widen8<T>(cur[p], f);
              affine_quantize8<T, ZP, false>(f, s, 0.f, z, static_cast<int>(QMAX), BITS * p, tmp);
#pragma unroll
              for (int i = 0; i < 4; ++i) acc[i] |= tmp[2 * i] | (tmp[2 * i + 1] << 16);
            }
          } else {
            if (fast) affine_quantize8<T, ZP, true>(f, s, r, z, static_cast<int>(QMAX), BITS * p, bytes);
            else affine_quantize8<T, ZP, false>(f, s, 0.f, z, static_cast<int>(QMAX), BITS * p, bytes);
          }
        }
        if ((lane % TL) == 0) {
          scale[row] = from_float<T>(s);
          if constexpr (ZP) static_cast<uint8_t*>(shift)[row] = static_cast<uint8_t>(z);
          else static_cast<T*>(shift)[row] = from_float<T>(z);
        }
      }
    }
    if (team_valid && lane_active) {
      uint2 o;
      if constexpr (PACKED_BF16) {
        o.x = __byte_perm(acc[0], acc[1], 0x6420);
        o.y = __byte_perm(acc[2], acc[3], 0x6420);
      } else {
        o.x = bytes[0] | (bytes[1] << 8) | (bytes[2] << 16) | (bytes[3] << 24);
        o.y = bytes[4] | (bytes[5] << 8) | (bytes[6] << 16) | (bytes[7] << 24);
      }
      __stcs(reinterpret_cast<uint2*>(packed + pr * group + col0), o);
    }
#pragma unroll
    for (int p = 0; p < PLANES; ++p) cur[p] = nxt[p];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// absmax (per tensor): out[0] = max |base| as float32.  Non-negative floats order like their bit patterns, so the
// cross-CTA step is one atomicMax on the int view; `out` is zeroed on the stream by the launcher.
// ---------------------------------------------------------------------------------------------------------------
// max that PROPAGATES NaN (max.NaN.f32), as torch.max / amax do (calibrate.py:54-57, absmax_optimizer.py:29-36): a NaN
// activation or weight yields a NaN scale in the reference, and must here too (fmaxf would silently drop it)
__device__ __forceinline__ float nanmax(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

__device__ __forceinline__ float block_max_256(float m, float* red) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) m = nanmax(m, __shfl_xor_sync(0xffffffffu, m, off));
  __syncthreads();  // red[] may still be read by the previous use
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  float r = red[0];
#pragma unroll
  for (int w = 1; w < kFzThreads / 32; ++w) r = nanmax(r, red[w]);
  return r;
}

// One thread's max |base[i]| over its grid-stride share: 16-byte vector loads when `vec_ok` (base 16-byte aligned) with
// a scalar tail, scalar loads otherwise.
template <typename T>
__device__ __forceinline__ float thread_absmax(const T* __restrict__ base, int64_t numel, int vec_ok) {
  const int64_t tid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  float m = 0.f;
  if (vec_ok) {
    const int64_t n_vec = numel / 8;
    int64_t v = tid;
    for (; v + stride < n_vec; v += 2 * stride) {  // two independent 16-byte loads in flight per thread
      float f[8], g[8];
      load8_stream<T>(base + v * 8, f);
      load8_stream<T>(base + (v + stride) * 8, g);
#pragma unroll
      for (int j = 0; j < 8; ++j) m = nanmax(m, nanmax(fabsf(f[j]), fabsf(g[j])));
    }
    if (v < n_vec) {
      float f[8];
      load8_stream<T>(base + v * 8, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) m = nanmax(m, fabsf(f[j]));
    }
    for (int64_t i = n_vec * 8 + tid; i < numel; i += stride) m = nanmax(m, fabsf(to_float<T>(base[i])));
  } else {
    for (int64_t i = tid; i < numel; i += stride) m = nanmax(m, fabsf(to_float<T>(base[i])));
  }
  return m;
}

// Thread 0 of each CTA folds the CTA's maximum `m` into scratch[0] (bit pattern of a non-negative float; a NaN's
// pattern is the largest of all, so the integer atomicMax propagates it) and takes a ticket from scratch[1].  Returns
// true in the last CTA only, with *total = the maximum over the whole grid.
__device__ __forceinline__ bool publish_absmax(float m, int* __restrict__ scratch, float* total) {
  atomicMax(scratch, __float_as_int(m));
  __threadfence();
  const int done = atomicAdd(scratch + 1, 1);
  if (done != static_cast<int>(gridDim.x) - 1) return false;
  __threadfence();
  *total = __int_as_float(atomicMax(scratch, 0));
  return true;
}

template <typename T>
__global__ void __launch_bounds__(kFzThreads)
    absmax_kernel(const T* __restrict__ base, T* __restrict__ out, int* __restrict__ scratch, int64_t numel, int vec_ok) {
  __shared__ float red[kFzThreads / 32];
  const float m = block_max_256(thread_absmax<T>(base, numel, vec_ok), red);
  float total;
  // the last CTA publishes the result in T, so the caller needs no conversion launch
  if (threadIdx.x == 0 && publish_absmax(m, scratch, &total)) out[0] = from_float<T>(total);
}

// ---------------------------------------------------------------------------------------------------------------
// absmax_update: one calibration step of a per-tensor scale, in place (optimum/quanto/calibrate.py:31-34 with
// absmax_scale, :37-61).  The last CTA evaluates, each rounding to T where the reference's ATen ops round:
//   new   = rnd(max / qmax)                                         (true division, as absmax_scale)
//   scale = scale == 1 ? new : rnd(rnd(scale * m) + rnd(new * om))  (m = float(momentum), om = float(1 - momentum))
// The `scale == 1` test is read here on the device: the reference's torch.all(scale == 1) is a host synchronisation.
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kFzThreads)
    absmax_update_kernel(const T* __restrict__ base, T* __restrict__ scale, int* __restrict__ scratch, int64_t numel,
                         int vec_ok, float qmax, float m, float om) {
  __shared__ float red[kFzThreads / 32];
  const float bm = block_max_256(thread_absmax<T>(base, numel, vec_ok), red);
  float total;
  if (threadIdx.x == 0 && publish_absmax(bm, scratch, &total)) {
    const float fresh = rnd<T>(__fdiv_rn(total, qmax));
    const float old = to_float<T>(scale[0]);
    const float upd = old == 1.f ? fresh : rnd<T>(__fadd_rn(rnd<T>(__fmul_rn(old, m)), rnd<T>(__fmul_rn(fresh, om))));
    scale[0] = from_float<T>(upd);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// quantize_qbytes_absmax: per out-feature row, scale = rnd(max|w| / qmax), data = quantize_symmetric(w, scale).
// One CTA per row (grid-stride over rows); the second pass re-reads the row the CTA has just streamed (L1/L2 hit).
// ---------------------------------------------------------------------------------------------------------------
template <typename T, int OUT_DT>
__global__ void __launch_bounds__(kFzThreads)
    quantize_qbytes_absmax_kernel(const T* __restrict__ base, uint8_t* __restrict__ out, T* __restrict__ scale,
                                  int64_t n_rows, int64_t k, float qmax, int vec_ok) {
  __shared__ float red[kFzThreads / 32];
  const int tid = threadIdx.x;
  for (int64_t row = blockIdx.x; row < n_rows; row += gridDim.x) {
    const T* src = base + row * k;
    uint8_t* dst = out + row * k;
    float m = 0.f;
    if (vec_ok) {
      for (int64_t v = tid; v < k / 8; v += kFzThreads) {
        const uint4 r = *reinterpret_cast<const uint4*>(src + v * 8);  // default caching: read again below
        float f[8];
        if constexpr (sizeof(T) == 2) {
          const T* e = reinterpret_cast<const T*>(&r);
#pragma unroll
          for (int j = 0; j < 8; ++j) f[j] = to_float<T>(e[j]);
        } else {
          const uint4 r2 = *(reinterpret_cast<const uint4*>(src + v * 8) + 1);
          f[0] = __uint_as_float(r.x); f[1] = __uint_as_float(r.y); f[2] = __uint_as_float(r.z); f[3] = __uint_as_float(r.w);
          f[4] = __uint_as_float(r2.x); f[5] = __uint_as_float(r2.y); f[6] = __uint_as_float(r2.z); f[7] = __uint_as_float(r2.w);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) m = nanmax(m, fabsf(f[j]));
      }
    } else {
      for (int64_t i = tid; i < k; i += kFzThreads) m = nanmax(m, fabsf(to_float<T>(src[i])));
    }
    m = block_max_256(m, red);
    const float s = rnd<T>(__fdiv_rn(m, qmax));  // absmax_optimizer.py:36: rmax / qtype.qmax, rounded to T
    if (tid == 0) scale[row] = from_float<T>(s);
    const bool fast = rcp_is_safe<T>(s);  // bf16: x * rcp(s) rounds to the same bf16 as x / s (quantize_math.cuh)
    const float r = fast ? __frcp_rn(s) : 0.f;
    if (vec_ok) {
      for (int64_t v = tid; v < k / 8; v += kFzThreads) {
        float f[8];
        load8_stream<T>(src + v * 8, f);
        alignas(8) uint8_t q[8];
        if (fast) {
#pragma unroll
          for (int j = 0; j < 8; ++j) f[j] = __fmul_rn(f[j], r);
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) f[j] = __fdiv_rn(f[j], s);
        }
#pragma unroll
        for (int j = 0; j < 8; j += 2) rnd_pair<T>(f[j], f[j + 1]);
        if constexpr (sizeof(T) == 4) { /* rnd_pair is the identity for fp32 */ }
#pragma unroll
        for (int j = 0; j < 8; ++j) q[j] = quantize_one<OUT_DT>(f[j]);
        __stcs(reinterpret_cast<uint2*>(dst + v * 8), *reinterpret_cast<uint2*>(q));
      }
    } else {
      for (int64_t i = tid; i < k; i += kFzThreads) dst[i] = quantize_one<OUT_DT>(rnd<T>(__fdiv_rn(to_float<T>(src[i]), s)));
    }
  }
}

}  // namespace qb

using namespace qb;

extern "C" {

int qb200_quantize_affine(const void* base, const void* scale, const void* shift, uint8_t* out, int64_t outer,
                          int64_t inner, int axis_mode, int bits, int dtype, int shift_is_int, void* stream) {
  if (bits < 1 || bits > 8) return fail(ERR_ARG, "quantize_affine: bits must be in 1..8, got %d", bits);
  if (outer < 0 || inner < 0 || axis_mode < 0 || axis_mode > 2)
    return fail(ERR_ARG, "quantize_affine: bad shape / axis_mode (%lld x %lld, mode %d)", (long long)outer,
                (long long)inner, axis_mode);
  const int64_t numel = outer * inner;
  if (numel == 0) return OK;
  if (!base || !scale || !shift || !out) return fail(ERR_ARG, "quantize_affine: null buffer");
  if (!is_float_dtype(dtype)) return fail(ERR_ARG, "quantize_affine: dtype %d not floating point", dtype);
  const float qmax = static_cast<float>((1 << bits) - 1);
  const int zp_signed = shift_is_int == 2 ? 1 : 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool vec = inner % 8 == 0 && aligned16(base) && reinterpret_cast<uintptr_t>(out) % 8 == 0;
  return dispatch_float(dtype, [&](auto dt) {
    return dispatch_zp(shift_is_int, [&](auto ZP) {
      using T = typename decltype(dt)::T;
      const T* b = static_cast<const T*>(base);
      const T* s = static_cast<const T*>(scale);
      if (vec)
        quantize_affine_kernel<T, ZP, 8><<<capped_grid(numel / 8, kFzThreads, 16), kFzThreads, 0, st>>>(
            b, s, shift, out, numel, inner, axis_mode, qmax, ZP ? zp_signed : 0);
      else
        quantize_affine_kernel<T, ZP, 1><<<capped_grid(numel, kFzThreads, 16), kFzThreads, 0, st>>>(
            b, s, shift, out, numel, inner, axis_mode, qmax, ZP ? zp_signed : 0);
      return check_cuda(cudaGetLastError(), "quantize_affine launch");
    });
  });
}

int qb200_pack(const uint8_t* in, uint8_t* out, int64_t rows, int64_t cols, int bits, void* stream) {
  if (bits != 2 && bits != 4) return fail(ERR_ARG, "pack: bits must be 2 or 4, got %d", bits);
  if (rows < 0 || cols < 0) return fail(ERR_ARG, "pack: negative shape");
  if (rows * cols > 0 && (!in || !out)) return fail(ERR_ARG, "pack: null buffer");
  const int planes = 8 / bits;
  const int64_t packed_rows = (rows + planes - 1) / planes;
  const int64_t plane = packed_rows * cols, total = rows * cols;
  if (plane == 0) return OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool vec = plane % 16 == 0 && total % 16 == 0 && aligned16(in) && aligned16(out);
  return dispatch_bits(bits, [&](auto BITS) {
    if (vec)
      pack_vec_kernel<BITS><<<capped_grid(plane / 16, kFzThreads, 16), kFzThreads, 0, st>>>(
          reinterpret_cast<const uint4*>(in), reinterpret_cast<uint4*>(out), plane / 16, total / 16);
    else
      pack_scalar_kernel<BITS><<<capped_grid(plane, kFzThreads, 16), kFzThreads, 0, st>>>(in, out, plane, total);
    return check_cuda(cudaGetLastError(), "pack launch");
  });
}

int qb200_quantize_qbits_max(const void* base, uint8_t* packed, void* scale, void* shift, int64_t n, int64_t k,
                             int group, int bits, int dtype, int zeropoint, void* stream) {
  if (bits != 2 && bits != 4) return fail(ERR_ARG, "quantize_qbits_max: bits must be 2 or 4, got %d", bits);
  if (n <= 0 || k <= 0 || group <= 0) return fail(ERR_ARG, "quantize_qbits_max: bad shape");
  if (k % group != 0) return fail(ERR_ARG, "quantize_qbits_max: group %d does not divide K=%lld", group, (long long)k);
  if (group % 8 != 0 || group > 256)
    return fail(ERR_UNSUPPORTED, "quantize_qbits_max: group %d (needs a multiple of 8, <= 256)", group);
  if (!base || !packed || !scale || !shift) return fail(ERR_ARG, "quantize_qbits_max: null buffer");
  if (!aligned16(base) || reinterpret_cast<uintptr_t>(packed) % 8 != 0)
    return fail(ERR_UNSUPPORTED, "quantize_qbits_max: base must be 16-byte and packed 8-byte aligned");
  if (!is_float_dtype(dtype)) return fail(ERR_ARG, "quantize_qbits_max: dtype %d not floating point", dtype);
  const int64_t rows = n * k / group;
  const int planes = 8 / bits;
  const int64_t packed_rows = (rows + planes - 1) / planes;
  const int grid = capped_grid(packed_rows * team_lanes(group), kFzThreads, 8);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return dispatch_float(dtype, [&](auto dt) {
    return dispatch_bits(bits, [&](auto BITS) {
      return dispatch_zp(zeropoint, [&](auto ZP) {
        return dispatch_team_lanes(group, [&](auto TL) {
          using T = typename decltype(dt)::T;
          quantize_qbits_max_kernel<T, BITS, ZP, TL><<<grid, kFzThreads, 0, st>>>(
              static_cast<const T*>(base), packed, static_cast<T*>(scale), shift, rows, packed_rows, group);
          return check_cuda(cudaGetLastError(), "quantize_qbits_max launch");
        });
      });
    });
  });
}

int qb200_absmax(const void* base, void* out, void* scratch, int64_t numel, int dtype, void* stream) {
  if (numel < 0 || !out || !scratch || (numel > 0 && !base)) return fail(ERR_ARG, "absmax: bad buffer");
  if (reinterpret_cast<uintptr_t>(scratch) % 4 != 0) return fail(ERR_ARG, "absmax: scratch must be 4-byte aligned");
  if (!is_float_dtype(dtype)) return fail(ERR_ARG, "absmax: dtype %d not floating point", dtype);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = check_cuda(cudaMemsetAsync(scratch, 0, 8, st), "absmax: scratch memset");
  if (rc != OK) return rc;
  const int vec_ok = aligned16(base);
  const int grid = capped_grid((numel + 15) / 16, kFzThreads, 8);
  return dispatch_float(dtype, [&](auto dt) {
    using T = typename decltype(dt)::T;
    absmax_kernel<T><<<grid, kFzThreads, 0, st>>>(static_cast<const T*>(base), static_cast<T*>(out),
                                                  static_cast<int*>(scratch), numel, vec_ok);
    return check_cuda(cudaGetLastError(), "absmax launch");
  });
}

int qb200_absmax_update(const void* base, void* scale, void* scratch, int64_t numel, int dtype, double qmax,
                        double momentum, void* stream) {
  if (numel < 1) return fail(ERR_ARG, "absmax_update: the tensor is empty (numel %lld)", (long long)numel);
  if (!base || !scale || !scratch) return fail(ERR_ARG, "absmax_update: null buffer");
  if (reinterpret_cast<uintptr_t>(scratch) % 4 != 0) return fail(ERR_ARG, "absmax_update: scratch must be 4-byte aligned");
  if (!(qmax > 0.0)) return fail(ERR_ARG, "absmax_update: qmax must be positive");
  if (!is_float_dtype(dtype)) return fail(ERR_ARG, "absmax_update: dtype %d not floating point", dtype);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = check_cuda(cudaMemsetAsync(scratch, 0, 8, st), "absmax_update: scratch memset");
  if (rc != OK) return rc;
  const int vec_ok = aligned16(base);
  const int grid = capped_grid((numel + 15) / 16, kFzThreads, 8);
  // the python scalars become float operands of ATen's float opmath: momentum, and 1 - momentum evaluated in double
  const float q = static_cast<float>(qmax), m = static_cast<float>(momentum), om = static_cast<float>(1.0 - momentum);
  return dispatch_float(dtype, [&](auto dt) {
    using T = typename decltype(dt)::T;
    absmax_update_kernel<T><<<grid, kFzThreads, 0, st>>>(static_cast<const T*>(base), static_cast<T*>(scale),
                                                         static_cast<int*>(scratch), numel, vec_ok, q, m, om);
    return check_cuda(cudaGetLastError(), "absmax_update launch");
  });
}

int qb200_quantize_qbytes_absmax(const void* base, void* out, void* scale, int64_t n, int64_t k, int dtype,
                                 int out_dtype, void* stream) {
  if (n < 0 || k < 0) return fail(ERR_ARG, "quantize_qbytes_absmax: negative shape");
  if (n == 0 || k == 0) return OK;
  if (!base || !out || !scale) return fail(ERR_ARG, "quantize_qbytes_absmax: null buffer");
  if (!is_code_dtype(out_dtype)) return fail(ERR_ARG, "quantize_qbytes_absmax: unsupported target dtype %d", out_dtype);
  if (!is_float_dtype(dtype)) return fail(ERR_ARG, "quantize_qbytes_absmax: dtype %d not floating point", dtype);
  const int vec_ok = k % 8 == 0 && aligned16(base) && reinterpret_cast<uintptr_t>(out) % 8 == 0;
  const float qmax = out_dtype == DT_I8 ? 127.f : (out_dtype == DT_E4M3 ? 448.f : 57344.f);
  const int grid = capped_grid(n, 1, 8);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return dispatch_float(dtype, [&](auto dt) {
    return dispatch_code8(out_dtype, [&](auto OUT) {
      using T = typename decltype(dt)::T;
      if constexpr (decltype(OUT)::value == DT_E4M3FNUZ) {  // no kernel: int8, e4m3fn and e5m2 targets only
        return fail(ERR_ARG, "quantize_qbytes_absmax: unsupported target dtype %d", out_dtype);
      } else {
        quantize_qbytes_absmax_kernel<T, OUT><<<grid, kFzThreads, 0, st>>>(
            static_cast<const T*>(base), static_cast<uint8_t*>(out), static_cast<T*>(scale), n, k, qmax, vec_ok);
        return check_cuda(cudaGetLastError(), "quantize_qbytes_absmax launch");
      }
    });
  });
}

}  // extern "C"
