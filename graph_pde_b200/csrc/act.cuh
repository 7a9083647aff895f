// Hidden activation of the edge MLP (include/nnconv_b200.h NNCONV_ACT_*), as a compile-time template argument of the
// kernels that fuse it.  act_fwd is f(z); act_grad is f'(z) written as a function of the output y = f(z), which is all
// the backward keeps or recomputes (the stored activation, never the pre-activation).  At y = 0 it follows torch's
// backward: LeakyReLU gives the slope, ELU gives alpha, ReLU gives 0.  q is the kind's parameter block (plan.h
// ActParams).
//
// Every function is fp32-accurate to a few ulp (tanhf, expf, expm1f, log1pf; the reciprocals of the sigmoid and of
// softsign's 1 + |z| are refined by one Newton step), so f16x2 and fp32 keep their tolerances; at f16 / bf16 the
// 16-bit store of y dominates the error.  Nothing calls a slow-path subroutine: an IEEE division's call would make
// ptxas serialise the wgmma of the GEMMs whose epilogues apply the activation.
//
// CLAMP has kinks at its bounds, and f' is decided from the STORED y: an entry is saturated exactly when its stored
// image equals the stored image of a bound (q.v[1], q.v[2]: the 16-bit value at f16 / bf16, hi + lo of the (hi, lo)
// split at f16x2, the bound itself at fp32).  Every 16-bit writer therefore stores an interior y whose image would
// land on a bound's image one 16-bit step inward (act_store16, act_split_lo); a saturated y (== lo or hi in fp32) is
// stored as the bound's own image by the rounding itself.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <type_traits>
#include "../../include/nnconv_b200.h"
#include "plan.h"

namespace nnc {

enum { ACT_RELU = NNCONV_ACT_RELU, ACT_LEAKY_RELU = NNCONV_ACT_LEAKY_RELU, ACT_ELU = NNCONV_ACT_ELU,
       ACT_TANH = NNCONV_ACT_TANH, ACT_SIGMOID = NNCONV_ACT_SIGMOID, ACT_CLAMP = NNCONV_ACT_CLAMP,
       ACT_SCALED_ELU = NNCONV_ACT_SCALED_ELU, ACT_SOFTSIGN = NNCONV_ACT_SOFTSIGN, ACT_LOGSIGMOID = NNCONV_ACT_LOGSIGMOID };

template <int ACT>
__device__ __forceinline__ float act_fwd(float z, const ActParams& q) {
  if (ACT == ACT_RELU) return fmaxf(z, 0.f);
  if (ACT == ACT_LEAKY_RELU) return z > 0.f ? z : q.v[0] * z;
  if (ACT == ACT_ELU) return z > 0.f ? z : q.v[0] * expm1f(z);
  if (ACT == ACT_TANH) return tanhf(z);
  // clamp(a z + b, lo, hi)
  if (ACT == ACT_CLAMP) return fminf(fmaxf(fmaf(q.v[0], z, q.v[3]), q.v[4]), q.v[5]);
  // lambda (z > 0 ? z : alpha expm1(c z)), with lambda * alpha folded on the host
  if (ACT == ACT_SCALED_ELU) return z > 0.f ? q.v[0] * z : q.v[2] * expm1f(q.v[1] * z);
  if (ACT == ACT_SOFTSIGN) {
    // z / (1 + |z|); beyond 2^24 the reciprocal would leave the range of __fdividef, and y is +-1 to the ulp
    const float d = 1.f + fabsf(z);
    float r = __fdividef(1.f, d);
    r = fmaf(r, fmaf(-d, r, 1.f), r);
    return !(fabsf(z) >= 0x1p24f) ? z * r : copysignf(1.f, z);
  }
  if (ACT == ACT_LOGSIGMOID) return fminf(z, 0.f) - log1pf(expf(-fabsf(z)));
  // ACT_SIGMOID: e / (1 + e) for z < 0 keeps the relative accuracy of the small values
  const float e = expf(-fabsf(z)), d = 1.f + e;
  float r = __fdividef(1.f, d);
  r = fmaf(r, fmaf(-d, r, 1.f), r);
  return z >= 0.f ? r : e * r;
}

template <int ACT>
__device__ __forceinline__ float act_grad(float y, const ActParams& q) {
  if (ACT == ACT_RELU) return y > 0.f ? 1.f : 0.f;
  if (ACT == ACT_LEAKY_RELU) return y > 0.f ? 1.f : q.v[0];
  if (ACT == ACT_ELU) return y > 0.f ? 1.f : y + q.v[0];
  if (ACT == ACT_TANH) return 1.f - y * y;
  if (ACT == ACT_CLAMP) return y > q.v[1] && y < q.v[2] ? q.v[0] : 0.f;   // strictly between the bounds' images
  if (ACT == ACT_SCALED_ELU) return y > 0.f ? q.v[0] : q.v[1] * (y + q.v[2]);
  if (ACT == ACT_SOFTSIGN) {       // 1 / (1 + |z|)^2 = (1 - |y|)^2
    const float t = 1.f - fabsf(y);
    return t * t;
  }
  if (ACT == ACT_LOGSIGMOID) return -expm1f(y);   // sigmoid(-z) = 1 - e^y
  return y * (1.f - y);            // ACT_SIGMOID
}

// the neighbouring value of a 16-bit float (sign and magnitude bits: fp16 or bf16) toward +inf (up) or -inf
__device__ __forceinline__ uint16_t bits16_step(uint16_t b, bool up) {
  if ((b & 0x7FFFu) == 0u) return up ? 0x0001u : 0x8001u;
  return ((b & 0x8000u) != 0u) != up ? b + 1 : b - 1;
}

// The value a 16-bit writer (FMT 0: fp16, 1: bf16) converts to store the activation y.  ACT_CLAMP: an interior y whose
// 16-bit image equals a bound's image becomes the 16-bit value one step inward (exact, so the store keeps it); every
// other y is returned as it is.
template <int ACT, int FMT>
__device__ __forceinline__ float act_store16(float y, const ActParams& q) {
  if (ACT != ACT_CLAMP || !(y > q.v[4] && y < q.v[5])) return y;
  uint16_t b = FMT == 0 ? __half_as_ushort(__float2half_rn(y)) : __bfloat16_as_ushort(__float2bfloat16_rn(y));
  auto widen = [](uint16_t u) {
    return FMT == 0 ? __half2float(__ushort_as_half(u)) : __bfloat162float(__ushort_as_bfloat16(u));
  };
  const float s = widen(b);
  if (s == q.v[2]) b = bits16_step(b, false);
  else if (s == q.v[1]) b = bits16_step(b, true);
  else return y;
  return widen(b);
}

// ACT_CLAMP at f16x2: y is stored as hi = fp16(y), lo = fp16(y - hi) and read as hi + lo.  Returns the lo half to
// store: for an interior y whose pair widens onto a bound's image, lo moved one fp16 step inward.
template <int ACT>
__device__ __forceinline__ __half act_split_lo(float y, __half hi, __half lo, const ActParams& q) {
  if (ACT != ACT_CLAMP || !(y > q.v[4] && y < q.v[5])) return lo;
  const float w = __half2float(hi) + __half2float(lo);
  if (w == q.v[2]) return __ushort_as_half(bits16_step(__half_as_ushort(lo), false));
  if (w == q.v[1]) return __ushort_as_half(bits16_step(__half_as_ushort(lo), true));
  return lo;
}

// The fp16 range check of an activation writer: the magnitude that is compared against 65504.  Counting the stored
// y alone would miss a non-finite pre-activation that the activation maps into the range (tanh(inf) = 1,
// sigmoid(-inf) = 0, clamp(inf) = hi, ReLU(NaN) = 0 through fmaxf), so a z that is not finite counts as out of range
// whatever f makes of it.  ReLU keeps its check on y (a NaN z there is dropped by the max, as it always was).
template <int ACT>
__device__ __forceinline__ float act_range(float z, float y) {
  if (ACT == ACT_RELU) return fabsf(y);
  return fabsf(z) < INFINITY ? fabsf(y) : INFINITY;
}

// two stored 16-bit activations (FMT 0: fp16, 1: bf16) as floats
template <int FMT>
__device__ __forceinline__ float2 unpack2(uint32_t w) {
  if (FMT == 0) return __half22float2(*reinterpret_cast<const __half2*>(&w));
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w));
}

// Runtime kind -> compile-time ACT for host dispatch: f(std::integral_constant<int, ACT>()) for the nine kinds.
template <typename F>
inline auto act_dispatch(int kind, F&& f) {
  switch (kind) {
    case ACT_LEAKY_RELU: return f(std::integral_constant<int, ACT_LEAKY_RELU>());
    case ACT_ELU: return f(std::integral_constant<int, ACT_ELU>());
    case ACT_TANH: return f(std::integral_constant<int, ACT_TANH>());
    case ACT_SIGMOID: return f(std::integral_constant<int, ACT_SIGMOID>());
    case ACT_CLAMP: return f(std::integral_constant<int, ACT_CLAMP>());
    case ACT_SCALED_ELU: return f(std::integral_constant<int, ACT_SCALED_ELU>());
    case ACT_SOFTSIGN: return f(std::integral_constant<int, ACT_SOFTSIGN>());
    case ACT_LOGSIGMOID: return f(std::integral_constant<int, ACT_LOGSIGMOID>());
    default: return f(std::integral_constant<int, ACT_RELU>());
  }
}

}  // namespace nnc
