// Hidden activation of the edge MLP (include/nnconv_b200.h NNCONV_ACT_*), as a compile-time template argument of the
// kernels that fuse it.  act_fwd is f(z); act_grad is f'(z) written as a function of the output y = f(z), which is all
// the backward keeps or recomputes (the stored activation, never the pre-activation).  At y = 0 it follows torch's
// backward: LeakyReLU gives the slope, ELU gives alpha, ReLU gives 0.
//
// Every function is fp32-accurate to a few ulp (tanhf, expf, expm1f; the sigmoid's reciprocal of 1 + e^-|z| in (1, 2]
// is refined by one Newton step), so f16x2 and fp32 keep their tolerances; at f16 / bf16 the 16-bit store of y
// dominates the error.  Nothing calls a slow-path subroutine: an IEEE division's call would make ptxas serialise the
// wgmma of the GEMMs whose epilogues apply the activation.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <type_traits>
#include "../../include/nnconv_b200.h"

namespace nnc {

enum { ACT_RELU = NNCONV_ACT_RELU, ACT_LEAKY_RELU = NNCONV_ACT_LEAKY_RELU, ACT_ELU = NNCONV_ACT_ELU,
       ACT_TANH = NNCONV_ACT_TANH, ACT_SIGMOID = NNCONV_ACT_SIGMOID };

template <int ACT>
__device__ __forceinline__ float act_fwd(float z, float p) {
  if (ACT == ACT_RELU) return fmaxf(z, 0.f);
  if (ACT == ACT_LEAKY_RELU) return z > 0.f ? z : p * z;
  if (ACT == ACT_ELU) return z > 0.f ? z : p * expm1f(z);
  if (ACT == ACT_TANH) return tanhf(z);
  // ACT_SIGMOID: e / (1 + e) for z < 0 keeps the relative accuracy of the small values
  const float e = expf(-fabsf(z)), d = 1.f + e;
  float r = __fdividef(1.f, d);
  r = fmaf(r, fmaf(-d, r, 1.f), r);
  return z >= 0.f ? r : e * r;
}

template <int ACT>
__device__ __forceinline__ float act_grad(float y, float p) {
  if (ACT == ACT_RELU) return y > 0.f ? 1.f : 0.f;
  if (ACT == ACT_LEAKY_RELU) return y > 0.f ? 1.f : p;
  if (ACT == ACT_ELU) return y > 0.f ? 1.f : y + p;
  if (ACT == ACT_TANH) return 1.f - y * y;
  return y * (1.f - y);            // ACT_SIGMOID
}

// The fp16 range check of an activation writer: the magnitude that is compared against 65504.  Counting the stored
// y alone would miss a non-finite pre-activation that the activation maps into the range (tanh(inf) = 1,
// sigmoid(-inf) = 0, ReLU(NaN) = 0 through fmaxf), so a z that is not finite counts as out of range whatever f makes
// of it.  ReLU keeps its check on y (a NaN z there is dropped by the max, as it always was).
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

// Runtime kind -> compile-time ACT for host dispatch: f(std::integral_constant<int, ACT>()) for the five kinds.
template <typename F>
inline auto act_dispatch(int kind, F&& f) {
  switch (kind) {
    case ACT_LEAKY_RELU: return f(std::integral_constant<int, ACT_LEAKY_RELU>());
    case ACT_ELU: return f(std::integral_constant<int, ACT_ELU>());
    case ACT_TANH: return f(std::integral_constant<int, ACT_TANH>());
    case ACT_SIGMOID: return f(std::integral_constant<int, ACT_SIGMOID>());
    default: return f(std::integral_constant<int, ACT_RELU>());
  }
}

}  // namespace nnc
