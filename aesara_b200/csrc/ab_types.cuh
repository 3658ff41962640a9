// ab_types.cuh — element types and scalar helpers shared by every JIT module.
// (Concatenated in front of the generated code; NVRTC sees one translation unit.)
//
// The typedefs have exactly the width/signedness of the NumPy C types the
// reference C-linker uses (npy_bool = unsigned char, npy_int8 = signed char, …;
// aesara/scalar/basic.py:272 ScalarType.dtype_specs), so generated expressions
// follow the same C promotion rules as the reference's generated C++.
#pragma once

typedef unsigned char ab_bool;
typedef signed char ab_i8;
typedef short ab_i16;
typedef int ab_i32;
typedef long long ab_i64;
typedef unsigned char ab_u8;
typedef unsigned short ab_u16;
typedef unsigned int ab_u32;
typedef unsigned long long ab_u64;

#define AB_MAX_DIMS 8
#define AB_INF_F __int_as_float(0x7f800000)
#define AB_NAN_F __int_as_float(0x7fc00000)
#define AB_INF_D __longlong_as_double(0x7ff0000000000000LL)
#define AB_NAN_D __longlong_as_double(0x7ff8000000000000LL)

// ---- integer floor-division / Python-sign modulo -----------------------------
// aesara/scalar/basic.py:2055-2127 (FloorDivide) and :2165-2240 (Mod): the
// reference raises ZeroDivisionError on the host for y == 0; a device kernel
// cannot raise, it follows the reference's own `#ifdef KERNEL` branch (x / y,
// x % y evaluated by the hardware) but returns 0 to stay defined.  y == -1 is answered
// without dividing: MIN / -1 overflows (undefined in C++); NumPy gives MIN // -1 = MIN (the
// negation wraps) and MIN % -1 = 0.
template <typename T>
__device__ __forceinline__ T ab_floordiv_int(T x, T y) {
  if (y == 0) return (T)0;
  if (y == (T)-1) return (T)(0ULL - (unsigned long long)x);
  T q = x / y;
  T r = x % y;
  if ((r != 0) && ((r < 0) != (y < 0))) q -= 1;
  return q;
}
template <typename T>
__device__ __forceinline__ T ab_mod_int(T x, T y) {
  if (y == 0 || y == (T)-1) return (T)0;
  T r = x % y;
  if ((r != 0) && ((r < 0) != (y < 0))) r += y;
  return r;
}
template <typename T>
__device__ __forceinline__ T ab_floordiv_uint(T x, T y) { return y == 0 ? (T)0 : x / y; }
template <typename T>
__device__ __forceinline__ T ab_mod_uint(T x, T y) { return y == 0 ? (T)0 : x % y; }

// IntDiv on floats is NOT floor(x / y) in the reference: the C code (basic.py:2083-2121)
// divides magnitudes and corrects with fmod, which differs for infinite divisors
// (0.5 // -inf = -1) and when |x| / |y| rounds up to an integer.
__device__ __forceinline__ float ab_floordiv_f(float x, float y) {
  if (y == 0.0f) return floorf(x / y);
  if (y < 0.0f) {
    if (x < 0.0f) return floorf((-x) / (-y));
    return -floorf(x / (-y)) - ((fmodf(x, -y) == 0.0f) ? 0.0f : 1.0f);
  }
  if (x < 0.0f) return -floorf((-x) / y) - ((fmodf(-x, y) == 0.0f) ? 0.0f : 1.0f);
  return floorf(x / y);
}
__device__ __forceinline__ double ab_floordiv_f(double x, double y) {
  if (y == 0.0) return floor(x / y);
  if (y < 0.0) {
    if (x < 0.0) return floor((-x) / (-y));
    return -floor(x / (-y)) - ((fmod(x, -y) == 0.0) ? 0.0 : 1.0);
  }
  if (x < 0.0) return -floor((-x) / y) - ((fmod(-x, y) == 0.0) ? 0.0 : 1.0);
  return floor(x / y);
}
// Python-sign floating modulo (basic.py:2207-2236)
// branch for branch, so that a zero remainder has the reference's sign (-6 % 3 = +0, not the
// -0 of fmod(-6, 3))
__device__ __forceinline__ float ab_mod_f(float x, float y) {
  if (y == 0.0f) return fmodf(x, y);
  if (y < 0.0f) {
    if (x < 0.0f) return -fmodf(-x, -y);
    const float m = fmodf(x, -y);
    return m + (m != 0.0f ? y : 0.0f);
  }
  if (x < 0.0f) {
    const float m = fmodf(-x, y);
    return -m + (m != 0.0f ? y : 0.0f);
  }
  return fmodf(x, y);
}
__device__ __forceinline__ double ab_mod_f(double x, double y) {
  if (y == 0.0) return fmod(x, y);
  if (y < 0.0) {
    if (x < 0.0) return -fmod(-x, -y);
    const double m = fmod(x, -y);
    return m + (m != 0.0 ? y : 0.0);
  }
  if (x < 0.0) {
    const double m = fmod(-x, y);
    return -m + (m != 0.0 ? y : 0.0);
  }
  return fmod(x, y);
}

// ---- maximum / minimum with the reference's NaN rule (basic.py:1745-1752) ------
template <typename T>
__device__ __forceinline__ T ab_max_int(T x, T y) { return y > x ? y : x; }
template <typename T>
__device__ __forceinline__ T ab_min_int(T x, T y) { return y < x ? y : x; }
__device__ __forceinline__ float ab_max_f(float x, float y) {
  return y > x ? y : (x >= y ? x : AB_NAN_F);
}
__device__ __forceinline__ double ab_max_f(double x, double y) {
  return y > x ? y : (x >= y ? x : AB_NAN_D);
}
__device__ __forceinline__ float ab_min_f(float x, float y) {
  return y < x ? y : (x <= y ? x : AB_NAN_F);
}
__device__ __forceinline__ double ab_min_f(double x, double y) {
  return y < x ? y : (x <= y ? x : AB_NAN_D);
}

// ---- sigmoid / softplus / log1mexp (aesara/scalar/math.py:1110-1258) ----------
__device__ __forceinline__ float ab_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ double ab_sigmoid(double x) { return 1.0 / (1.0 + exp(-x)); }
// The reference evaluates softplus piecewise (scalar/math.py:1172-1198):
//   x < -37: exp(x) | x < 18: log1p(exp(x)) | x < 33.3: x + exp(-x) | else x.
// All four branches are the same function max(x,0) + log1p(exp(-|x|)) to within
// one ulp of the result (log1p(e) = e(1 - e/2 + ...) and e = exp(-|x|) is below
// 1e-16 / 1.5e-8 / 3.4e-15 where the reference switches formula), so the device
// code uses that single branch-free form with one exponential instead of three
// (measured: -30% instructions on the cfg2 kernel).  NaN propagates like the
// reference (every comparison false -> returns x).
__device__ __forceinline__ float ab_softplus(float x) {
  return fmaxf(x, 0.0f) + log1pf(expf(-fabsf(x)));
}
__device__ __forceinline__ double ab_softplus(double x) {
  return fmax(x, 0.0) + log1p(exp(-fabs(x)));
}
__device__ __forceinline__ float ab_log1mexp(float x) {
  return x < -0.6931471805599453f ? log1pf(-expf(x)) : logf(-expm1f(x));
}
__device__ __forceinline__ double ab_log1mexp(double x) {
  return x < -0.6931471805599453 ? log1p(-exp(x)) : log(-expm1(x));
}
// sign (basic.py:2614-2630)
__device__ __forceinline__ float ab_sgn_f(float x) {
  return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : (isnan(x) ? AB_NAN_F : 0.0f));
}
__device__ __forceinline__ double ab_sgn_f(double x) {
  return x > 0.0 ? 1.0 : (x < 0.0 ? -1.0 : (isnan(x) ? AB_NAN_D : 0.0));
}

// ---- streaming vector loads/stores -------------------------------------------
// NB bytes (1,2,4,8,16) moved with one instruction; .cs = evict-first streaming
// (every Elemwise operand is touched exactly once).
template <int NB> struct ab_bytes;
template <> struct ab_bytes<1> { typedef unsigned char type; };
template <> struct ab_bytes<2> { typedef unsigned short type; };
template <> struct ab_bytes<4> { typedef unsigned int type; };
template <> struct ab_bytes<8> { typedef uint2 type; };
template <> struct ab_bytes<16> { typedef uint4 type; };

template <typename T, int N>
struct ab_pack {
  union {
    T v[N];
    typename ab_bytes<sizeof(T) * N>::type raw;
  };
};

template <typename T, int N>
__device__ __forceinline__ void ab_load_pack(ab_pack<T, N>& dst, const T* p) {
  typedef typename ab_bytes<sizeof(T) * N>::type R;
  dst.raw = __ldcs(reinterpret_cast<const R*>(p));
}
template <typename T, int N>
__device__ __forceinline__ void ab_store_pack(T* p, const ab_pack<T, N>& src) {
  typedef typename ab_bytes<sizeof(T) * N>::type R;
  __stcs(reinterpret_cast<R*>(p), src.raw);
}
