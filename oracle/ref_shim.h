// oracle/ref_shim.h -- TEST INFRASTRUCTURE ONLY.
//
// What CuPy places around the body of an ElementwiseKernel, restated so that the
// reference's CUDA-C kernel strings (kernels/custom_kernels.py, plugins/min_filter.py)
// compile unmodified with g++ (host) or nvcc (sm_90a).  See oracle/build_ref.py.
//
// Third-party arithmetic restated here (NOT under /root/reference): CuPy's
// `class float16` from cupy/_core/include/cupy/carray.cuh (version unpinned by the
// reference, requirements.txt:11): storage is one IEEE binary16; the only IMPLICIT
// conversions are float -> float16 (round-to-nearest-even) and float16 -> float;
// conversions from double / int / bool are explicit and go through float;
// `a op= b` is `a = a op b`; min/max of two float16 compare as float.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef REF_SHIM_GPU
// ------------------------------------------------------------------ device flavour
#include <cuda_fp16.h>
#include <cuda_runtime.h>
// CuPy hands a `raw` argument to the kernel body as a CArray whose operator[] takes a ptrdiff_t: bodies that index with
// a float (fusion/*.py: `U id = floorf(...); p[id * n]`) rely on the implicit float -> integer conversion.
template <typename T> struct CArr { T* d; __device__ T& operator[](long long i) const { return d[i]; } };
class float16 {
  __half data_;
 public:
  __device__ float16() {}
  __device__ float16(float v) : data_(__float2half(v)) {}
  explicit __device__ float16(bool v) : data_(__float2half(float(v))) {}
  explicit __device__ float16(double v) : data_(__float2half(float(v))) {}
  explicit __device__ float16(int v) : data_(__float2half(float(v))) {}
  explicit __device__ float16(unsigned int v) : data_(__float2half(float(v))) {}
  explicit __device__ float16(long long v) : data_(__float2half(float(v))) {}
  __device__ operator float() const { return __half2float(data_); }
  template <typename T> __device__ float16& operator+=(const T& rhs) { *this = *this + rhs; return *this; }
  template <typename T> __device__ float16& operator-=(const T& rhs) { *this = *this - rhs; return *this; }
  template <typename T> __device__ float16& operator*=(const T& rhs) { *this = *this * rhs; return *this; }
  template <typename T> __device__ float16& operator/=(const T& rhs) { *this = *this / rhs; return *this; }
};
__device__ inline float16 min(float16 x, float16 y) { return float16(fminf(float(x), float(y))); }
__device__ inline float16 max(float16 x, float16 y) { return float16(fmaxf(float(x), float(y))); }

#else
// ------------------------------------------------------------------ host flavour
#include <cmath>
#define __device__
template <typename T> struct CArr { T* d; T& operator[](long long i) const { return d[i]; } };
namespace refshim {
class float16 {
  _Float16 data_;
 public:
  float16() {}
  float16(float v) : data_((_Float16)v) {}
  explicit float16(bool v) : data_((_Float16)(float)v) {}
  explicit float16(double v) : data_((_Float16)(float)v) {}
  explicit float16(int v) : data_((_Float16)(float)v) {}
  explicit float16(unsigned int v) : data_((_Float16)(float)v) {}
  explicit float16(long long v) : data_((_Float16)(float)v) {}
  operator float() const { return (float)data_; }
  template <typename T> float16& operator+=(const T& rhs) { *this = *this + rhs; return *this; }
  template <typename T> float16& operator-=(const T& rhs) { *this = *this - rhs; return *this; }
  template <typename T> float16& operator*=(const T& rhs) { *this = *this * rhs; return *this; }
  template <typename T> float16& operator/=(const T& rhs) { *this = *this / rhs; return *this; }
};
// CUDA's overload set for the functions the kernel bodies call (math_functions.hpp):
inline float16 min(float16 x, float16 y) { return float16(fminf(float(x), float(y))); }
inline float16 max(float16 x, float16 y) { return float16(fmaxf(float(x), float(y))); }
inline float min(float a, float b) { return fminf(a, b); }
inline float max(float a, float b) { return fmaxf(a, b); }
inline double min(double a, double b) { return fmin(a, b); }
inline double max(double a, double b) { return fmax(a, b); }
inline double min(float a, double b) { return fmin((double)a, b); }
inline double max(float a, double b) { return fmax((double)a, b); }
inline double min(double a, float b) { return fmin(a, (double)b); }
inline double max(double a, float b) { return fmax(a, (double)b); }
inline int min(int a, int b) { return a < b ? a : b; }
inline int max(int a, int b) { return a > b ? a : b; }
inline float sqrt(float a) { return sqrtf(a); }
inline double sqrt(double a) { return ::sqrt(a); }
inline float abs(float a) { return fabsf(a); }
inline double abs(double a) { return ::fabs(a); }
inline int abs(int a) { return a < 0 ? -a : a; }
inline float fabs(float a) { return fabsf(a); }
inline double fabs(double a) { return ::fabs(a); }
// atomicAdd(float*, float): relaxed CAS loop, usable from OpenMP threads.
inline float atomicAdd(float* addr, float val) {
  uint32_t* a = reinterpret_cast<uint32_t*>(addr);
  uint32_t old = __atomic_load_n(a, __ATOMIC_RELAXED), nw;
  float f;
  do {
    __builtin_memcpy(&f, &old, 4);
    float g = f + val;
    __builtin_memcpy(&nw, &g, 4);
  } while (!__atomic_compare_exchange_n(a, &old, nw, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED));
  __builtin_memcpy(&f, &old, 4);
  return f;
}
// integer atomicAdd and the bit casts the colour fusion kernels use (fusion/pointcloud_color.py)
inline unsigned int atomicAdd(unsigned int* addr, unsigned int val) { return __atomic_fetch_add(addr, val, __ATOMIC_RELAXED); }
inline unsigned int atomicAdd(unsigned int* addr, int val) { return __atomic_fetch_add(addr, (unsigned int)val, __ATOMIC_RELAXED); }
inline unsigned int __float_as_uint(float f) { unsigned int u; __builtin_memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(unsigned int u) { float f; __builtin_memcpy(&f, &u, 4); return f; }
}  // namespace refshim
#endif
