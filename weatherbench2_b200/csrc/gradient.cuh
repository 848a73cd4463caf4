// np.gradient(f, x, edge_order=1) on the device, shared by wind_dynamics.cu and
// thermo.cu.  Not part of the C ABI.
//
// The host passes np.gradient's coefficients per index as a [n][3] float64
// table (_derived_wind.gradient_table): index 0 and n-1 hold the edge spacing,
// a uniform interior holds 2*dx, a non-uniform interior holds a, b, c for
// f[i-1], f[i], f[i+1].  With T the data type, every derivative is NumPy's
// float64 expression rounded once to T:
//   edges             T(f[1] - f[0]) / dx[0] and T(f[n-1] - f[n-2]) / dx[n-2]
//   uniform interior  T(f[i+1] - f[i-1]) / (2 dx)
//   otherwise         (a f[i-1] + b f[i]) + c f[i+1], left to right
// The differences are subtractions in T, everything else float64, all with
// correctly rounded intrinsics, so nothing is contracted into an FMA.
#pragma once

#include <cstdint>

namespace wb2 {
namespace grad {

__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }

template <typename T>
__device__ __forceinline__ T round_to(double x);
template <>
__device__ __forceinline__ float round_to<float>(double x) { return __double2float_rn(x); }
template <>
__device__ __forceinline__ double round_to<double>(double x) { return x; }

// (hi - lo) / d: an edge, or a uniform interior with d = 2*dx
template <typename T>
__device__ __forceinline__ T difference(T hi, T lo, double d) {
  return round_to<T>(__ddiv_rn(double(sub_rn(hi, lo)), d));
}

// (c[0] fm + c[1] f0) + c[2] fp: a non-uniform interior
template <typename T>
__device__ __forceinline__ T three_point(T fm, T f0, T fp, const double* __restrict__ c) {
  return round_to<T>(__dadd_rn(__dadd_rn(__dmul_rn(__ldg(c), double(fm)),
                                         __dmul_rn(__ldg(c + 1), double(f0))),
                               __dmul_rn(__ldg(c + 2), double(fp))));
}

// The derivative at index i of an axis of n points whose values are fm, f0, fp
// at i-1, i, i+1 (fm is not read at i = 0, fp not at i = n-1).
template <typename T>
__device__ __forceinline__ T at_index(T fm, T f0, T fp, int i, int n,
                                      const double* __restrict__ coef, bool uniform) {
  const double* c = coef + 3 * i;
  if (i == 0) return difference(fp, f0, __ldg(c));
  if (i == n - 1) return difference(f0, fm, __ldg(c));
  if (uniform) return difference(fp, fm, __ldg(c));
  return three_point(fm, f0, fp, c);
}

}  // namespace grad

// np.gradient at index i of an axis of n points, element stride s, read from
// memory: only the points the stencil uses are loaded.
template <typename T>
__device__ __forceinline__ T gradient(const T* __restrict__ p, int i, int n, int64_t s,
                                      const double* __restrict__ coef, bool uniform) {
  const double* c = coef + 3 * i;
  if (i == 0) return grad::difference(__ldg(p + s), __ldg(p), __ldg(c));
  if (i == n - 1) return grad::difference(__ldg(p), __ldg(p - s), __ldg(c));
  const T fm = __ldg(p - s), fp = __ldg(p + s);
  if (uniform) return grad::difference(fp, fm, __ldg(c));
  return grad::three_point(fm, __ldg(p), fp, c);
}

}  // namespace wb2
