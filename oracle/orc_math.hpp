// ORACLE — TEST INFRASTRUCTURE ONLY. Not part of the shipped product path.
// CPU restatement of the arithmetic the reference gets from Eigen / Ceres Jets.
// PARITY UNPINNED: the reference ships no golden vectors and its Eigen/Ceres/PCL
// dependencies are absent from this container (SURVEY.md §8c); this file follows
// the published semantics of those libraries and is cross-checked in tests/ against
// scipy / finite differences instead.
//
// Follows: Eigen::Quaternion product / _transformVector / angularDistance / slerp,
//          ceres::Jet forward-mode autodiff (used by AutoDiffCostFunction at
//          loam_livox/source/ceres_icp.hpp:297-299,376-378).
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

namespace orc {

// ---------------------------------------------------------------- Jet<N>
// Forward-mode dual number, mirrors ceres::Jet<double,N>: value a + N partials v.
template <int N> struct Jet {
  double a; double v[N];
  Jet() : a(0) { for (int i = 0; i < N; i++) v[i] = 0; }
  Jet(double s) : a(s) { for (int i = 0; i < N; i++) v[i] = 0; }  // NOLINT implicit, like ceres
  Jet(double s, int k) : a(s) { for (int i = 0; i < N; i++) v[i] = 0; v[k] = 1.0; }
};
template <int N> inline Jet<N> operator+(const Jet<N>& f, const Jet<N>& g) { Jet<N> h; h.a = f.a + g.a; for (int i = 0; i < N; i++) h.v[i] = f.v[i] + g.v[i]; return h; }
template <int N> inline Jet<N> operator-(const Jet<N>& f, const Jet<N>& g) { Jet<N> h; h.a = f.a - g.a; for (int i = 0; i < N; i++) h.v[i] = f.v[i] - g.v[i]; return h; }
template <int N> inline Jet<N> operator-(const Jet<N>& f) { Jet<N> h; h.a = -f.a; for (int i = 0; i < N; i++) h.v[i] = -f.v[i]; return h; }
template <int N> inline Jet<N> operator*(const Jet<N>& f, const Jet<N>& g) { Jet<N> h; h.a = f.a * g.a; for (int i = 0; i < N; i++) h.v[i] = f.a * g.v[i] + f.v[i] * g.a; return h; }
template <int N> inline Jet<N> operator/(const Jet<N>& f, const Jet<N>& g) {
  // ceres/jet.h: h = f/g ; dh = (df - h*dg)/g
  Jet<N> h; const double gi = 1.0 / g.a; h.a = f.a * gi; for (int i = 0; i < N; i++) h.v[i] = (f.v[i] - h.a * g.v[i]) * gi; return h;
}
template <int N> inline Jet<N>& operator+=(Jet<N>& f, const Jet<N>& g) { f = f + g; return f; }
template <int N> inline Jet<N> sqrt(const Jet<N>& f) { Jet<N> h; h.a = std::sqrt(f.a); const double t = 1.0 / (2.0 * h.a); for (int i = 0; i < N; i++) h.v[i] = f.v[i] * t; return h; }
template <int N> inline Jet<N> sin(const Jet<N>& f) { Jet<N> h; h.a = std::sin(f.a); const double c = std::cos(f.a); for (int i = 0; i < N; i++) h.v[i] = c * f.v[i]; return h; }
template <int N> inline Jet<N> cos(const Jet<N>& f) { Jet<N> h; h.a = std::cos(f.a); const double s = -std::sin(f.a); for (int i = 0; i < N; i++) h.v[i] = s * f.v[i]; return h; }
template <int N> inline Jet<N> acos(const Jet<N>& f) { Jet<N> h; h.a = std::acos(f.a); const double t = -1.0 / std::sqrt(1.0 - f.a * f.a); for (int i = 0; i < N; i++) h.v[i] = t * f.v[i]; return h; }
template <int N> inline Jet<N> abs(const Jet<N>& f) { return f.a < 0.0 ? -f : f; }
template <int N> inline bool operator<(const Jet<N>& f, const Jet<N>& g) { return f.a < g.a; }
template <int N> inline bool operator>=(const Jet<N>& f, const Jet<N>& g) { return f.a >= g.a; }
inline double sqrt(double x) { return std::sqrt(x); }
inline double sin(double x) { return std::sin(x); }
inline double cos(double x) { return std::cos(x); }
inline double acos(double x) { return std::acos(x); }
inline double abs(double x) { return std::fabs(x); }
inline double scalar_of(double x) { return x; }
template <int N> inline double scalar_of(const Jet<N>& x) { return x.a; }

// ---------------------------------------------------------------- small vectors
template <typename T> struct Vec3 { T x, y, z; };
template <typename T> inline Vec3<T> operator+(const Vec3<T>& a, const Vec3<T>& b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
template <typename T> inline Vec3<T> operator-(const Vec3<T>& a, const Vec3<T>& b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
template <typename T> inline Vec3<T> operator*(const Vec3<T>& a, const T& s) { return {a.x * s, a.y * s, a.z * s}; }
template <typename T> inline Vec3<T> operator*(const T& s, const Vec3<T>& a) { return {s * a.x, s * a.y, s * a.z}; }
template <typename T> inline T dot(const Vec3<T>& a, const Vec3<T>& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <typename T> inline Vec3<T> cross(const Vec3<T>& a, const Vec3<T>& b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
template <typename T> inline T norm(const Vec3<T>& a) { return sqrt(dot(a, a)); }
typedef Vec3<double> V3d;

// ---------------------------------------------------------------- quaternion (Eigen semantics)
template <typename T> struct Quat { T w, x, y, z; };  // Eigen ctor order (w,x,y,z)
typedef Quat<double> Qd;

// Eigen::Quaternion product (Hamilton).
template <typename T> inline Quat<T> qmul(const Quat<T>& a, const Quat<T>& b) {
  return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z,
          a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
          a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
          a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
}
// Eigen QuaternionBase::_transformVector: uv = 2 * (u x v); v + w*uv + u x uv (no normalisation).
template <typename T> inline Vec3<T> qrot(const Quat<T>& q, const Vec3<T>& v) {
  Vec3<T> u{q.x, q.y, q.z};
  Vec3<T> uv = cross(u, v);
  uv = uv + uv;
  return v + uv * q.w + cross(u, uv);
}
inline Qd qconj(const Qd& q) { return {q.w, -q.x, -q.y, -q.z}; }
// Eigen (>=3.3) angularDistance: d = a * conj(b); 2*atan2(|d.vec|, |d.w|)
inline double angular_distance(const Qd& a, const Qd& b) {
  Qd d = qmul(a, qconj(b));
  return 2.0 * std::atan2(std::sqrt(d.x * d.x + d.y * d.y + d.z * d.z), std::fabs(d.w));
}
// Eigen QuaternionBase::slerp (3.3): t in [0,1], *this -> other.
template <typename T> inline Quat<T> qslerp(const Quat<T>& a, const T& t, const Quat<T>& b) {
  const double one = 1.0 - 2.220446049250313e-16;
  T d = a.w * b.w + a.x * b.x + a.y * b.y + a.z * b.z;
  T absD = abs(d);
  T scale0, scale1;
  if (scalar_of(absD) >= one) { scale0 = T(1.0) - t; scale1 = t; }
  else {
    T theta = acos(absD);
    T sinTheta = sin(theta);
    scale0 = sin((T(1.0) - t) * theta) / sinTheta;
    scale1 = sin(t * theta) / sinTheta;
  }
  if (scalar_of(d) < 0.0) scale1 = -scale1;
  return {scale0 * a.w + scale1 * b.w, scale0 * a.x + scale1 * b.x, scale0 * a.y + scale1 * b.y, scale0 * a.z + scale1 * b.z};
}

}  // namespace orc
