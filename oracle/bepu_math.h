// ORACLE — test infrastructure only. A CPU restatement of bepuphysics2's wide math, written from scratch.
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may use anything
// under oracle/. The product (libbepucuda) never includes, links or calls this.
//
// PARITY: the reference ships no golden numeric vectors for the solver path (SURVEY.md §8c) and cannot be built here
// (no .NET). This restatement follows the reference source operation-for-operation; each function cites the file:line it
// restates. The constraint functions (all 44 types), the wide math underneath and PoseIntegration are PINNED to the C# text:
// oracle/ref_transpile/cs2cpp.py transpiles those reference sources mechanically (syntax only) into oracle/_ref/libbepu_ref.so
// and tests/test_oracle_pinned_to_reference.py holds this restatement to it bit for bit, live and through the committed
// known-answer vectors tests/golden/reference_vectors.npz. UNPINNED (by construction + closed-form tests only): the solver
// driver in bepu_oracle.cpp (substep loop, batch order, integration responsibilities, gather/scatter, bundle loops).
//
// Everything is templated on a lane type F: `float` (scalar-per-lane checker), `f8` (8 x fp32 GCC vector, the
// AVX2 shape of System.Numerics.Vector<float> on the reference's usual hosts; used for the timed CPU baseline) or
// `double` (the same operations evaluated in float64: the precision yardstick of tests/precision/isolated_solve.cpp).
// Compile with -ffp-contract=off: RyuJIT never contracts a*b+c in Vector<T> code.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#if defined(__AVX2__)
#include <immintrin.h>
#endif

namespace bepu_oracle {

typedef float f8 __attribute__((vector_size(32)));
typedef int32_t i8 __attribute__((vector_size(32)));

// ---- lane traits -------------------------------------------------------------------------------------------------
template <class F> struct LaneTraits;
// Scalar: the element type of the rows a lane reads and writes (Rows<F>).
template <> struct LaneTraits<float> {
    typedef bool Mask;
    typedef float Scalar;
    static constexpr int Width = 1;
};
template <> struct LaneTraits<f8> {
    typedef i8 Mask;
    typedef float Scalar;
    static constexpr int Width = 8;
};
template <> struct LaneTraits<double> {
    typedef bool Mask;
    typedef double Scalar;
    static constexpr int Width = 1;
};
template <class F> using MaskOf = typename LaneTraits<F>::Mask;

template <class F> inline F bc(float v);
template <> inline float bc<float>(float v) { return v; }
template <> inline f8 bc<f8>(float v) { return f8{v, v, v, v, v, v, v, v}; }
template <> inline double bc<double>(float v) { return v; }

inline float get_lane(float v, int) { return v; }
inline float get_lane(const f8& v, int i) { return v[i]; }
inline void set_lane(float& v, int, float x) { v = x; }
inline void set_lane(f8& v, int i, float x) { v[i] = x; }
inline double get_lane(double v, int) { return v; }
inline void set_lane(double& v, int, double x) { v = x; }

// Vector.SquareRoot / Math.Sqrt: IEEE correctly rounded.
inline float vsqrt(float a) { return sqrtf(a); }
inline float vfloor(float a) { return floorf(a); }
inline float vabs(float a) { return fabsf(a); }
// Vector.Min/Max lower to minps/maxps on x86: (a < b) ? a : b and (a > b) ? a : b.
inline float vmin(float a, float b) { return a < b ? a : b; }
inline float vmax(float a, float b) { return a > b ? a : b; }
inline bool lt(float a, float b) { return a < b; }
inline bool gt(float a, float b) { return a > b; }
inline bool eq(float a, float b) { return a == b; }
inline float sel(bool m, float a, float b) { return m ? a : b; }
inline bool mand(bool a, bool b) { return a && b; }
inline bool mor(bool a, bool b) { return a || b; }
inline bool mnot(bool a) { return !a; }
inline bool any(bool a) { return a; }
// The float64 lane: the same operations in double. These must precede every template that calls them: a double argument
// brings no namespace for argument-dependent lookup, so a template defined earlier would bind the float overloads and round.
inline double vsqrt(double a) { return std::sqrt(a); }
inline double vfloor(double a) { return std::floor(a); }
inline double vabs(double a) { return std::fabs(a); }
inline double vmin(double a, double b) { return a < b ? a : b; }
inline double vmax(double a, double b) { return a > b ? a : b; }
inline bool lt(double a, double b) { return a < b; }
inline bool gt(double a, double b) { return a > b; }
inline bool eq(double a, double b) { return a == b; }
inline double sel(bool m, double a, double b) { return m ? a : b; }

#if defined(__AVX2__)
inline f8 vsqrt(f8 a) { return (f8)_mm256_sqrt_ps((__m256)a); }
inline f8 vfloor(f8 a) { return (f8)_mm256_floor_ps((__m256)a); }
inline f8 vabs(f8 a) { return (f8)_mm256_andnot_ps(_mm256_set1_ps(-0.0f), (__m256)a); }
inline f8 vmin(f8 a, f8 b) { return (f8)_mm256_min_ps((__m256)a, (__m256)b); }
inline f8 vmax(f8 a, f8 b) { return (f8)_mm256_max_ps((__m256)a, (__m256)b); }
#else
inline f8 vsqrt(f8 a) { f8 r; for (int i = 0; i < 8; ++i) r[i] = sqrtf(a[i]); return r; }
inline f8 vfloor(f8 a) { f8 r; for (int i = 0; i < 8; ++i) r[i] = floorf(a[i]); return r; }
inline f8 vabs(f8 a) { f8 r; for (int i = 0; i < 8; ++i) r[i] = fabsf(a[i]); return r; }
inline f8 vmin(f8 a, f8 b) { f8 r; for (int i = 0; i < 8; ++i) r[i] = a[i] < b[i] ? a[i] : b[i]; return r; }
inline f8 vmax(f8 a, f8 b) { f8 r; for (int i = 0; i < 8; ++i) r[i] = a[i] > b[i] ? a[i] : b[i]; return r; }
#endif
inline i8 lt(f8 a, f8 b) { return a < b; }
inline i8 gt(f8 a, f8 b) { return a > b; }
inline i8 eq(f8 a, f8 b) { return a == b; }
inline f8 sel(i8 m, f8 a, f8 b) { return m ? a : b; }
inline i8 mand(i8 a, i8 b) { return a & b; }
inline i8 mor(i8 a, i8 b) { return a | b; }
inline i8 mnot(i8 a) { return ~a; }
inline bool any(i8 a) {
    for (int i = 0; i < 8; ++i) if (a[i]) return true;
    return false;
}

// ---- small aggregates --------------------------------------------------------------------------------------------
template <class F> struct V2 { F x, y; };
template <class F> struct V3 { F x, y, z; };
template <class F> struct Q4 { F x, y, z, w; };
template <class F> struct Sym2 { F xx, yx, yy; };
template <class F> struct Sym3 { F xx, yx, yy, zx, zy, zz; };
template <class F> struct M23 { V3<F> x, y; };
template <class F> struct M33 { V3<F> x, y, z; };
template <class F> struct Velocity { V3<F> lin, ang; };
template <class F> struct Inertia { Sym3<F> t; F inv_mass; };

template <class F> inline V3<F> v3bc(float x, float y, float z) { return V3<F>{bc<F>(x), bc<F>(y), bc<F>(z)}; }

// BepuUtilities/Vector3Wide.cs:L55-66, L127-138, L343-350
template <class F> inline V3<F> add(const V3<F>& a, const V3<F>& b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
template <class F> inline V3<F> sub(const V3<F>& a, const V3<F>& b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
template <class F> inline V3<F> scale(const V3<F>& a, const F& s) { return {a.x * s, a.y * s, a.z * s}; }
template <class F> inline V3<F> neg(const V3<F>& a) { return {-a.x, -a.y, -a.z}; }
// Vector3Wide.cs:L201-204
template <class F> inline F dot(const V3<F>& a, const V3<F>& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
// Vector3Wide.cs:L519-525
template <class F> inline V3<F> cross(const V3<F>& a, const V3<F>& b) {
    return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
// Vector3Wide.cs:L562-576
template <class F> inline F length_squared(const V3<F>& v) { return v.x * v.x + v.y * v.y + v.z * v.z; }
template <class F> inline F length(const V3<F>& v) { return vsqrt(v.x * v.x + v.y * v.y + v.z * v.z); }
// Vector3Wide.cs:L627-633
template <class F> inline F distance(const V3<F>& a, const V3<F>& b) {
    F x = b.x - a.x, y = b.y - a.y, z = b.z - a.z;
    return vsqrt(x * x + y * y + z * z);
}
// Vector3Wide.cs:L688-693
template <class F> inline V3<F> normalize(const V3<F>& v) {
    F s = bc<F>(1.0f) / length(v);
    return scale(v, s);
}
// Vector3Wide.cs:L716-721
template <class F> inline V3<F> sel3(const MaskOf<F>& m, const V3<F>& a, const V3<F>& b) {
    return {sel(m, a.x, b.x), sel(m, a.y, b.y), sel(m, a.z, b.z)};
}
template <class F> inline Q4<F> sel4(const MaskOf<F>& m, const Q4<F>& a, const Q4<F>& b) {
    return {sel(m, a.x, b.x), sel(m, a.y, b.y), sel(m, a.z, b.z), sel(m, a.w, b.w)};
}
template <class F> inline V2<F> add(const V2<F>& a, const V2<F>& b) { return {a.x + b.x, a.y + b.y}; }
template <class F> inline V2<F> sub(const V2<F>& a, const V2<F>& b) { return {a.x - b.x, a.y - b.y}; }
template <class F> inline V2<F> scale(const V2<F>& a, const F& s) { return {a.x * s, a.y * s}; }
// BepuUtilities/Vector2Wide.cs Length
template <class F> inline F length(const V2<F>& v) { return vsqrt(v.x * v.x + v.y * v.y); }

// ---- Symmetric3x3Wide (BepuUtilities/Symmetric3x3Wide.cs) --------------------------------------------------------
// L42-66 Invert
template <class F> inline Sym3<F> invert(const Sym3<F>& m) {
    F xx = m.yy * m.zz - m.zy * m.zy;
    F yx = m.zy * m.zx - m.zz * m.yx;
    F zx = m.yx * m.zy - m.zx * m.yy;
    F det_inv = bc<F>(1.0f) / (xx * m.xx + yx * m.yx + zx * m.zx);
    F yy = m.zz * m.xx - m.zx * m.zx;
    F zy = m.zx * m.yx - m.xx * m.zy;
    F zz = m.xx * m.yy - m.yx * m.yx;
    Sym3<F> r;
    r.xx = xx * det_inv; r.yx = yx * det_inv; r.zx = zx * det_inv;
    r.yy = yy * det_inv; r.zy = zy * det_inv; r.zz = zz * det_inv;
    return r;
}
template <class F> inline Sym3<F> add(const Sym3<F>& a, const Sym3<F>& b) {
    return {a.xx + b.xx, a.yx + b.yx, a.yy + b.yy, a.zx + b.zx, a.zy + b.zy, a.zz + b.zz};
}
template <class F> inline Sym3<F> scale(const Sym3<F>& m, const F& s) {
    return {m.xx * s, m.yx * s, m.yy * s, m.zx * s, m.zy * s, m.zz * s};
}
// L182-208 SkewSandwichWithoutOverlap: skew(v) * m * transpose(skew(v))
template <class F> inline Sym3<F> skew_sandwich(const V3<F>& v, const Sym3<F>& m) {
    F xzy = v.x * m.zy, yzx = v.y * m.zx, zyx = v.z * m.yx;
    F ixy = v.y * m.zy - v.z * m.yy;
    F ixz = v.y * m.zz - v.z * m.zy;
    F iyx = v.z * m.xx - v.x * m.zx;
    F iyy = zyx - xzy;
    F iyz = v.z * m.zx - v.x * m.zz;
    F izx = v.x * m.yx - v.y * m.xx;
    F izy = v.x * m.yy - v.y * m.yx;
    F izz = xzy - yzx;
    Sym3<F> s;
    s.xx = v.y * ixz - v.z * ixy;
    s.yx = v.y * iyz - v.z * iyy;
    s.yy = v.z * iyx - v.x * iyz;
    s.zx = v.y * izz - v.z * izy;
    s.zy = v.z * izx - v.x * izz;
    s.zz = v.x * izy - v.y * izx;
    return s;
}
// L214-222 VectorSandwich: v * m * vT
template <class F> inline F vector_sandwich(const V3<F>& v, const Sym3<F>& m) {
    F x = v.x * m.xx + v.y * m.yx + v.z * m.zx;
    F y = v.x * m.yx + v.y * m.yy + v.z * m.zy;
    F z = v.x * m.zx + v.y * m.zy + v.z * m.zz;
    return x * v.x + y * v.y + z * v.z;
}
// L231-258 RotationSandwich: rT * m * r
template <class F> inline Sym3<F> rotation_sandwich(const M33<F>& r, const Sym3<F>& m) {
    F ixx = r.x.x * m.xx + r.y.x * m.yx + r.z.x * m.zx;
    F ixy = r.x.x * m.yx + r.y.x * m.yy + r.z.x * m.zy;
    F ixz = r.x.x * m.zx + r.y.x * m.zy + r.z.x * m.zz;
    F iyx = r.x.y * m.xx + r.y.y * m.yx + r.z.y * m.zx;
    F iyy = r.x.y * m.yx + r.y.y * m.yy + r.z.y * m.zy;
    F iyz = r.x.y * m.zx + r.y.y * m.zy + r.z.y * m.zz;
    F izx = r.x.z * m.xx + r.y.z * m.yx + r.z.z * m.zx;
    F izy = r.x.z * m.yx + r.y.z * m.yy + r.z.z * m.zy;
    F izz = r.x.z * m.zx + r.y.z * m.zy + r.z.z * m.zz;
    Sym3<F> s;
    s.xx = ixx * r.x.x + ixy * r.y.x + ixz * r.z.x;
    s.yx = iyx * r.x.x + iyy * r.y.x + iyz * r.z.x;
    s.yy = iyx * r.x.y + iyy * r.y.y + iyz * r.z.y;
    s.zx = izx * r.x.x + izy * r.y.x + izz * r.z.x;
    s.zy = izx * r.x.y + izy * r.y.y + izz * r.z.y;
    s.zz = izx * r.x.z + izy * r.y.z + izz * r.z.z;
    return s;
}
// MatrixSandwich(Matrix2x3Wide, Symmetric3x3Wide) -> Symmetric2x2Wide
template <class F> inline Sym2<F> matrix_sandwich(const M23<F>& m, const Sym3<F>& t) {
    F ixx = m.x.x * t.xx + m.x.y * t.yx + m.x.z * t.zx;
    F ixy = m.x.x * t.yx + m.x.y * t.yy + m.x.z * t.zy;
    F ixz = m.x.x * t.zx + m.x.y * t.zy + m.x.z * t.zz;
    F iyx = m.y.x * t.xx + m.y.y * t.yx + m.y.z * t.zx;
    F iyy = m.y.x * t.yx + m.y.y * t.yy + m.y.z * t.zy;
    F iyz = m.y.x * t.zx + m.y.y * t.zy + m.y.z * t.zz;
    Sym2<F> r;
    r.xx = ixx * m.x.x + ixy * m.x.y + ixz * m.x.z;
    r.yx = iyx * m.x.x + iyy * m.x.y + iyz * m.x.z;
    r.yy = iyx * m.y.x + iyy * m.y.y + iyz * m.y.z;
    return r;
}
// TransformWithoutOverlap(Vector3Wide, Symmetric3x3Wide): v * m
template <class F> inline V3<F> transform(const V3<F>& v, const Sym3<F>& m) {
    return {v.x * m.xx + v.y * m.yx + v.z * m.zx, v.x * m.yx + v.y * m.yy + v.z * m.zy, v.x * m.zx + v.y * m.zy + v.z * m.zz};
}
// MultiplyWithoutOverlap(Matrix2x3Wide a, Symmetric3x3Wide b)
template <class F> inline M23<F> multiply(const M23<F>& a, const Sym3<F>& b) {
    M23<F> r;
    r.x.x = a.x.x * b.xx + a.x.y * b.yx + a.x.z * b.zx;
    r.x.y = a.x.x * b.yx + a.x.y * b.yy + a.x.z * b.zy;
    r.x.z = a.x.x * b.zx + a.x.y * b.zy + a.x.z * b.zz;
    r.y.x = a.y.x * b.xx + a.y.y * b.yx + a.y.z * b.zx;
    r.y.y = a.y.x * b.yx + a.y.y * b.yy + a.y.z * b.zy;
    r.y.z = a.y.x * b.zx + a.y.y * b.zy + a.y.z * b.zz;
    return r;
}
// MultiplyWithoutOverlap(Matrix3x3Wide a, Symmetric3x3Wide b)
template <class F> inline M33<F> multiply(const M33<F>& a, const Sym3<F>& b) {
    M33<F> r;
    r.x.x = a.x.x * b.xx + a.x.y * b.yx + a.x.z * b.zx;
    r.x.y = a.x.x * b.yx + a.x.y * b.yy + a.x.z * b.zy;
    r.x.z = a.x.x * b.zx + a.x.y * b.zy + a.x.z * b.zz;
    r.y.x = a.y.x * b.xx + a.y.y * b.yx + a.y.z * b.zx;
    r.y.y = a.y.x * b.yx + a.y.y * b.yy + a.y.z * b.zy;
    r.y.z = a.y.x * b.zx + a.y.y * b.zy + a.y.z * b.zz;
    r.z.x = a.z.x * b.xx + a.z.y * b.yx + a.z.z * b.zx;
    r.z.y = a.z.x * b.yx + a.z.y * b.yy + a.z.z * b.zy;
    r.z.z = a.z.x * b.zx + a.z.y * b.zy + a.z.z * b.zz;
    return r;
}
// CompleteMatrixSandwich(Matrix2x3Wide a, Matrix2x3Wide b) -> Symmetric3x3Wide : aT * b
template <class F> inline Sym3<F> complete_matrix_sandwich_t(const M23<F>& a, const M23<F>& b) {
    Sym3<F> r;
    r.xx = a.x.x * b.x.x + a.y.x * b.y.x;
    r.yx = a.x.y * b.x.x + a.y.y * b.y.x;
    r.yy = a.x.y * b.x.y + a.y.y * b.y.y;
    r.zx = a.x.z * b.x.x + a.y.z * b.y.x;
    r.zy = a.x.z * b.x.y + a.y.z * b.y.y;
    r.zz = a.x.z * b.x.z + a.y.z * b.y.z;
    return r;
}

// ---- Symmetric2x2Wide (BepuUtilities/Symmetric2x2Wide.cs) ---------------------------------------------------------
// L14-19 SandwichScale
template <class F> inline Sym2<F> sandwich_scale(const M23<F>& m, const F& s) {
    Sym2<F> r;
    r.xx = s * (m.x.x * m.x.x + m.x.y * m.x.y + m.x.z * m.x.z);
    r.yx = s * (m.y.x * m.x.x + m.y.y * m.x.y + m.y.z * m.x.z);
    r.yy = s * (m.y.x * m.y.x + m.y.y * m.y.y + m.y.z * m.y.z);
    return r;
}
template <class F> inline Sym2<F> add(const Sym2<F>& a, const Sym2<F>& b) { return {a.xx + b.xx, a.yx + b.yx, a.yy + b.yy}; }
// L55-62 InvertWithoutOverlap
template <class F> inline Sym2<F> invert(const Sym2<F>& m) {
    F denom = bc<F>(1.0f) / (m.yx * m.yx - m.xx * m.yy);
    return {-m.yy * denom, m.yx * denom, -m.xx * denom};
}
// TransformWithoutOverlap(Vector2Wide, Symmetric2x2Wide)
template <class F> inline V2<F> transform(const V2<F>& v, const Sym2<F>& m) {
    return {v.x * m.xx + v.y * m.yx, v.x * m.yx + v.y * m.yy};
}
// CompleteMatrixSandwich(Matrix2x3Wide a, Matrix2x3Wide b) -> Symmetric2x2Wide : a * bT
template <class F> inline Sym2<F> complete_matrix_sandwich(const M23<F>& a, const M23<F>& b) {
    Sym2<F> r;
    r.xx = a.x.x * b.x.x + a.x.y * b.x.y + a.x.z * b.x.z;
    r.yx = a.y.x * b.x.x + a.y.y * b.x.y + a.y.z * b.x.z;
    r.yy = a.y.x * b.y.x + a.y.y * b.y.y + a.y.z * b.y.z;
    return r;
}

// ---- Matrix2x3Wide (BepuUtilities/Matrix2x3Wide.cs) ---------------------------------------------------------------
// TransformByTransposeWithoutOverlap: v * mT
template <class F> inline V2<F> transform_by_transpose(const V3<F>& v, const M23<F>& m) {
    return {v.x * m.x.x + v.y * m.x.y + v.z * m.x.z, v.x * m.y.x + v.y * m.y.y + v.z * m.y.z};
}
// Transform(Vector2Wide, Matrix2x3Wide): v * m
template <class F> inline V3<F> transform(const V2<F>& v, const M23<F>& m) {
    return {v.x * m.x.x + v.y * m.y.x, v.x * m.x.y + v.y * m.y.y, v.x * m.x.z + v.y * m.y.z};
}

// ---- Matrix3x3Wide (BepuUtilities/Matrix3x3Wide.cs) ---------------------------------------------------------------
// L238-265 CreateFromQuaternion
template <class F> inline M33<F> matrix_from_quaternion(const Q4<F>& q) {
    F qx2 = q.x + q.x, qy2 = q.y + q.y, qz2 = q.z + q.z;
    F YY = qy2 * q.y, ZZ = qz2 * q.z;
    M33<F> r;
    r.x.x = bc<F>(1.0f) - YY - ZZ;
    F XY = qx2 * q.y, ZW = qz2 * q.w;
    r.x.y = XY + ZW;
    F XZ = qx2 * q.z, YW = qy2 * q.w;
    r.x.z = XZ - YW;
    F XX = qx2 * q.x;
    r.y.x = XY - ZW;
    r.y.y = bc<F>(1.0f) - XX - ZZ;
    F XW = qx2 * q.w, YZ = qy2 * q.z;
    r.y.z = YZ + XW;
    r.z.x = XZ + YW;
    r.z.y = YZ - XW;
    r.z.z = bc<F>(1.0f) - XX - YY;
    return r;
}
// TransformWithoutOverlap(v, m): v * m
template <class F> inline V3<F> transform(const V3<F>& v, const M33<F>& m) {
    return {v.x * m.x.x + v.y * m.y.x + v.z * m.z.x, v.x * m.x.y + v.y * m.y.y + v.z * m.z.y, v.x * m.x.z + v.y * m.y.z + v.z * m.z.z};
}
// TransformByTransposedWithoutOverlap(v, m): v * mT
template <class F> inline V3<F> transform_by_transposed(const V3<F>& v, const M33<F>& m) {
    return {v.x * m.x.x + v.y * m.x.y + v.z * m.x.z, v.x * m.y.x + v.y * m.y.y + v.z * m.y.z, v.x * m.z.x + v.y * m.z.y + v.z * m.z.z};
}

// ---- QuaternionWide (BepuUtilities/QuaternionWide.cs) -------------------------------------------------------------
// L124-134 Normalize
template <class F> inline Q4<F> normalize(const Q4<F>& q) {
    F inv = bc<F>(1.0f) / vsqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    return {q.x * inv, q.y * inv, q.z * inv, q.w * inv};
}
// L500-506 ConcatenateWithoutOverlap
template <class F> inline Q4<F> concatenate(const Q4<F>& a, const Q4<F>& b) {
    Q4<F> r;
    r.x = a.w * b.x + a.x * b.w + a.z * b.y - a.y * b.z;
    r.y = a.w * b.y + a.y * b.w + a.x * b.z - a.z * b.x;
    r.z = a.w * b.z + a.z * b.w + a.y * b.x - a.x * b.y;
    r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
    return r;
}
// L546-553 Conjugate (negates W, as the reference does)
template <class F> inline Q4<F> conjugate(const Q4<F>& q) { return {q.x, q.y, q.z, -q.w}; }
// L252-274 TransformWithoutOverlap(v, rotation)
template <class F> inline V3<F> transform(const V3<F>& v, const Q4<F>& r) {
    F x2 = r.x + r.x, y2 = r.y + r.y, z2 = r.z + r.z;
    F xx2 = r.x * x2, xy2 = r.x * y2, xz2 = r.x * z2;
    F yy2 = r.y * y2, yz2 = r.y * z2, zz2 = r.z * z2;
    F wx2 = r.w * x2, wy2 = r.w * y2, wz2 = r.w * z2;
    F one = bc<F>(1.0f);
    V3<F> o;
    o.x = v.x * (one - yy2 - zz2) + v.y * (xy2 - wz2) + v.z * (xz2 + wy2);
    o.y = v.x * (xy2 + wz2) + v.y * (one - xx2 - zz2) + v.z * (yz2 - wx2);
    o.z = v.x * (xz2 - wy2) + v.y * (yz2 + wx2) + v.z * (one - xx2 - yy2);
    return o;
}
// L366-381 TransformUnitX, L389-405 TransformUnitY, L413-429 TransformUnitZ
template <class F> inline V3<F> transform_unit_x(const Q4<F>& r) {
    F y2 = r.y + r.y, z2 = r.z + r.z;
    F xy2 = r.x * y2, xz2 = r.x * z2, yy2 = r.y * y2, zz2 = r.z * z2, wy2 = r.w * y2, wz2 = r.w * z2;
    return {bc<F>(1.0f) - yy2 - zz2, xy2 + wz2, xz2 - wy2};
}
template <class F> inline V3<F> transform_unit_y(const Q4<F>& r) {
    F x2 = r.x + r.x, y2 = r.y + r.y, z2 = r.z + r.z;
    F xx2 = r.x * x2, xy2 = r.x * y2, yz2 = r.y * z2, zz2 = r.z * z2, wx2 = r.w * x2, wz2 = r.w * z2;
    return {xy2 - wz2, bc<F>(1.0f) - xx2 - zz2, yz2 + wx2};
}
template <class F> inline V3<F> transform_unit_z(const Q4<F>& r) {
    F x2 = r.x + r.x, y2 = r.y + r.y, z2 = r.z + r.z;
    F xx2 = r.x * x2, xz2 = r.x * z2, yy2 = r.y * y2, yz2 = r.y * z2, wx2 = r.w * x2, wy2 = r.w * y2;
    return {xz2 + wy2, yz2 - wx2, bc<F>(1.0f) - xx2 - yy2};
}
// L438-459 TransformUnitXY
template <class F> inline void transform_unit_xy(const Q4<F>& r, V3<F>& x, V3<F>& y) {
    F x2 = r.x + r.x, y2 = r.y + r.y, z2 = r.z + r.z;
    F xx2 = r.x * x2, xy2 = r.x * y2, xz2 = r.x * z2, yy2 = r.y * y2, yz2 = r.y * z2, zz2 = r.z * z2;
    F wx2 = r.w * x2, wy2 = r.w * y2, wz2 = r.w * z2;
    F one = bc<F>(1.0f);
    x = {one - yy2 - zz2, xy2 + wz2, xz2 - wy2};
    y = {xy2 - wz2, one - xx2 - zz2, yz2 + wx2};
}

// ---- MathHelper (BepuUtilities/MathHelper.cs) ---------------------------------------------------------------------
static constexpr float kPi = 3.141592653589793239f;        // L17
static constexpr float kTwoPi = 6.283185307179586477f;     // L22
static constexpr float kPiOver2 = 1.570796326794896619f;   // L27
static constexpr float kInvTwoPi = (float)(0.5 / 3.14159265358979323846);  // (float)(0.5 / Math.PI)

// L274-311 Cos(Vector<float>)
template <class F> inline F cos_approx(const F& x) {
    F periodCount = x * bc<F>(kInvTwoPi);
    F periodFraction = periodCount - vfloor(periodCount);
    F periodX = periodFraction * bc<F>(kTwoPi);
    F piOver2 = bc<F>(kPiOver2), pi = bc<F>(kPi), pi3Over2 = bc<F>(3 * kPiOver2);
    F y = sel(gt(periodX, piOver2), pi - periodX, periodX);
    y = sel(gt(periodX, pi), periodX - pi, y);
    y = sel(gt(periodX, pi3Over2), bc<F>(kTwoPi) - periodX, y);
    F numerator = ((((bc<F>(-0.003436308368583229f) * y + bc<F>(0.021317031205957775f)) * y + bc<F>(0.06955843390178032f)) * y - bc<F>(0.4578088075324152f)) * y - bc<F>(0.15082367674208508f)) * y + bc<F>(1.0f);
    F denominator = ((((bc<F>(-0.00007650398834677185f) * y + bc<F>(0.0007451378206294365f)) * y - bc<F>(0.00585321045829395f)) * y + bc<F>(0.04219116713777847f)) * y - bc<F>(0.15082367538305258f)) * y + bc<F>(1.0f);
    F result = numerator / denominator;
    return sel(mand(gt(periodX, piOver2), lt(periodX, pi3Over2)), -result, result);
}
// L317-351 Sin(Vector<float>)
template <class F> inline F sin_approx(const F& x) {
    F periodCount = x * bc<F>(kInvTwoPi);
    F periodFraction = periodCount - vfloor(periodCount);
    F twoPi = bc<F>(kTwoPi);
    F periodX = periodFraction * twoPi;
    F pi = bc<F>(kPi), piOver2 = bc<F>(kPiOver2);
    F y = sel(gt(periodX, piOver2), pi - periodX, periodX);
    MaskOf<F> inSecondHalf = gt(periodX, pi);
    y = sel(inSecondHalf, periodX - pi, y);
    y = sel(gt(periodX, bc<F>(3 * kPiOver2)), twoPi - periodX, y);
    F numerator = ((((bc<F>(0.0040507708755727605f) * y - bc<F>(0.006685815219853882f)) * y - bc<F>(0.13993701695343166f)) * y + bc<F>(0.06174562337697123f)) * y + bc<F>(1.00000000151466040f)) * y;
    F denominator = ((((bc<F>(0.00009018370615921334f) * y + bc<F>(0.0001700784176413186f)) * y + bc<F>(0.003606014457152456f)) * y + bc<F>(0.02672943625500751f)) * y + bc<F>(0.061745651499203795f)) * y + bc<F>(1.0f);
    F result = numerator / denominator;
    return sel(inSecondHalf, -result, result);
}
// L353-362 Acos(Vector<float>)
template <class F> inline F acos_approx(const F& xin) {
    MaskOf<F> negativeInput = lt(xin, bc<F>(0.0f));
    F x = vmin(bc<F>(1.0f), vabs(xin));
    F numerator = vsqrt(bc<F>(1.0f) - x) * (bc<F>(62.95741097600742f) + x * (bc<F>(69.6550664543659f) + x * (bc<F>(17.54512349463405f) + x * bc<F>(0.6022076120669532f))));
    F denominator = bc<F>(40.07993264439811f) + x * (bc<F>(49.81949855726789f) + x * (bc<F>(15.703851745284796f) + x));
    F result = numerator / denominator;
    return sel(negativeInput, bc<F>(kPi) - result, result);
}
// L369-375 GetSignedAngleDifference
template <class F> inline F signed_angle_difference(const F& a, const F& b) {
    F half = bc<F>(0.5f);
    F x = (b - a) * bc<F>(1.0f / kTwoPi) + half;
    return (x - vfloor(x) - half) * bc<F>(kTwoPi);
}

// QuaternionWide.cs:L162-186 GetQuaternionBetweenNormalizedVectors
template <class F> inline Q4<F> quaternion_between_normalized(const V3<F>& v1, const V3<F>& v2) {
    F d = dot(v1, v2);
    V3<F> c = cross(v1, v2);
    MaskOf<F> useNormalCase = gt(d, bc<F>(-0.999999f));
    F absX = vabs(v1.x), absY = vabs(v1.y), absZ = vabs(v1.z);
    MaskOf<F> xIsSmallest = mand(lt(absX, absY), lt(absX, absZ));
    MaskOf<F> yIsSmaller = lt(absY, absZ);
    F zero = bc<F>(0.0f);
    Q4<F> q;
    q.x = sel(useNormalCase, c.x, sel(xIsSmallest, zero, sel(yIsSmaller, -v1.z, -v1.y)));
    q.y = sel(useNormalCase, c.y, sel(xIsSmallest, -v1.z, sel(yIsSmaller, zero, v1.x)));
    q.z = sel(useNormalCase, c.z, sel(xIsSmallest, v1.y, sel(yIsSmaller, v1.x, zero)));
    q.w = sel(useNormalCase, d + bc<F>(1.0f), zero);
    return normalize(q);
}
// QuaternionWide.cs:L227-243 GetAxisAngleFromQuaternion
template <class F> inline void axis_angle_from_quaternion(const Q4<F>& q, V3<F>& axis, F& angle) {
    MaskOf<F> shouldNegate = lt(q.w, bc<F>(0.0f));
    axis.x = sel(shouldNegate, -q.x, q.x);
    axis.y = sel(shouldNegate, -q.y, q.y);
    axis.z = sel(shouldNegate, -q.z, q.z);
    F qw = sel(shouldNegate, -q.w, q.w);
    F axisLength = length(axis);
    axis = scale(axis, F(bc<F>(1.0f) / axisLength));
    MaskOf<F> useFallback = lt(axisLength, bc<F>(1e-14f));
    axis.x = sel(useFallback, bc<F>(1.0f), axis.x);
    axis.y = sel(useFallback, bc<F>(0.0f), axis.y);
    axis.z = sel(useFallback, bc<F>(0.0f), axis.z);
    F halfAngle = acos_approx(qw);
    angle = bc<F>(2.0f) * halfAngle;
}

// BepuPhysics/Helpers.cs:L21-35 BuildOrthonormalBasis
template <class F> inline void build_orthonormal_basis(const V3<F>& n, V3<F>& t1, V3<F>& t2) {
    F sign = sel(lt(n.z, bc<F>(0.0f)), bc<F>(-1.0f), bc<F>(1.0f));
    F scl = bc<F>(-1.0f) / (sign + n.z);
    t1.x = n.x * n.y * scl;
    t1.y = sign + n.y * n.y * scl;
    t1.z = -n.y;
    t2.x = bc<F>(1.0f) + sign * n.x * n.x * scl;
    t2.y = sign * t1.x;
    t2.z = -sign * n.x;
}
// Helpers.cs:L37-47 FindPerpendicular
template <class F> inline V3<F> find_perpendicular(const V3<F>& n) {
    F sign = sel(lt(n.z, bc<F>(0.0f)), bc<F>(-1.0f), bc<F>(1.0f));
    F scl = bc<F>(-1.0f) / (sign + n.z);
    return {n.x * n.y * scl, sign + n.y * n.y * scl, -n.y};
}

// BepuPhysics/Constraints/SpringSettings.cs:L37-55 ComputeSpringiness
template <class F> inline void compute_springiness(const F& angular_frequency, const F& twice_damping_ratio, float dt,
                                                   F& position_error_to_velocity, F& effective_mass_cfm_scale, F& softness_impulse_scale) {
    F angularFrequencyDt = angular_frequency * bc<F>(dt);
    position_error_to_velocity = angular_frequency / (angularFrequencyDt + twice_damping_ratio);
    F extra = bc<F>(1.0f) / (angularFrequencyDt * (angularFrequencyDt + twice_damping_ratio));
    effective_mass_cfm_scale = bc<F>(1.0f) / (bc<F>(1.0f) + extra);
    softness_impulse_scale = extra * effective_mass_cfm_scale;
}

}  // namespace bepu_oracle
