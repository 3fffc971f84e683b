// Device-side fp32 math for the sm_90a constraint kernels. One thread = one constraint lane, so everything here is
// plain scalar code on small register-resident aggregates.
//
// Expression shapes follow the reference's wide math (file:line cited per function) so that the strict build
// (-fmad=false, IEEE div/sqrt) reproduces a non-contracting CPU evaluation bit for bit; the fast build lets ptxas
// contract the same expressions into FFMA.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace BEPU_NS {

#define BEPU_DI __device__ __forceinline__

struct V2 { float x, y; };
struct V3 { float x, y, z; };
struct Q4 { float x, y, z, w; };
struct Sym2 { float xx, yx, yy; };
struct Sym3 { float xx, yx, yy, zx, zy, zz; };
struct M23 { V3 x, y; };
struct M33 { V3 x, y, z; };
struct Velocity { V3 lin, ang; };
struct Inertia { Sym3 t; float inv_mass; };
struct BodyState { V3 pos; Q4 q; Inertia inertia; };  // what a constraint function may see of one body

// minps / maxps semantics of Vector.Min / Vector.Max: (a < b) ? a : b, (a > b) ? a : b.
BEPU_DI float fmin_ps(float a, float b) { return a < b ? a : b; }
BEPU_DI float fmax_ps(float a, float b) { return a > b ? a : b; }

// BepuUtilities/Vector3Wide.cs:L55-66, L127-138, L201-204, L343-350, L519-525, L562-576, L627-633
BEPU_DI V3 operator+(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
BEPU_DI V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
BEPU_DI V3 operator*(V3 a, float s) { return {a.x * s, a.y * s, a.z * s}; }
BEPU_DI V3 operator-(V3 a) { return {-a.x, -a.y, -a.z}; }
BEPU_DI float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
BEPU_DI V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
BEPU_DI float length_squared(V3 v) { return v.x * v.x + v.y * v.y + v.z * v.z; }
BEPU_DI float length(V3 v) { return sqrtf(v.x * v.x + v.y * v.y + v.z * v.z); }
BEPU_DI float distance(V3 a, V3 b) {
    float x = b.x - a.x, y = b.y - a.y, z = b.z - a.z;
    return sqrtf(x * x + y * y + z * z);
}
BEPU_DI V3 normalize(V3 v) { return v * (1.0f / length(v)); }  // Vector3Wide.cs:L688-693
BEPU_DI V3 select(bool m, V3 a, V3 b) { return m ? a : b; }
BEPU_DI V2 operator+(V2 a, V2 b) { return {a.x + b.x, a.y + b.y}; }
BEPU_DI V2 operator-(V2 a, V2 b) { return {a.x - b.x, a.y - b.y}; }
BEPU_DI V2 operator*(V2 a, float s) { return {a.x * s, a.y * s}; }
BEPU_DI float length(V2 v) { return sqrtf(v.x * v.x + v.y * v.y); }

// ---- BepuUtilities/Symmetric3x3Wide.cs ----
BEPU_DI Sym3 invert(Sym3 m) {  // L42-66
    float xx = m.yy * m.zz - m.zy * m.zy;
    float yx = m.zy * m.zx - m.zz * m.yx;
    float zx = m.yx * m.zy - m.zx * m.yy;
    float det_inv = 1.0f / (xx * m.xx + yx * m.yx + zx * m.zx);
    float yy = m.zz * m.xx - m.zx * m.zx;
    float zy = m.zx * m.yx - m.xx * m.zy;
    float zz = m.xx * m.yy - m.yx * m.yx;
    return {xx * det_inv, yx * det_inv, yy * det_inv, zx * det_inv, zy * det_inv, zz * det_inv};
}
BEPU_DI Sym3 operator+(Sym3 a, Sym3 b) { return {a.xx + b.xx, a.yx + b.yx, a.yy + b.yy, a.zx + b.zx, a.zy + b.zy, a.zz + b.zz}; }
BEPU_DI Sym3 operator*(Sym3 m, float s) { return {m.xx * s, m.yx * s, m.yy * s, m.zx * s, m.zy * s, m.zz * s}; }
BEPU_DI Sym3 skew_sandwich(V3 v, Sym3 m) {  // L182-208: skew(v) * m * skew(v)^T
    float xzy = v.x * m.zy, yzx = v.y * m.zx, zyx = v.z * m.yx;
    float ixy = v.y * m.zy - v.z * m.yy;
    float ixz = v.y * m.zz - v.z * m.zy;
    float iyx = v.z * m.xx - v.x * m.zx;
    float iyy = zyx - xzy;
    float iyz = v.z * m.zx - v.x * m.zz;
    float izx = v.x * m.yx - v.y * m.xx;
    float izy = v.x * m.yy - v.y * m.yx;
    float izz = xzy - yzx;
    Sym3 s;
    s.xx = v.y * ixz - v.z * ixy;
    s.yx = v.y * iyz - v.z * iyy;
    s.yy = v.z * iyx - v.x * iyz;
    s.zx = v.y * izz - v.z * izy;
    s.zy = v.z * izx - v.x * izz;
    s.zz = v.x * izy - v.y * izx;
    return s;
}
BEPU_DI float vector_sandwich(V3 v, Sym3 m) {  // L214-222
    float x = v.x * m.xx + v.y * m.yx + v.z * m.zx;
    float y = v.x * m.yx + v.y * m.yy + v.z * m.zy;
    float z = v.x * m.zx + v.y * m.zy + v.z * m.zz;
    return x * v.x + y * v.y + z * v.z;
}
BEPU_DI Sym3 rotation_sandwich(const M33& r, Sym3 m) {  // L231-258: r^T * m * r
    float ixx = r.x.x * m.xx + r.y.x * m.yx + r.z.x * m.zx;
    float ixy = r.x.x * m.yx + r.y.x * m.yy + r.z.x * m.zy;
    float ixz = r.x.x * m.zx + r.y.x * m.zy + r.z.x * m.zz;
    float iyx = r.x.y * m.xx + r.y.y * m.yx + r.z.y * m.zx;
    float iyy = r.x.y * m.yx + r.y.y * m.yy + r.z.y * m.zy;
    float iyz = r.x.y * m.zx + r.y.y * m.zy + r.z.y * m.zz;
    float izx = r.x.z * m.xx + r.y.z * m.yx + r.z.z * m.zx;
    float izy = r.x.z * m.yx + r.y.z * m.yy + r.z.z * m.zy;
    float izz = r.x.z * m.zx + r.y.z * m.zy + r.z.z * m.zz;
    Sym3 s;
    s.xx = ixx * r.x.x + ixy * r.y.x + ixz * r.z.x;
    s.yx = iyx * r.x.x + iyy * r.y.x + iyz * r.z.x;
    s.yy = iyx * r.x.y + iyy * r.y.y + iyz * r.z.y;
    s.zx = izx * r.x.x + izy * r.y.x + izz * r.z.x;
    s.zy = izx * r.x.y + izy * r.y.y + izz * r.z.y;
    s.zz = izx * r.x.z + izy * r.y.z + izz * r.z.z;
    return s;
}
BEPU_DI Sym2 matrix_sandwich(const M23& m, Sym3 t) {  // MatrixSandwich(Matrix2x3Wide, Symmetric3x3Wide)
    float ixx = m.x.x * t.xx + m.x.y * t.yx + m.x.z * t.zx;
    float ixy = m.x.x * t.yx + m.x.y * t.yy + m.x.z * t.zy;
    float ixz = m.x.x * t.zx + m.x.y * t.zy + m.x.z * t.zz;
    float iyx = m.y.x * t.xx + m.y.y * t.yx + m.y.z * t.zx;
    float iyy = m.y.x * t.yx + m.y.y * t.yy + m.y.z * t.zy;
    float iyz = m.y.x * t.zx + m.y.y * t.zy + m.y.z * t.zz;
    Sym2 r;
    r.xx = ixx * m.x.x + ixy * m.x.y + ixz * m.x.z;
    r.yx = iyx * m.x.x + iyy * m.x.y + iyz * m.x.z;
    r.yy = iyx * m.y.x + iyy * m.y.y + iyz * m.y.z;
    return r;
}
BEPU_DI V3 transform(V3 v, Sym3 m) {  // TransformWithoutOverlap(Vector3Wide, Symmetric3x3Wide)
    return {v.x * m.xx + v.y * m.yx + v.z * m.zx, v.x * m.yx + v.y * m.yy + v.z * m.zy, v.x * m.zx + v.y * m.zy + v.z * m.zz};
}
BEPU_DI M23 multiply(const M23& a, Sym3 b) {  // MultiplyWithoutOverlap(Matrix2x3Wide, Symmetric3x3Wide)
    M23 r;
    r.x.x = a.x.x * b.xx + a.x.y * b.yx + a.x.z * b.zx;
    r.x.y = a.x.x * b.yx + a.x.y * b.yy + a.x.z * b.zy;
    r.x.z = a.x.x * b.zx + a.x.y * b.zy + a.x.z * b.zz;
    r.y.x = a.y.x * b.xx + a.y.y * b.yx + a.y.z * b.zx;
    r.y.y = a.y.x * b.yx + a.y.y * b.yy + a.y.z * b.zy;
    r.y.z = a.y.x * b.zx + a.y.y * b.zy + a.y.z * b.zz;
    return r;
}
BEPU_DI M33 multiply(const M33& a, Sym3 b) {  // MultiplyWithoutOverlap(Matrix3x3Wide, Symmetric3x3Wide)
    M33 r;
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
BEPU_DI Sym3 complete_matrix_sandwich_t(const M23& a, const M23& b) {  // CompleteMatrixSandwich(Matrix2x3Wide, Matrix2x3Wide) -> Symmetric3x3Wide: a^T b
    Sym3 r;
    r.xx = a.x.x * b.x.x + a.y.x * b.y.x;
    r.yx = a.x.y * b.x.x + a.y.y * b.y.x;
    r.yy = a.x.y * b.x.y + a.y.y * b.y.y;
    r.zx = a.x.z * b.x.x + a.y.z * b.y.x;
    r.zy = a.x.z * b.x.y + a.y.z * b.y.y;
    r.zz = a.x.z * b.x.z + a.y.z * b.y.z;
    return r;
}

// ---- BepuUtilities/Symmetric2x2Wide.cs ----
BEPU_DI Sym2 sandwich_scale(const M23& m, float s) {  // L14-19
    Sym2 r;
    r.xx = s * (m.x.x * m.x.x + m.x.y * m.x.y + m.x.z * m.x.z);
    r.yx = s * (m.y.x * m.x.x + m.y.y * m.x.y + m.y.z * m.x.z);
    r.yy = s * (m.y.x * m.y.x + m.y.y * m.y.y + m.y.z * m.y.z);
    return r;
}
BEPU_DI Sym2 operator+(Sym2 a, Sym2 b) { return {a.xx + b.xx, a.yx + b.yx, a.yy + b.yy}; }
BEPU_DI Sym2 invert(Sym2 m) {  // L55-62
    float denom = 1.0f / (m.yx * m.yx - m.xx * m.yy);
    return {-m.yy * denom, m.yx * denom, -m.xx * denom};
}
BEPU_DI V2 transform(V2 v, Sym2 m) { return {v.x * m.xx + v.y * m.yx, v.x * m.yx + v.y * m.yy}; }
BEPU_DI Sym2 complete_matrix_sandwich(const M23& a, const M23& b) {  // a * b^T
    Sym2 r;
    r.xx = a.x.x * b.x.x + a.x.y * b.x.y + a.x.z * b.x.z;
    r.yx = a.y.x * b.x.x + a.y.y * b.x.y + a.y.z * b.x.z;
    r.yy = a.y.x * b.y.x + a.y.y * b.y.y + a.y.z * b.y.z;
    return r;
}

// ---- BepuUtilities/Matrix2x3Wide.cs ----
BEPU_DI V2 transform_by_transpose(V3 v, const M23& m) {
    return {v.x * m.x.x + v.y * m.x.y + v.z * m.x.z, v.x * m.y.x + v.y * m.y.y + v.z * m.y.z};
}
BEPU_DI V3 transform(V2 v, const M23& m) {
    return {v.x * m.x.x + v.y * m.y.x, v.x * m.x.y + v.y * m.y.y, v.x * m.x.z + v.y * m.y.z};
}

// ---- BepuUtilities/Matrix3x3Wide.cs ----
BEPU_DI M33 matrix_from_quaternion(Q4 q) {  // L238-265
    float qx2 = q.x + q.x, qy2 = q.y + q.y, qz2 = q.z + q.z;
    float YY = qy2 * q.y, ZZ = qz2 * q.z;
    M33 r;
    r.x.x = 1.0f - YY - ZZ;
    float XY = qx2 * q.y, ZW = qz2 * q.w;
    r.x.y = XY + ZW;
    float XZ = qx2 * q.z, YW = qy2 * q.w;
    r.x.z = XZ - YW;
    float XX = qx2 * q.x;
    r.y.x = XY - ZW;
    r.y.y = 1.0f - XX - ZZ;
    float XW = qx2 * q.w, YZ = qy2 * q.z;
    r.y.z = YZ + XW;
    r.z.x = XZ + YW;
    r.z.y = YZ - XW;
    r.z.z = 1.0f - XX - YY;
    return r;
}
BEPU_DI V3 transform(V3 v, const M33& m) {
    return {v.x * m.x.x + v.y * m.y.x + v.z * m.z.x, v.x * m.x.y + v.y * m.y.y + v.z * m.z.y, v.x * m.x.z + v.y * m.y.z + v.z * m.z.z};
}
BEPU_DI V3 transform_by_transposed(V3 v, const M33& m) {
    return {v.x * m.x.x + v.y * m.x.y + v.z * m.x.z, v.x * m.y.x + v.y * m.y.y + v.z * m.y.z, v.x * m.z.x + v.y * m.z.y + v.z * m.z.z};
}
BEPU_DI M33 invert(const M33& m) {  // L142-166
    float m11 = m.y.y * m.z.z - m.z.y * m.y.z;
    float m21 = m.y.z * m.z.x - m.z.z * m.y.x;
    float m31 = m.y.x * m.z.y - m.z.x * m.y.y;
    float di = 1.0f / (m11 * m.x.x + m21 * m.x.y + m31 * m.x.z);
    float m12 = m.z.y * m.x.z - m.x.y * m.z.z;
    float m22 = m.z.z * m.x.x - m.x.z * m.z.x;
    float m32 = m.z.x * m.x.y - m.x.x * m.z.y;
    float m13 = m.x.y * m.y.z - m.y.y * m.x.z;
    float m23 = m.x.z * m.y.x - m.y.z * m.x.x;
    float m33 = m.x.x * m.y.y - m.y.x * m.x.y;
    M33 r;
    r.x = {m11 * di, m12 * di, m13 * di};
    r.y = {m21 * di, m22 * di, m23 * di};
    r.z = {m31 * di, m32 * di, m33 * di};
    return r;
}

// ---- BepuUtilities/QuaternionWide.cs ----
BEPU_DI Q4 normalize(Q4 q) {  // L124-134
    float inv = 1.0f / sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    return {q.x * inv, q.y * inv, q.z * inv, q.w * inv};
}
BEPU_DI Q4 concatenate(Q4 a, Q4 b) {  // L500-506
    Q4 r;
    r.x = a.w * b.x + a.x * b.w + a.z * b.y - a.y * b.z;
    r.y = a.w * b.y + a.y * b.w + a.x * b.z - a.z * b.x;
    r.z = a.w * b.z + a.z * b.w + a.y * b.x - a.x * b.y;
    r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
    return r;
}
BEPU_DI Q4 conjugate(Q4 q) { return {q.x, q.y, q.z, -q.w}; }  // L546-553 (negates W)
BEPU_DI V3 transform(V3 v, Q4 r) {  // L252-274
    float x2 = r.x + r.x, y2 = r.y + r.y, z2 = r.z + r.z;
    float xx2 = r.x * x2, xy2 = r.x * y2, xz2 = r.x * z2;
    float yy2 = r.y * y2, yz2 = r.y * z2, zz2 = r.z * z2;
    float wx2 = r.w * x2, wy2 = r.w * y2, wz2 = r.w * z2;
    V3 o;
    o.x = v.x * (1.0f - yy2 - zz2) + v.y * (xy2 - wz2) + v.z * (xz2 + wy2);
    o.y = v.x * (xy2 + wz2) + v.y * (1.0f - xx2 - zz2) + v.z * (yz2 - wx2);
    o.z = v.x * (xz2 - wy2) + v.y * (yz2 + wx2) + v.z * (1.0f - xx2 - yy2);
    return o;
}
BEPU_DI V3 transform_unit_x(Q4 r) {  // L366-381
    float y2 = r.y + r.y, z2 = r.z + r.z;
    float xy2 = r.x * y2, xz2 = r.x * z2, yy2 = r.y * y2, zz2 = r.z * z2, wy2 = r.w * y2, wz2 = r.w * z2;
    return {1.0f - yy2 - zz2, xy2 + wz2, xz2 - wy2};
}
BEPU_DI V3 transform_unit_y(Q4 r) {  // L389-405
    float x2 = r.x + r.x, y2 = r.y + r.y, z2 = r.z + r.z;
    float xx2 = r.x * x2, xy2 = r.x * y2, yz2 = r.y * z2, zz2 = r.z * z2, wx2 = r.w * x2, wz2 = r.w * z2;
    return {xy2 - wz2, 1.0f - xx2 - zz2, yz2 + wx2};
}
BEPU_DI V3 transform_unit_z(Q4 r) {  // L413-429
    float x2 = r.x + r.x, y2 = r.y + r.y, z2 = r.z + r.z;
    float xx2 = r.x * x2, xz2 = r.x * z2, yy2 = r.y * y2, yz2 = r.y * z2, wx2 = r.w * x2, wy2 = r.w * y2;
    return {xz2 + wy2, yz2 - wx2, 1.0f - xx2 - yy2};
}
BEPU_DI void transform_unit_xy(Q4 r, V3& x, V3& y) {  // L438-459
    float x2 = r.x + r.x, y2 = r.y + r.y, z2 = r.z + r.z;
    float xx2 = r.x * x2, xy2 = r.x * y2, xz2 = r.x * z2, yy2 = r.y * y2, yz2 = r.y * z2, zz2 = r.z * z2;
    float wx2 = r.w * x2, wy2 = r.w * y2, wz2 = r.w * z2;
    x = {1.0f - yy2 - zz2, xy2 + wz2, xz2 - wy2};
    y = {xy2 - wz2, 1.0f - xx2 - zz2, yz2 + wx2};
}

// ---- BepuUtilities/MathHelper.cs: custom rational approximations, NOT sinf/cosf/acosf ----
#define BEPU_PI 3.141592653589793239f
#define BEPU_TWO_PI 6.283185307179586477f
#define BEPU_PI_OVER_2 1.570796326794896619f
#define BEPU_INV_TWO_PI 0.15915494309189533577f  // (float)(0.5 / Math.PI)

BEPU_DI float cos_approx(float x) {  // L274-311
    float periodCount = x * BEPU_INV_TWO_PI;
    float periodFraction = periodCount - floorf(periodCount);
    float periodX = periodFraction * BEPU_TWO_PI;
    const float pi3Over2 = 3 * BEPU_PI_OVER_2;
    float y = periodX > BEPU_PI_OVER_2 ? BEPU_PI - periodX : periodX;
    y = periodX > BEPU_PI ? periodX - BEPU_PI : y;
    y = periodX > pi3Over2 ? BEPU_TWO_PI - periodX : y;
    float numerator = ((((-0.003436308368583229f * y + 0.021317031205957775f) * y + 0.06955843390178032f) * y - 0.4578088075324152f) * y - 0.15082367674208508f) * y + 1.0f;
    float denominator = ((((-0.00007650398834677185f * y + 0.0007451378206294365f) * y - 0.00585321045829395f) * y + 0.04219116713777847f) * y - 0.15082367538305258f) * y + 1.0f;
    float result = numerator / denominator;
    return (periodX > BEPU_PI_OVER_2 && periodX < pi3Over2) ? -result : result;
}
BEPU_DI float sin_approx(float x) {  // L317-351
    float periodCount = x * BEPU_INV_TWO_PI;
    float periodFraction = periodCount - floorf(periodCount);
    float periodX = periodFraction * BEPU_TWO_PI;
    float y = periodX > BEPU_PI_OVER_2 ? BEPU_PI - periodX : periodX;
    bool inSecondHalf = periodX > BEPU_PI;
    y = inSecondHalf ? periodX - BEPU_PI : y;
    y = periodX > 3 * BEPU_PI_OVER_2 ? BEPU_TWO_PI - periodX : y;
    float numerator = ((((0.0040507708755727605f * y - 0.006685815219853882f) * y - 0.13993701695343166f) * y + 0.06174562337697123f) * y + 1.00000000151466040f) * y;
    float denominator = ((((0.00009018370615921334f * y + 0.0001700784176413186f) * y + 0.003606014457152456f) * y + 0.02672943625500751f) * y + 0.061745651499203795f) * y + 1.0f;
    float result = numerator / denominator;
    return inSecondHalf ? -result : result;
}
BEPU_DI float acos_approx(float xin) {  // L353-362
    bool negativeInput = xin < 0.0f;
    float x = fmin_ps(1.0f, fabsf(xin));
    float numerator = sqrtf(1.0f - x) * (62.95741097600742f + x * (69.6550664543659f + x * (17.54512349463405f + x * 0.6022076120669532f)));
    float denominator = 40.07993264439811f + x * (49.81949855726789f + x * (15.703851745284796f + x));
    float result = numerator / denominator;
    return negativeInput ? BEPU_PI - result : result;
}
BEPU_DI float signed_angle_difference(float a, float b) {  // L369-375
    float x = (b - a) * (1.0f / BEPU_TWO_PI) + 0.5f;
    return (x - floorf(x) - 0.5f) * BEPU_TWO_PI;
}

BEPU_DI Q4 quaternion_between_normalized(V3 v1, V3 v2) {  // QuaternionWide.cs:L162-186
    float d = dot(v1, v2);
    V3 c = cross(v1, v2);
    bool useNormalCase = d > -0.999999f;
    float absX = fabsf(v1.x), absY = fabsf(v1.y), absZ = fabsf(v1.z);
    bool xIsSmallest = absX < absY && absX < absZ;
    bool yIsSmaller = absY < absZ;
    Q4 q;
    q.x = useNormalCase ? c.x : (xIsSmallest ? 0.0f : (yIsSmaller ? -v1.z : -v1.y));
    q.y = useNormalCase ? c.y : (xIsSmallest ? -v1.z : (yIsSmaller ? 0.0f : v1.x));
    q.z = useNormalCase ? c.z : (xIsSmallest ? v1.y : (yIsSmaller ? v1.x : 0.0f));
    q.w = useNormalCase ? d + 1.0f : 0.0f;
    return normalize(q);
}
BEPU_DI void axis_angle_from_quaternion(Q4 q, V3& axis, float& angle) {  // QuaternionWide.cs:L227-243
    bool shouldNegate = q.w < 0.0f;
    axis.x = shouldNegate ? -q.x : q.x;
    axis.y = shouldNegate ? -q.y : q.y;
    axis.z = shouldNegate ? -q.z : q.z;
    float qw = shouldNegate ? -q.w : q.w;
    float axisLength = length(axis);
    axis = axis * (1.0f / axisLength);
    bool useFallback = axisLength < 1e-14f;
    axis.x = useFallback ? 1.0f : axis.x;
    axis.y = useFallback ? 0.0f : axis.y;
    axis.z = useFallback ? 0.0f : axis.z;
    angle = 2.0f * acos_approx(qw);
}

// BepuPhysics/Helpers.cs:L21-35
BEPU_DI void build_orthonormal_basis(V3 n, V3& t1, V3& t2) {
    float sign = n.z < 0.0f ? -1.0f : 1.0f;
    float scl = -1.0f / (sign + n.z);
    t1.x = n.x * n.y * scl;
    t1.y = sign + n.y * n.y * scl;
    t1.z = -n.y;
    t2.x = 1.0f + sign * n.x * n.x * scl;
    t2.y = sign * t1.x;
    t2.z = -sign * n.x;
}
BEPU_DI V3 find_perpendicular(V3 n) {  // Helpers.cs:L37-47
    float sign = n.z < 0.0f ? -1.0f : 1.0f;
    float scl = -1.0f / (sign + n.z);
    return {n.x * n.y * scl, sign + n.y * n.y * scl, -n.y};
}

// BepuPhysics/Constraints/SpringSettings.cs:L37-55
struct Springiness { float position_error_to_velocity, effective_mass_cfm_scale, softness_impulse_scale; };
BEPU_DI Springiness compute_springiness(float angular_frequency, float twice_damping_ratio, float dt) {
    float angularFrequencyDt = angular_frequency * dt;
    Springiness s;
    s.position_error_to_velocity = angular_frequency / (angularFrequencyDt + twice_damping_ratio);
    float extra = 1.0f / (angularFrequencyDt * (angularFrequencyDt + twice_damping_ratio));
    s.effective_mass_cfm_scale = 1.0f / (1.0f + extra);
    s.softness_impulse_scale = extra * s.effective_mass_cfm_scale;
    return s;
}

}  // namespace BEPU_NS
