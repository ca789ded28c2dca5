// Device float math for the step / raster kernels (sm_90a).  Compiled with -fmad=false: every +,-,*,/ and sqrt is a
// single IEEE-754 round-to-nearest operation in the order written, so results are reproducible against a CPU that also
// keeps contraction off.  Accumulation orders follow the reference's libraries:
//   4x4 product / inverse / rotation : Magnum (Math/RectangularMatrix.h:753-764, Math/Matrix.h:379-421,491-522,
//                                      Math/Matrix4.h:959-999)
//   3x3 product, quaternion <-> matrix, axis/angle : Bullet btMatrix3x3 / btQuaternion (upstream 2.89; not vendored)
// Transcendentals: evaluated in double and rounded once to float (DESIGN.md "numerics").
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dm {

struct V3 { float x, y, z; };
__device__ __forceinline__ V3 v3(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ V3 operator+(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ V3 operator-(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ V3 operator-(V3 a) { return v3(-a.x, -a.y, -a.z); }
__device__ __forceinline__ V3 operator*(V3 a, float s) { return v3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float length2(V3 a) { return dot(a, a); }
__device__ __forceinline__ float length(V3 a) { return sqrtf(dot(a, a)); }
__device__ __forceinline__ V3 btNormalized(V3 a) { const float l = length(a); return a * (1.0f / l); }
__device__ __forceinline__ V3 mgNormalized(V3 a) { const float l = 1.0f / sqrtf(dot(a, a)); return a * l; }
__device__ __forceinline__ float comp(V3 a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }
__device__ __forceinline__ void setComp(V3 &a, int i, float v) { if (i == 0) a.x = v; else if (i == 1) a.y = v; else a.z = v; }

__device__ __forceinline__ float crsin(float x) { return float(sin(double(x))); }
__device__ __forceinline__ float crcos(float x) { return float(cos(double(x))); }
__device__ __forceinline__ float cracos(float x) { return float(acos(double(x))); }

struct M3 { float r[9]; };  // rows
__device__ __forceinline__ M3 mul3(const M3 &a, const M3 &b) {
    M3 o;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        o.r[i * 3 + 0] = a.r[i * 3] * b.r[0] + a.r[i * 3 + 1] * b.r[3] + a.r[i * 3 + 2] * b.r[6];
        o.r[i * 3 + 1] = a.r[i * 3] * b.r[1] + a.r[i * 3 + 1] * b.r[4] + a.r[i * 3 + 2] * b.r[7];
        o.r[i * 3 + 2] = a.r[i * 3] * b.r[2] + a.r[i * 3 + 1] * b.r[5] + a.r[i * 3 + 2] * b.r[8];
    }
    return o;
}

struct M4 { float c[16]; };  // column-major, c[col*4+row]
__device__ __forceinline__ M4 identity4() {
    M4 m;
#pragma unroll
    for (int i = 0; i < 16; ++i) m.c[i] = (i % 5 == 0) ? 1.0f : 0.0f;
    return m;
}
__device__ __forceinline__ M4 mul4(const M4 &a, const M4 &b) {
    M4 o;
#pragma unroll
    for (int col = 0; col < 4; ++col)
#pragma unroll
        for (int row = 0; row < 4; ++row) {
            float acc = 0.0f;
#pragma unroll
            for (int pos = 0; pos < 4; ++pos) acc += a.c[pos * 4 + row] * b.c[col * 4 + pos];
            o.c[col * 4 + row] = acc;
        }
    return o;
}
__device__ __forceinline__ M4 translation4(V3 t) { M4 m = identity4(); m.c[12] = t.x; m.c[13] = t.y; m.c[14] = t.z; return m; }
__device__ __forceinline__ M4 scaling4(V3 s) { M4 m = identity4(); m.c[0] = s.x; m.c[5] = s.y; m.c[10] = s.z; return m; }
__device__ __forceinline__ M4 rotationX4(float a) {
    const float s = crsin(a), c = crcos(a);
    M4 m = identity4();
    m.c[5] = c; m.c[6] = s; m.c[9] = -s; m.c[10] = c;
    return m;
}
__device__ __forceinline__ M4 rotation4(float angle, V3 ax) {
    const float sine = crsin(angle), cosine = crcos(angle), omc = 1.0f - cosine;
    const float xx = ax.x * ax.x, xy = ax.x * ax.y, xz = ax.x * ax.z, yy = ax.y * ax.y, yz = ax.y * ax.z, zz = ax.z * ax.z;
    M4 m = identity4();
    m.c[0] = cosine + xx * omc; m.c[1] = xy * omc + ax.z * sine; m.c[2] = xz * omc - ax.y * sine;
    m.c[4] = xy * omc - ax.z * sine; m.c[5] = cosine + yy * omc; m.c[6] = yz * omc + ax.x * sine;
    m.c[8] = xz * omc + ax.y * sine; m.c[9] = yz * omc - ax.x * sine; m.c[10] = cosine + zz * omc;
    return m;
}
__device__ __forceinline__ V3 translationOf(const M4 &m) { return v3(m.c[12], m.c[13], m.c[14]); }
__device__ __forceinline__ V3 scalingOf(const M4 &m) {
    return v3(sqrtf(m.c[0] * m.c[0] + m.c[1] * m.c[1] + m.c[2] * m.c[2]), sqrtf(m.c[4] * m.c[4] + m.c[5] * m.c[5] + m.c[6] * m.c[6]),
              sqrtf(m.c[8] * m.c[8] + m.c[9] * m.c[9] + m.c[10] * m.c[10]));
}
__device__ __forceinline__ V3 transformPoint(const M4 &m, V3 p) {
    V3 o;
    { float acc = 0.0f; acc += m.c[0] * p.x; acc += m.c[4] * p.y; acc += m.c[8] * p.z; acc += m.c[12] * 1.0f; o.x = acc; }
    { float acc = 0.0f; acc += m.c[1] * p.x; acc += m.c[5] * p.y; acc += m.c[9] * p.z; acc += m.c[13] * 1.0f; o.y = acc; }
    { float acc = 0.0f; acc += m.c[2] * p.x; acc += m.c[6] * p.y; acc += m.c[10] * p.z; acc += m.c[14] * 1.0f; o.z = acc; }
    return o;
}
__device__ __forceinline__ float det3skip(const M4 &m, int skipCol, int skipRow) {
#define MV_E(ci, ri) m.c[((ci) + ((ci) >= skipCol)) * 4 + ((ri) + ((ri) >= skipRow))]
    return MV_E(0, 0) * ((MV_E(1, 1) * MV_E(2, 2)) - (MV_E(2, 1) * MV_E(1, 2))) - MV_E(0, 1) * (MV_E(1, 0) * MV_E(2, 2) - MV_E(2, 0) * MV_E(1, 2)) +
           MV_E(0, 2) * (MV_E(1, 0) * MV_E(2, 1) - MV_E(2, 0) * MV_E(1, 1));
#undef MV_E
}
__device__ __forceinline__ float cofactor4(const M4 &m, int col, int row) { return (((row + col) & 1) ? -1 : 1) * det3skip(m, col, row); }
__device__ __forceinline__ M4 inverted4(const M4 &m) {
    float d = 0.0f;
#pragma unroll
    for (int col = 0; col < 4; ++col) d += m.c[col * 4] * cofactor4(m, col, 0);
    M4 o;
#pragma unroll
    for (int col = 0; col < 4; ++col)
#pragma unroll
        for (int row = 0; row < 4; ++row) o.c[col * 4 + row] = cofactor4(m, row, col) / d;
    return o;
}
// inverse-transpose of the upper 3x3 (cofactor matrix / determinant); n[col*3+row]
__device__ __forceinline__ float normalMatrix(const M4 &mv, float n[9]) {  // returns the determinant of the 3x3
    const float a00 = mv.c[0], a01 = mv.c[1], a02 = mv.c[2];
    const float a10 = mv.c[4], a11 = mv.c[5], a12 = mv.c[6];
    const float a20 = mv.c[8], a21 = mv.c[9], a22 = mv.c[10];
    const float c00 = a11 * a22 - a21 * a12, c01 = a20 * a12 - a10 * a22, c02 = a10 * a21 - a20 * a11;
    const float c10 = a21 * a02 - a01 * a22, c11 = a00 * a22 - a20 * a02, c12 = a20 * a01 - a00 * a21;
    const float c20 = a01 * a12 - a11 * a02, c21 = a10 * a02 - a00 * a12, c22 = a00 * a11 - a10 * a01;
    const float det = a00 * c00 + a01 * c01 + a02 * c02;
    const float id = 1.0f / det;
    n[0] = c00 * id; n[1] = c01 * id; n[2] = c02 * id;
    n[3] = c10 * id; n[4] = c11 * id; n[5] = c12 * id;
    n[6] = c20 * id; n[7] = c21 * id; n[8] = c22 * id;
    return det;
}

}  // namespace dm
