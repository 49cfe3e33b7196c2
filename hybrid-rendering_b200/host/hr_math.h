// hr_math.h — minimal column-major mat4 / vec3 helpers for the host side (glm-compatible conventions).
// Camera follows dw::Camera (external/dwSampleFramework/src/camera.cpp:11-111): glm::perspective with the
// OpenGL clip convention (no GLM_FORCE_DEPTH_ZERO_TO_ONE anywhere in the reference), glm::lookAt right-handed.
#pragma once
#include <cmath>
#include <cstring>

namespace hrm {

struct V3 { float x, y, z; };
inline V3    operator+(V3 a, V3 b) { return { a.x + b.x, a.y + b.y, a.z + b.z }; }
inline V3    operator-(V3 a, V3 b) { return { a.x - b.x, a.y - b.y, a.z - b.z }; }
inline V3    operator*(V3 a, float s) { return { a.x * s, a.y * s, a.z * s }; }
inline float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
inline V3    cross(V3 a, V3 b) { return { a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x }; }
inline float length(V3 a) { return std::sqrt(dot(a, a)); }
inline V3    normalize(V3 a) { float l = length(a); return l > 0 ? a * (1.0f / l) : a; }

struct M4 {
    float m[16]; // m[c*4+r]
    float&       at(int r, int c) { return m[c * 4 + r]; }
    const float& at(int r, int c) const { return m[c * 4 + r]; }
};

inline M4 identity()
{
    M4 r;
    std::memset(r.m, 0, sizeof(r.m));
    r.m[0] = r.m[5] = r.m[10] = r.m[15] = 1.0f;
    return r;
}
inline M4 mul(const M4& a, const M4& b)
{
    M4 r;
    for (int c = 0; c < 4; c++)
        for (int row = 0; row < 4; row++)
        {
            float s = 0;
            for (int k = 0; k < 4; k++) s += a.at(row, k) * b.at(k, c);
            r.at(row, c) = s;
        }
    return r;
}
inline void mul_point(const M4& a, const float v[4], float out[4])
{
    for (int r = 0; r < 4; r++) out[r] = a.at(r, 0) * v[0] + a.at(r, 1) * v[1] + a.at(r, 2) * v[2] + a.at(r, 3) * v[3];
}
// glm::perspective (RH, clip z in [-1,1])
inline M4 perspective(float fovy_rad, float aspect, float zn, float zf)
{
    M4 r;
    std::memset(r.m, 0, sizeof(r.m));
    // tan in double, rounded once to float: the correctly rounded tangent, the value a compile-time fold of tanf gives for a
    // constant field of view, so a field of view passed at run time reproduces the constant's bits (libm's tanf can be 1 ulp off)
    const float t = (float)std::tan((double)(fovy_rad / 2.0f));
    r.at(0, 0)    = 1.0f / (aspect * t);
    r.at(1, 1)    = 1.0f / t;
    r.at(2, 2)    = -(zf + zn) / (zf - zn);
    r.at(3, 2)    = -1.0f;
    r.at(2, 3)    = -(2.0f * zf * zn) / (zf - zn);
    return r;
}
// glm::lookAt (RH)
inline M4 look_at(V3 eye, V3 center, V3 up)
{
    V3 f = normalize(center - eye);
    V3 s = normalize(cross(f, up));
    V3 u = cross(s, f);
    M4 r = identity();
    r.at(0, 0) = s.x; r.at(0, 1) = s.y; r.at(0, 2) = s.z;
    r.at(1, 0) = u.x; r.at(1, 1) = u.y; r.at(1, 2) = u.z;
    r.at(2, 0) = -f.x; r.at(2, 1) = -f.y; r.at(2, 2) = -f.z;
    r.at(0, 3) = -dot(s, eye);
    r.at(1, 3) = -dot(u, eye);
    r.at(2, 3) = dot(f, eye);
    return r;
}
inline M4 translate(V3 t) { M4 r = identity(); r.at(0, 3) = t.x; r.at(1, 3) = t.y; r.at(2, 3) = t.z; return r; }
inline M4 scale(V3 s) { M4 r = identity(); r.at(0, 0) = s.x; r.at(1, 1) = s.y; r.at(2, 2) = s.z; return r; }
inline M4 rotate_axis(float angle, V3 axis)
{
    axis = normalize(axis);
    float c = std::cos(angle), s = std::sin(angle), t = 1 - c;
    M4    r = identity();
    r.at(0, 0) = c + axis.x * axis.x * t;
    r.at(1, 0) = axis.y * axis.x * t + axis.z * s;
    r.at(2, 0) = axis.z * axis.x * t - axis.y * s;
    r.at(0, 1) = axis.x * axis.y * t - axis.z * s;
    r.at(1, 1) = c + axis.y * axis.y * t;
    r.at(2, 1) = axis.z * axis.y * t + axis.x * s;
    r.at(0, 2) = axis.x * axis.z * t + axis.y * s;
    r.at(1, 2) = axis.y * axis.z * t - axis.x * s;
    r.at(2, 2) = c + axis.z * axis.z * t;
    return r;
}
// General 4x4 inverse by cofactors in double, rounded to float (glm::inverse equivalent up to rounding).
inline M4 inverse(const M4& a)
{
    double m[16], inv[16];
    for (int i = 0; i < 16; i++) m[i] = a.m[i];
    inv[0]  = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
    inv[4]  = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
    inv[8]  = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
    inv[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
    inv[1]  = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
    inv[5]  = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
    inv[9]  = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
    inv[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
    inv[2]  = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
    inv[6]  = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
    inv[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
    inv[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
    inv[3]  = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
    inv[7]  = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
    inv[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
    inv[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
    double det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12];
    M4     r;
    double id = det != 0.0 ? 1.0 / det : 0.0;
    for (int i = 0; i < 16; i++) r.m[i] = (float)(inv[i] * id);
    return r;
}

} // namespace hrm
