// llq_math.cuh -- small fixed-size linear algebra for the sm_90a rollout kernels (fp32, registers only).
#pragma once
#include <cuda_runtime.h>

namespace llq {

struct V3 { float x, y, z; };
struct Sym3 { float xx, xy, xz, yy, yz, zz; };          // symmetric 3x3
struct M3 { float a00, a01, a02, a10, a11, a12, a20, a21, a22; };  // general 3x3, row major
struct Q4 { float x, y, z, w; };                         // quaternion, scalar last (scipy / pybullet)

#define LLQ_DI __device__ __forceinline__

LLQ_DI V3 v3(float x, float y, float z) { return V3{x, y, z}; }
LLQ_DI V3 operator+(V3 a, V3 b) { return V3{a.x + b.x, a.y + b.y, a.z + b.z}; }
LLQ_DI V3 operator-(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
LLQ_DI V3 operator*(float s, V3 a) { return V3{s * a.x, s * a.y, s * a.z}; }
LLQ_DI V3 neg(V3 a) { return V3{-a.x, -a.y, -a.z}; }
LLQ_DI float dot(V3 a, V3 b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, a.z * b.z)); }
LLQ_DI V3 cross(V3 a, V3 b) {
  return V3{fmaf(a.y, b.z, -a.z * b.y), fmaf(a.z, b.x, -a.x * b.z), fmaf(a.x, b.y, -a.y * b.x)};
}
LLQ_DI V3 fma3(float s, V3 a, V3 b) { return V3{fmaf(s, a.x, b.x), fmaf(s, a.y, b.y), fmaf(s, a.z, b.z)}; }  // s*a + b
LLQ_DI float norm3(V3 a) { return sqrtf(dot(a, a)); }
LLQ_DI float comp(V3 a, int k) { return k == 0 ? a.x : (k == 1 ? a.y : a.z); }

LLQ_DI V3 mul(Sym3 A, V3 v) {
  return V3{fmaf(A.xx, v.x, fmaf(A.xy, v.y, A.xz * v.z)), fmaf(A.xy, v.x, fmaf(A.yy, v.y, A.yz * v.z)),
            fmaf(A.xz, v.x, fmaf(A.yz, v.y, A.zz * v.z))};
}
LLQ_DI V3 mul(M3 A, V3 v) {
  return V3{fmaf(A.a00, v.x, fmaf(A.a01, v.y, A.a02 * v.z)), fmaf(A.a10, v.x, fmaf(A.a11, v.y, A.a12 * v.z)),
            fmaf(A.a20, v.x, fmaf(A.a21, v.y, A.a22 * v.z))};
}
LLQ_DI V3 tmul(M3 A, V3 v) {  // A^T v
  return V3{fmaf(A.a00, v.x, fmaf(A.a10, v.y, A.a20 * v.z)), fmaf(A.a01, v.x, fmaf(A.a11, v.y, A.a21 * v.z)),
            fmaf(A.a02, v.x, fmaf(A.a12, v.y, A.a22 * v.z))};
}
LLQ_DI V3 row(M3 A, int i) { return i == 0 ? V3{A.a00, A.a01, A.a02} : (i == 1 ? V3{A.a10, A.a11, A.a12} : V3{A.a20, A.a21, A.a22}); }
LLQ_DI V3 col(Sym3 A, int i) { return i == 0 ? V3{A.xx, A.xy, A.xz} : (i == 1 ? V3{A.xy, A.yy, A.yz} : V3{A.xz, A.yz, A.zz}); }
LLQ_DI float diag(Sym3 A, int i) { return i == 0 ? A.xx : (i == 1 ? A.yy : A.zz); }
LLQ_DI Sym3 operator+(Sym3 A, Sym3 B) { return Sym3{A.xx + B.xx, A.xy + B.xy, A.xz + B.xz, A.yy + B.yy, A.yz + B.yz, A.zz + B.zz}; }
LLQ_DI M3 operator+(M3 A, M3 B) {
  return M3{A.a00 + B.a00, A.a01 + B.a01, A.a02 + B.a02, A.a10 + B.a10, A.a11 + B.a11, A.a12 + B.a12, A.a20 + B.a20, A.a21 + B.a21, A.a22 + B.a22};
}
LLQ_DI M3 skew(V3 h) { return M3{0.f, -h.z, h.y, h.z, 0.f, -h.x, -h.y, h.x, 0.f}; }
// A - s * u u^T
LLQ_DI Sym3 sub_outer(Sym3 A, V3 u, float s) {
  return Sym3{fmaf(-s * u.x, u.x, A.xx), fmaf(-s * u.x, u.y, A.xy), fmaf(-s * u.x, u.z, A.xz),
              fmaf(-s * u.y, u.y, A.yy), fmaf(-s * u.y, u.z, A.yz), fmaf(-s * u.z, u.z, A.zz)};
}
// B - s * u v^T
LLQ_DI M3 sub_outer(M3 B, V3 u, V3 v, float s) {
  float ux = -s * u.x, uy = -s * u.y, uz = -s * u.z;
  return M3{fmaf(ux, v.x, B.a00), fmaf(ux, v.y, B.a01), fmaf(ux, v.z, B.a02), fmaf(uy, v.x, B.a10), fmaf(uy, v.y, B.a11),
            fmaf(uy, v.z, B.a12), fmaf(uz, v.x, B.a20), fmaf(uz, v.y, B.a21), fmaf(uz, v.z, B.a22)};
}

// Rotation E = Rot(coordinate axis AX, angle) given (c, s) = (cos, sin) of the angle.  AX: 0 = x, 1 = y.
template <int AX> LLQ_DI V3 rot(V3 v, float c, float s) {   // E v
  if (AX == 0) return V3{v.x, fmaf(c, v.y, -s * v.z), fmaf(s, v.y, c * v.z)};
  return V3{fmaf(c, v.x, s * v.z), v.y, fmaf(-s, v.x, c * v.z)};
}
template <int AX> LLQ_DI V3 rotT(V3 v, float c, float s) {  // E^T v
  return rot<AX>(v, c, -s);
}
template <int AX> LLQ_DI Sym3 rot_sym(Sym3 A, float c, float s) {  // E A E^T
  float cc = c * c, ss = s * s, cs = c * s;
  if (AX == 0) {
    return Sym3{A.xx, fmaf(c, A.xy, -s * A.xz), fmaf(s, A.xy, c * A.xz),
                fmaf(cc, A.yy, fmaf(-2.f * cs, A.yz, ss * A.zz)), fmaf(cs, A.yy - A.zz, (cc - ss) * A.yz),
                fmaf(ss, A.yy, fmaf(2.f * cs, A.yz, cc * A.zz))};
  }
  return Sym3{fmaf(cc, A.xx, fmaf(2.f * cs, A.xz, ss * A.zz)), fmaf(c, A.xy, s * A.yz), fmaf(cs, A.zz - A.xx, (cc - ss) * A.xz),
              A.yy, fmaf(-s, A.xy, c * A.yz), fmaf(ss, A.xx, fmaf(-2.f * cs, A.xz, cc * A.zz))};
}
template <int AX> LLQ_DI M3 rot_mat(M3 B, float c, float s) {  // E B E^T
  // rows first (T = E B), then columns (T E^T)
  V3 r0 = row(B, 0), r1 = row(B, 1), r2 = row(B, 2), t0, t1, t2;
  if (AX == 0) { t0 = r0; t1 = fma3(c, r1, (-s) * r2); t2 = fma3(s, r1, c * r2); }
  else { t0 = fma3(c, r0, s * r2); t1 = r1; t2 = fma3(-s, r0, c * r2); }
  // each row vector x becomes E x  (since (T E^T)_row = E * row)
  V3 q0 = rot<AX>(t0, c, s), q1 = rot<AX>(t1, c, s), q2 = rot<AX>(t2, c, s);
  return M3{q0.x, q0.y, q0.z, q1.x, q1.y, q1.z, q2.x, q2.y, q2.z};
}

// quaternions
LLQ_DI Q4 qmul(Q4 a, Q4 b) {
  return Q4{a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x,
            a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
LLQ_DI Q4 qconj(Q4 q) { return Q4{-q.x, -q.y, -q.z, q.w}; }
LLQ_DI Q4 qnormalize(Q4 q) {
  float n = 1.0f / sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  return Q4{q.x * n, q.y * n, q.z * n, q.w * n};
}
LLQ_DI M3 qmat(Q4 q) {  // world <- body for a unit quaternion
  float x = q.x, y = q.y, z = q.z, w = q.w;
  return M3{1.f - 2.f * (y * y + z * z), 2.f * (x * y - z * w), 2.f * (x * z + y * w),
            2.f * (x * y + z * w), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - x * w),
            2.f * (x * z - y * w), 2.f * (y * z + x * w), 1.f - 2.f * (x * x + y * y)};
}
// sin / cos for |x| < 1e5 rad (joint angles, yaw, half rotation angles: all far below): three-term Cody-Waite reduction by pi/2
// and the degree-7 / degree-8 minimax kernels on [-pi/4, pi/4] -- max error 1.5 ulp (7e-8 absolute), checked against float64 over
// [-100, 100] (DESIGN.md 4.1).  Same accuracy class as sincosf(), but without its Payne-Hanek slow path: that branch (never taken
// here) cost ~120 SASS instructions per call site, 22 % of the step kernel's code and 23 % of its time through the instruction cache.
LLQ_DI void llq_sincosf(float x, float* sn, float* cs) {
  const float j = rintf(x * 0.636619747f);
  float a = fmaf(j, -1.5707962512969971f, x);
  a = fmaf(j, -7.5497894158615964e-8f, a);
  a = fmaf(j, -5.3903029534742384e-15f, a);
  const float s = a * a;
  float t = fmaf(-1.95152959e-4f, s, 8.33216087e-3f);
  t = fmaf(t, s, -1.66666546e-1f);
  const float sa = fmaf(t * s, a, a);
  float u = fmaf(2.44331571e-5f, s, -1.38873163e-3f);
  u = fmaf(u, s, 4.16666457e-2f);
  u = fmaf(u, s, -0.5f);
  const float ca = fmaf(u, s, 1.0f);
  const int q = (int)j;
  const float S = (q & 1) ? ca : sa, C = (q & 1) ? sa : ca;
  *sn = (q & 2) ? -S : S;
  *cs = ((q + 1) & 2) ? -C : C;
}
LLQ_DI float llq_sinf(float x) { float s, c; llq_sincosf(x, &s, &c); return s; }
LLQ_DI float llq_cosf(float x) { float s, c; llq_sincosf(x, &s, &c); return c; }

// scipy Rotation.as_rotvec (angle in [0, pi])
LLQ_DI V3 q_rotvec(Q4 q) {
  if (q.w < 0.f) q = Q4{-q.x, -q.y, -q.z, -q.w};
  float s = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z);
  float angle = 2.f * atan2f(s, q.w);
  float scale;
  if (angle <= 1e-3f) {
    float a2 = angle * angle;
    scale = 2.f + a2 * (1.f / 12.f) + 7.f * a2 * a2 * (1.f / 2880.f);
  } else {
    scale = angle / llq_sinf(0.5f * angle);
  }
  return V3{scale * q.x, scale * q.y, scale * q.z};
}
// scipy Rotation.from_rotvec
LLQ_DI Q4 rotvec_q(V3 r) {
  float angle = norm3(r), scale, sn, cs;
  llq_sincosf(0.5f * angle, &sn, &cs);
  if (angle <= 1e-3f) {
    float a2 = angle * angle;
    scale = 0.5f - a2 * (1.f / 48.f) + a2 * a2 * (1.f / 3840.f);
  } else {
    scale = sn / angle;
  }
  return Q4{scale * r.x, scale * r.y, scale * r.z, cs};
}

// 6x6 symmetric positive definite: packed lower Cholesky factor L (row-major lower triangle, 21 entries).
// LLQ_CHOL_T selects the arithmetic of the factorisation and of the triangular solves (float by default; the H100 runs
// fp64 FMA at half the fp32 rate, so -DLLQ_CHOL_T=double is affordable for these ~250 flops per sub-step).
#ifndef LLQ_CHOL_T
#define LLQ_CHOL_T float
#endif
typedef LLQ_CHOL_T chol_t;
struct Chol6 { chol_t l[21]; };
LLQ_DI constexpr int tri(int i, int j) { return i * (i + 1) / 2 + j; }  // i >= j
LLQ_DI chol_t cfma(chol_t a, chol_t b, chol_t c) { return sizeof(chol_t) == 8 ? (chol_t)fma((double)a, (double)b, (double)c) : (chol_t)fmaf((float)a, (float)b, (float)c); }
// m: packed lower triangle of the symmetric matrix (same indexing)
LLQ_DI Chol6 chol6(const float (&m)[21]) {
  Chol6 c;
#pragma unroll
  for (int i = 0; i < 6; i++) {
#pragma unroll
    for (int j = 0; j <= i; j++) {
      chol_t s = (chol_t)m[tri(i, j)];
#pragma unroll
      for (int k = 0; k < j; k++) s = cfma(-c.l[tri(i, k)], c.l[tri(j, k)], s);
      if (i == j) c.l[tri(i, i)] = sizeof(chol_t) == 8 ? (chol_t)rsqrt((double)s) : (chol_t)(1.0f / sqrtf((float)s));   // reciprocal of the diagonal
      else c.l[tri(i, j)] = s * c.l[tri(j, j)];
    }
  }
  return c;
}
// forward substitution: y = L^-1 b
LLQ_DI void chol6_fwd(const Chol6& c, const float (&b)[6], float (&y)[6]) {
  chol_t t[6];
#pragma unroll
  for (int i = 0; i < 6; i++) {
    chol_t s = (chol_t)b[i];
#pragma unroll
    for (int k = 0; k < i; k++) s = cfma(-c.l[tri(i, k)], t[k], s);
    t[i] = s * c.l[tri(i, i)];
    y[i] = (float)t[i];
  }
}
// backward substitution: x = L^-T y
LLQ_DI void chol6_bwd(const Chol6& c, const float (&y)[6], float (&x)[6]) {
  chol_t t[6];
#pragma unroll
  for (int i = 5; i >= 0; i--) {
    chol_t s = (chol_t)y[i];
#pragma unroll
    for (int k = i + 1; k < 6; k++) s = cfma(-c.l[tri(k, i)], t[k], s);
    t[i] = s * c.l[tri(i, i)];
    x[i] = (float)t[i];
  }
}
// solve (L L^T) x = b
LLQ_DI void chol6_solve(const Chol6& c, const float (&b)[6], float (&x)[6]) {
  chol_t t[6], u[6];
#pragma unroll
  for (int i = 0; i < 6; i++) {
    chol_t s = (chol_t)b[i];
#pragma unroll
    for (int k = 0; k < i; k++) s = cfma(-c.l[tri(i, k)], t[k], s);
    t[i] = s * c.l[tri(i, i)];
  }
#pragma unroll
  for (int i = 5; i >= 0; i--) {
    chol_t s = t[i];
#pragma unroll
    for (int k = i + 1; k < 6; k++) s = cfma(-c.l[tri(k, i)], u[k], s);
    u[i] = s * c.l[tri(i, i)];
    x[i] = (float)u[i];
  }
}

}  // namespace llq
