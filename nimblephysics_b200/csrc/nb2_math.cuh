// Small spatial-algebra toolkit for the per-world kernels.  Everything is scalar code meant to live in
// registers (no dynamically indexed local arrays).  Conventions follow the reference: spatial vectors are
// [angular; linear] in the body frame (dart/math/Geometry.cpp:1300-1312); a transform Xf{R,p} maps child
// coordinates to parent coordinates, x_parent = R x_child + p.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define NB2_HD __host__ __device__ __forceinline__
#else
#define NB2_HD inline
#endif

namespace nb2 {

template <class R> struct V3 { R x, y, z; };
template <class R> struct V6 { V3<R> a, l; };          // angular, linear
template <class R> struct M3 { R m00, m01, m02, m10, m11, m12, m20, m21, m22; };
template <class R> struct S3 { R xx, yy, zz, xy, xz, yz; };  // symmetric 3x3
template <class R> struct Xf { M3<R> R_; V3<R> p; };
// symmetric 6x6 in blocks [[A, B], [B^T, C]] (A rotational, C translational)
template <class R> struct SI { S3<R> A; M3<R> B; S3<R> C; };

NB2_HD void nb2_sincos(float x, float* s, float* c) {
#ifdef __CUDA_ARCH__
  // the library is built with --use_fast_math (fp32 division / sqrt / sincos are the special-function unit's): the hardware
  // sine is accurate to ~5e-7 absolute on [-pi, pi] only, so the argument is reduced first (two-term 2 pi, exact to ~1e-7
  // relative for |x| up to ~1e4 rad — an unbounded revolute joint may have wound up many turns)
  const float k = rintf(x * 0.15915494309189535f);
  float r = fmaf(-k, 6.2831854820251465f, x);   // 2 pi rounded to fp32
  r = fmaf(-k, -1.7484555e-07f, r);             // 2 pi - fp32(2 pi)
  __sincosf(r, s, c);
#else
  sincosf(x, s, c);
#endif
}
NB2_HD void nb2_sincos(double x, double* s, double* c) { sincos(x, s, c); }
NB2_HD float nb2_sqrt(float x) { return sqrtf(x); }
// fp64 division / square root are ~40-instruction dependent sequences on the GPU (scripts/dev/ubench/lat.cu measures their latency
// against a multiply-add).  The hot paths use a seed from the special-function unit refined by two Newton steps (~1 ulp);
// arguments outside the comfortable exponent range take the IEEE routine.
NB2_HD double nb2_rcp(double b) {
#ifdef __CUDA_ARCH__
  const unsigned ex = ((unsigned)__double2hiint(b) >> 20) & 0x7ffu;
  if (ex > 0x020u && ex < 0x7d0u) {
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(b));
    double e = fma(-b, r, 1.0); r = fma(r, e, r);
    e = fma(-b, r, 1.0); r = fma(r, e, r);
    return r;
  }
#endif
  return 1.0 / b;
}
NB2_HD float nb2_rcp(float b) { return 1.0f / b; }
NB2_HD double nb2_div(double a, double b) {
#ifdef __CUDA_ARCH__
  const unsigned ex = ((unsigned)__double2hiint(b) >> 20) & 0x7ffu, ea = ((unsigned)__double2hiint(a) >> 20) & 0x7ffu;
  if (ex > 0x020u && ex < 0x7d0u && ea > 0x040u && ea < 0x7b0u) {
    const double r = nb2_rcp(b);
    const double q = a * r;
    return fma(fma(-b, q, a), r, q);
  }
#endif
  return a / b;
}
NB2_HD float nb2_div(float a, float b) { return a / b; }
// 1 / sqrt(x) for x in the comfortable range, else via the IEEE routines
NB2_HD double nb2_rsqrt(double x) {
#ifdef __CUDA_ARCH__
  const int hi = __double2hiint(x);
  const unsigned ex = ((unsigned)hi >> 20) & 0x7ffu;
  if (hi > 0 && ex > 0x020u && ex < 0x7d0u) {
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
    double e = fma(-x * y, y, 1.0); y = fma(0.5 * y, e, y);
    e = fma(-x * y, y, 1.0); y = fma(0.5 * y, e, y);
    return y;
  }
#endif
  return 1.0 / sqrt(x);
}
NB2_HD double nb2_sqrt(double x) {
#ifdef __CUDA_ARCH__
  const int hi = __double2hiint(x);
  const unsigned ex = ((unsigned)hi >> 20) & 0x7ffu;
  if (hi > 0 && ex > 0x020u && ex < 0x7d0u) {
    const double y = nb2_rsqrt(x);
    const double s = x * y;
    return fma(fma(-s, s, x), 0.5 * y, s);
  }
#endif
  return sqrt(x);
}
NB2_HD float nb2_atan2(float y, float x) { return atan2f(y, x); }
NB2_HD double nb2_atan2(double y, double x) { return atan2(y, x); }
NB2_HD float nb2_abs(float x) { return fabsf(x); }
NB2_HD double nb2_abs(double x) { return fabs(x); }

template <class R> NB2_HD V3<R> mk3(R x, R y, R z) { V3<R> v; v.x = x; v.y = y; v.z = z; return v; }
template <class R> NB2_HD V3<R> zero3() { return mk3<R>(R(0), R(0), R(0)); }
template <class R> NB2_HD V6<R> zero6() { V6<R> v; v.a = zero3<R>(); v.l = zero3<R>(); return v; }
template <class R> NB2_HD V3<R> operator+(const V3<R>& a, const V3<R>& b) { return mk3<R>(a.x + b.x, a.y + b.y, a.z + b.z); }
template <class R> NB2_HD V3<R> operator-(const V3<R>& a, const V3<R>& b) { return mk3<R>(a.x - b.x, a.y - b.y, a.z - b.z); }
template <class R> NB2_HD V3<R> operator-(const V3<R>& a) { return mk3<R>(-a.x, -a.y, -a.z); }
template <class R> NB2_HD V3<R> operator*(const V3<R>& a, R s) { return mk3<R>(a.x * s, a.y * s, a.z * s); }
template <class R> NB2_HD R dot(const V3<R>& a, const V3<R>& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <class R> NB2_HD V3<R> cross(const V3<R>& a, const V3<R>& b) { return mk3<R>(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
template <class R> NB2_HD V6<R> operator+(const V6<R>& a, const V6<R>& b) { V6<R> r; r.a = a.a + b.a; r.l = a.l + b.l; return r; }
template <class R> NB2_HD V6<R> operator-(const V6<R>& a, const V6<R>& b) { V6<R> r; r.a = a.a - b.a; r.l = a.l - b.l; return r; }
template <class R> NB2_HD V6<R> operator*(const V6<R>& a, R s) { V6<R> r; r.a = a.a * s; r.l = a.l * s; return r; }
template <class R> NB2_HD R dot(const V6<R>& a, const V6<R>& b) { return dot(a.a, b.a) + dot(a.l, b.l); }

template <class R> NB2_HD V3<R> mul(const M3<R>& M, const V3<R>& v) {
  return mk3<R>(M.m00 * v.x + M.m01 * v.y + M.m02 * v.z, M.m10 * v.x + M.m11 * v.y + M.m12 * v.z, M.m20 * v.x + M.m21 * v.y + M.m22 * v.z);
}
template <class R> NB2_HD V3<R> mulT(const M3<R>& M, const V3<R>& v) {
  return mk3<R>(M.m00 * v.x + M.m10 * v.y + M.m20 * v.z, M.m01 * v.x + M.m11 * v.y + M.m21 * v.z, M.m02 * v.x + M.m12 * v.y + M.m22 * v.z);
}
template <class R> NB2_HD M3<R> mul(const M3<R>& A, const M3<R>& B) {
  M3<R> C;
  C.m00 = A.m00 * B.m00 + A.m01 * B.m10 + A.m02 * B.m20; C.m01 = A.m00 * B.m01 + A.m01 * B.m11 + A.m02 * B.m21; C.m02 = A.m00 * B.m02 + A.m01 * B.m12 + A.m02 * B.m22;
  C.m10 = A.m10 * B.m00 + A.m11 * B.m10 + A.m12 * B.m20; C.m11 = A.m10 * B.m01 + A.m11 * B.m11 + A.m12 * B.m21; C.m12 = A.m10 * B.m02 + A.m11 * B.m12 + A.m12 * B.m22;
  C.m20 = A.m20 * B.m00 + A.m21 * B.m10 + A.m22 * B.m20; C.m21 = A.m20 * B.m01 + A.m21 * B.m11 + A.m22 * B.m21; C.m22 = A.m20 * B.m02 + A.m21 * B.m12 + A.m22 * B.m22;
  return C;
}
template <class R> NB2_HD M3<R> mulABt(const M3<R>& A, const M3<R>& B) {  // A * B^T
  M3<R> C;
  C.m00 = A.m00 * B.m00 + A.m01 * B.m01 + A.m02 * B.m02; C.m01 = A.m00 * B.m10 + A.m01 * B.m11 + A.m02 * B.m12; C.m02 = A.m00 * B.m20 + A.m01 * B.m21 + A.m02 * B.m22;
  C.m10 = A.m10 * B.m00 + A.m11 * B.m01 + A.m12 * B.m02; C.m11 = A.m10 * B.m10 + A.m11 * B.m11 + A.m12 * B.m12; C.m12 = A.m10 * B.m20 + A.m11 * B.m21 + A.m12 * B.m22;
  C.m20 = A.m20 * B.m00 + A.m21 * B.m01 + A.m22 * B.m02; C.m21 = A.m20 * B.m10 + A.m21 * B.m11 + A.m22 * B.m12; C.m22 = A.m20 * B.m20 + A.m21 * B.m21 + A.m22 * B.m22;
  return C;
}
template <class R> NB2_HD M3<R> transpose(const M3<R>& A) { M3<R> C; C.m00 = A.m00; C.m01 = A.m10; C.m02 = A.m20; C.m10 = A.m01; C.m11 = A.m11; C.m12 = A.m21; C.m20 = A.m02; C.m21 = A.m12; C.m22 = A.m22; return C; }
template <class R> NB2_HD M3<R> eye3() { M3<R> C; C.m00 = C.m11 = C.m22 = R(1); C.m01 = C.m02 = C.m10 = C.m12 = C.m20 = C.m21 = R(0); return C; }
template <class R> NB2_HD M3<R> full(const S3<R>& S) { M3<R> C; C.m00 = S.xx; C.m11 = S.yy; C.m22 = S.zz; C.m01 = C.m10 = S.xy; C.m02 = C.m20 = S.xz; C.m12 = C.m21 = S.yz; return C; }
template <class R> NB2_HD V3<R> mul(const S3<R>& S, const V3<R>& v) {
  return mk3<R>(S.xx * v.x + S.xy * v.y + S.xz * v.z, S.xy * v.x + S.yy * v.y + S.yz * v.z, S.xz * v.x + S.yz * v.y + S.zz * v.z);
}
// R S R^T for symmetric S
template <class R> NB2_HD S3<R> rot_sym(const M3<R>& Rm, const S3<R>& S) {
  M3<R> T = mul(Rm, full(S));  // T = R S
  S3<R> o;
  o.xx = T.m00 * Rm.m00 + T.m01 * Rm.m01 + T.m02 * Rm.m02;
  o.yy = T.m10 * Rm.m10 + T.m11 * Rm.m11 + T.m12 * Rm.m12;
  o.zz = T.m20 * Rm.m20 + T.m21 * Rm.m21 + T.m22 * Rm.m22;
  o.xy = T.m00 * Rm.m10 + T.m01 * Rm.m11 + T.m02 * Rm.m12;
  o.xz = T.m00 * Rm.m20 + T.m01 * Rm.m21 + T.m02 * Rm.m22;
  o.yz = T.m10 * Rm.m20 + T.m11 * Rm.m21 + T.m12 * Rm.m22;
  return o;
}
template <class R> NB2_HD S3<R> operator+(const S3<R>& a, const S3<R>& b) { S3<R> o; o.xx = a.xx + b.xx; o.yy = a.yy + b.yy; o.zz = a.zz + b.zz; o.xy = a.xy + b.xy; o.xz = a.xz + b.xz; o.yz = a.yz + b.yz; return o; }
template <class R> NB2_HD M3<R> operator+(const M3<R>& a, const M3<R>& b) { M3<R> o; o.m00 = a.m00 + b.m00; o.m01 = a.m01 + b.m01; o.m02 = a.m02 + b.m02; o.m10 = a.m10 + b.m10; o.m11 = a.m11 + b.m11; o.m12 = a.m12 + b.m12; o.m20 = a.m20 + b.m20; o.m21 = a.m21 + b.m21; o.m22 = a.m22 + b.m22; return o; }
template <class R> NB2_HD SI<R> operator+(const SI<R>& a, const SI<R>& b) { SI<R> o; o.A = a.A + b.A; o.B = a.B + b.B; o.C = a.C + b.C; return o; }
template <class R> NB2_HD SI<R> zeroSI() {
  SI<R> o; o.A.xx = o.A.yy = o.A.zz = o.A.xy = o.A.xz = o.A.yz = R(0); o.C = o.A;
  o.B.m00 = o.B.m01 = o.B.m02 = o.B.m10 = o.B.m11 = o.B.m12 = o.B.m20 = o.B.m21 = o.B.m22 = R(0); return o;
}

// ---- SE(3) actions (dart/math/Geometry.cpp:1437-1445, 1529-1537)
template <class R> NB2_HD V6<R> AdInvT(const Xf<R>& T, const V6<R>& V) {  // motion: parent frame -> child frame
  V6<R> r; r.a = mulT(T.R_, V.a); r.l = mulT(T.R_, V.l + cross(V.a, T.p)); return r;
}
template <class R> NB2_HD V6<R> dAdInvT(const Xf<R>& T, const V6<R>& F) {  // force: child frame -> parent frame
  V6<R> r; r.l = mul(T.R_, F.l); r.a = mul(T.R_, F.a) + cross(T.p, r.l); return r;
}
template <class R> NB2_HD V6<R> ad(const V6<R>& X, const V6<R>& Y) {  // motion cross motion (:1470-1483)
  V6<R> r; r.a = cross(X.a, Y.a); r.l = cross(X.a, Y.l) + cross(X.l, Y.a); return r;
}
template <class R> NB2_HD V6<R> crf(const V6<R>& V, const V6<R>& F) {  // V x* F  ( = -dad(V,F), :3506-3513 )
  V6<R> r; r.a = cross(V.a, F.a) + cross(V.l, F.l); r.l = cross(V.a, F.l); return r;
}
// SI * motion -> force
template <class R> NB2_HD V6<R> mul(const SI<R>& I, const V6<R>& V) {
  V6<R> r; r.a = mul(I.A, V.a) + mul(I.B, V.l); r.l = mulT(I.B, V.a) + mul(I.C, V.l); return r;
}
// rigid-body inertia {m, h = m c, Ibar} times motion
template <class R> NB2_HD V6<R> mulG(R m, const V3<R>& h, const S3<R>& Ib, const V6<R>& V) {
  V6<R> r; r.a = mul(Ib, V.a) + cross(h, V.l); r.l = V.l * m + cross(V.a, h); return r;
}
template <class R> NB2_HD SI<R> rigidSI(R m, const V3<R>& h, const S3<R>& Ib) {
  SI<R> o; o.A = Ib;
  o.B.m00 = R(0); o.B.m01 = -h.z; o.B.m02 = h.y; o.B.m10 = h.z; o.B.m11 = R(0); o.B.m12 = -h.x; o.B.m20 = -h.y; o.B.m21 = h.x; o.B.m22 = R(0);
  o.C.xx = o.C.yy = o.C.zz = m; o.C.xy = o.C.xz = o.C.yz = R(0);
  return o;
}
// articulated inertia expressed in the child frame -> parent frame:  X* I X*^T with X* = [[R, [p]x R],[0, R]]
// (same value as math::transformInertia(T^-1, I), dart/math/Geometry.cpp:3515-3597)
template <class R> NB2_HD SI<R> xform_inertia(const Xf<R>& T, const SI<R>& I) {
  SI<R> o;
  S3<R> A1 = rot_sym(T.R_, I.A);
  S3<R> C1 = rot_sym(T.R_, I.C);
  M3<R> B1 = mulABt(mul(T.R_, I.B), T.R_);
  // P = [p]x ;  PC = P C1 ;  top-right = B1 + PC ; top-left = A1 + P B1^T + B1 P^T + P C1 P^T = A1 + P(B1 + PC)^T ... expanded
  const V3<R> p = T.p;
  M3<R> C1f = full(C1);
  // rows of P*C1: row i = p x (column... ) -> (P*M) column j = p x M[:,j]
  V3<R> c0 = cross(p, mk3<R>(C1f.m00, C1f.m10, C1f.m20));
  V3<R> c1 = cross(p, mk3<R>(C1f.m01, C1f.m11, C1f.m21));
  V3<R> c2 = cross(p, mk3<R>(C1f.m02, C1f.m12, C1f.m22));
  M3<R> Bn;  // B1 + P C1
  Bn.m00 = B1.m00 + c0.x; Bn.m10 = B1.m10 + c0.y; Bn.m20 = B1.m20 + c0.z;
  Bn.m01 = B1.m01 + c1.x; Bn.m11 = B1.m11 + c1.y; Bn.m21 = B1.m21 + c1.z;
  Bn.m02 = B1.m02 + c2.x; Bn.m12 = B1.m12 + c2.y; Bn.m22 = B1.m22 + c2.z;
  // A' = A1 + P B1^T + Bn P^T.   (P X)[:,j] = p x X[:,j] ;  (Bn P^T) = (P Bn^T)^T
  // P B1^T : column j of B1^T is row j of B1
  V3<R> d0 = cross(p, mk3<R>(B1.m00, B1.m01, B1.m02));
  V3<R> d1 = cross(p, mk3<R>(B1.m10, B1.m11, B1.m12));
  V3<R> d2 = cross(p, mk3<R>(B1.m20, B1.m21, B1.m22));
  // P Bn^T : column j = p x (row j of Bn)
  V3<R> e0 = cross(p, mk3<R>(Bn.m00, Bn.m01, Bn.m02));
  V3<R> e1 = cross(p, mk3<R>(Bn.m10, Bn.m11, Bn.m12));
  V3<R> e2 = cross(p, mk3<R>(Bn.m20, Bn.m21, Bn.m22));
  // (P B1^T)(i,j) = d_j[i] ; (Bn P^T)(i,j) = (P Bn^T)(j,i) = e_i[j]
  o.A.xx = A1.xx + d0.x + e0.x;
  o.A.yy = A1.yy + d1.y + e1.y;
  o.A.zz = A1.zz + d2.z + e2.z;
  o.A.xy = A1.xy + d1.x + e0.y;
  o.A.xz = A1.xz + d2.x + e0.z;
  o.A.yz = A1.yz + d2.y + e1.z;
  o.B = Bn;
  o.C = C1;
  return o;
}

// ---- SO(3) helpers.  Reference: expMapRot Geometry.cpp:539-554, logMap :720-760.
// (1-cos t)/t^2 is evaluated as 0.5 (sin(t/2)/(t/2))^2 and theta by atan2 so the fp32 path keeps full accuracy.
template <class R> NB2_HD void so3_coeffs(R th2, R* a, R* b, R* c) {
  // a = sin t / t ; b = (1 - cos t)/t^2 ; c = (t - sin t)/t^3
  if (th2 < R(1e-4)) {
    *a = R(1) - th2 * (R(1) / R(6)) * (R(1) - th2 * R(0.05));
    *b = R(0.5) - th2 * (R(1) / R(24)) * (R(1) - th2 * (R(1) / R(30)));
    *c = R(1) / R(6) - th2 * (R(1) / R(120)) * (R(1) - th2 * (R(1) / R(42)));
  } else {
    R th = nb2_sqrt(th2), s, co, sh, ch;
    nb2_sincos(th, &s, &co);
    nb2_sincos(R(0.5) * th, &sh, &ch);
    *a = s / th;
    R k = sh / (R(0.5) * th);
    *b = R(0.5) * k * k;
    *c = (R(1) - *a) / th2;  // (t - sin t)/t^3 ; fine for t^2 >= 1e-4 in fp64, and for fp32 handled below
    if (sizeof(R) == 4 && th2 < R(0.25)) {
      // series keeps fp32 accuracy where 1 - sin(t)/t cancels
      *c = R(1) / R(6) - th2 * (R(1) / R(120)) * (R(1) - th2 * (R(1) / R(42)) * (R(1) - th2 * (R(1) / R(72))));
    }
  }
}
template <class R> NB2_HD M3<R> skew_sq_combo(const V3<R>& q, R a, R b) {  // I + a [q]x + b [q]x^2
  M3<R> o;
  R xx = q.x * q.x, yy = q.y * q.y, zz = q.z * q.z, xy = q.x * q.y, xz = q.x * q.z, yz = q.y * q.z;
  o.m00 = R(1) - b * (yy + zz); o.m11 = R(1) - b * (xx + zz); o.m22 = R(1) - b * (xx + yy);
  o.m01 = b * xy - a * q.z; o.m10 = b * xy + a * q.z;
  o.m02 = b * xz + a * q.y; o.m20 = b * xz - a * q.y;
  o.m12 = b * yz - a * q.x; o.m21 = b * yz + a * q.x;
  return o;
}
template <class R> NB2_HD M3<R> expmap(const V3<R>& q) {
  R a, b, c; so3_coeffs(dot(q, q), &a, &b, &c);
  return skew_sq_combo(q, a, b);
}
// right Jacobian J_r(q) = I - b [q]x + c [q]x^2 :  R^T dR = [J_r dq]x
template <class R> NB2_HD M3<R> so3_Jr(const V3<R>& q) {
  R a, b, c; so3_coeffs(dot(q, q), &a, &b, &c);
  return skew_sq_combo(q, -b, c);
}
// J_r^{-1}(q) = I + 1/2 [q]x + d [q]x^2 , d = 1/t^2 - (1+cos t)/(2 t sin t)
template <class R> NB2_HD M3<R> so3_Jr_inv(const V3<R>& q) {
  R th2 = dot(q, q), d;
  const R thresh = (sizeof(R) == 4) ? R(1.0) : R(0.04);  // fp32: avoid the 1/t^2 - ... cancellation
  if (th2 < thresh) {
    d = R(1) / R(12) + th2 * (R(1) / R(720)) * (R(1) + th2 * (R(1) / R(42)) * (R(1) + th2 * (R(1) / R(40)) * (R(1) + th2 * (R(1) / R(39.6)) * (R(1) + th2 * (R(1) / R(39.5))))));
  } else {
    R th = nb2_sqrt(th2), sh, ch;
    nb2_sincos(R(0.5) * th, &sh, &ch);
    // (1+cos t)/(2 t sin t) = cos(t/2) / (2 t sin(t/2))
    d = R(1) / th2 - ch / (R(2) * th * sh);
  }
  return skew_sq_combo(q, R(0.5), d);
}
template <class R> NB2_HD V3<R> logmap(const M3<R>& Rm) {
  V3<R> vec = mk3<R>(R(0.5) * (Rm.m21 - Rm.m12), R(0.5) * (Rm.m02 - Rm.m20), R(0.5) * (Rm.m10 - Rm.m01));  // sin(t) * axis
  R co = R(0.5) * (Rm.m00 + Rm.m11 + Rm.m22 - R(1));
  R s2 = dot(vec, vec);
  R s = nb2_sqrt(s2);
  R th = nb2_atan2(s, co);
  const R PI = R(3.14159265358979323846);
  if (th > PI - R(1e-3)) {
    // near pi the skew part vanishes; reference branch (Geometry.cpp:730-743)
    R delta = R(0.5) + R(0.125) * (PI - th) * (PI - th);
    R a0 = th * nb2_sqrt(nb2_abs(R(1) + (Rm.m00 - R(1)) * delta));
    R a1 = th * nb2_sqrt(nb2_abs(R(1) + (Rm.m11 - R(1)) * delta));
    R a2 = th * nb2_sqrt(nb2_abs(R(1) + (Rm.m22 - R(1)) * delta));
    return mk3<R>(Rm.m21 > Rm.m12 ? a0 : -a0, Rm.m02 > Rm.m20 ? a1 : -a1, Rm.m10 > Rm.m01 ? a2 : -a2);
  }
  R k = (s2 < R(1e-8)) ? (R(1) + s2 * (R(1) / R(6))) : (th / s);
  return vec * k;
}

// Cholesky-based inverse of a symmetric positive definite 6x6 given as SI -> SI.  Fully unrolled at compile time.
template <class R> NB2_HD SI<R> spd6_inverse(const SI<R>& I) {
  R a[6][6];
  M3<R> Af = full(I.A), Cf = full(I.C);
  const R* Ap = &Af.m00; const R* Bp = &I.B.m00; const R* Cp = &Cf.m00;
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) { a[i][j] = Ap[3 * i + j]; a[i][3 + j] = Bp[3 * i + j]; a[3 + j][i] = Bp[3 * i + j]; a[3 + i][3 + j] = Cp[3 * i + j]; }
  R L[6][6], invd[6];  // invd[j] = 1 / L[j][j]: every later division by a diagonal entry becomes a multiplication
#pragma unroll
  for (int j = 0; j < 6; j++) {
    R d = a[j][j];
#pragma unroll
    for (int k = 0; k < 6; k++) if (k < j) d -= L[j][k] * L[j][k];
    R ljj = nb2_sqrt(d), inv = nb2_rcp(ljj);
    L[j][j] = ljj; invd[j] = inv;
#pragma unroll
    for (int i = 0; i < 6; i++) if (i > j) {
      R s = a[i][j];
#pragma unroll
      for (int k = 0; k < 6; k++) if (k < j) s -= L[i][k] * L[j][k];
      L[i][j] = s * inv;
    }
  }
  // Linv (lower)
  R Li[6][6];
#pragma unroll
  for (int j = 0; j < 6; j++) {
    Li[j][j] = invd[j];
#pragma unroll
    for (int i = 0; i < 6; i++) if (i > j) {
      R s = R(0);
#pragma unroll
      for (int k = 0; k < 6; k++) if (k >= j && k < i) s -= L[i][k] * Li[k][j];
      Li[i][j] = s * invd[i];
    }
  }
  // inv = Li^T Li
  R v[6][6];
#pragma unroll
  for (int i = 0; i < 6; i++)
#pragma unroll
    for (int j = 0; j < 6; j++) if (j >= i) {
      R s = R(0);
#pragma unroll
      for (int k = 0; k < 6; k++) if (k >= j) s += Li[k][i] * Li[k][j];
      v[i][j] = s;
    }
  SI<R> o;
  o.A.xx = v[0][0]; o.A.yy = v[1][1]; o.A.zz = v[2][2]; o.A.xy = v[0][1]; o.A.xz = v[0][2]; o.A.yz = v[1][2];
  o.C.xx = v[3][3]; o.C.yy = v[4][4]; o.C.zz = v[5][5]; o.C.xy = v[3][4]; o.C.xz = v[3][5]; o.C.yz = v[4][5];
  o.B.m00 = v[0][3]; o.B.m01 = v[0][4]; o.B.m02 = v[0][5]; o.B.m10 = v[1][3]; o.B.m11 = v[1][4]; o.B.m12 = v[1][5]; o.B.m20 = v[2][3]; o.B.m21 = v[2][4]; o.B.m22 = v[2][5];
  return o;
}

}  // namespace nb2
