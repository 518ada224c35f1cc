// rcvd_device.cuh -- device-side math of the temporal-consistency optimizer (sm_90a).
//
// What each function computes is fixed by the reference (file:line cited per
// function); how it is computed is ours: analytic Jacobians in "local"
// variables per frame (t, w, phi, D, u) that are later expanded through the
// spline gathers, instead of the reference's multi-pass Jet autodiff.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <float.h>
#include <stdint.h>
#include "../../include/rcvd.h"

namespace rcvd {

struct Layout {
  int k, G, nd, S, ns, nf, offD, offS;
  int npad;   // nf rounded up to a multiple of 16: leading dimension / size of a frame block
};

__host__ __device__ inline bool make_layout(const rcvd_config& c, Layout& L) {
  L.k = (c.value_xform == RCVD_VALUE_SCALESHIFT) ? 2 : 1;
  switch (c.depth_type) {
    case RCVD_DEPTH_IDENTITY: L.G = 0; break;
    case RCVD_DEPTH_GLOBAL: L.G = 1; break;
    case RCVD_DEPTH_GRID:
      if (c.depth_grid_x < 2 || c.depth_grid_y < 2) return false;
      // The reference's linear gather indexes params_[i] rather than params_[i*k]
      // (lib/DepthMapTransform.cpp:801-808,:829-832): not usable with ScaleShift.
      if (L.k == 2 && !c.depth_cubic) return false;
      L.G = c.depth_grid_x * c.depth_grid_y; break;
    default: return false;
  }
  if (c.depth_type != RCVD_DEPTH_IDENTITY && c.value_xform != RCVD_VALUE_SCALE && c.value_xform != RCVD_VALUE_SCALESHIFT) return false;
  L.nd = L.G * L.k;
  switch (c.spatial_type) {
    case RCVD_SPATIAL_IDENTITY: L.S = 0; break;
    case RCVD_SPATIAL_VERTICAL_LINEAR: L.S = 2; break;
    case RCVD_SPATIAL_CORNERS_BILINEAR: L.S = 4; break;
    case RCVD_SPATIAL_BILINEAR_GRID:
    case RCVD_SPATIAL_BICUBIC_GRID:
      if (c.spatial_grid_x < 2 || c.spatial_grid_y < 2) return false;
      L.S = c.spatial_grid_x * c.spatial_grid_y; break;
    default: return false;
  }
  L.ns = 2 * L.S; L.offD = 7; L.offS = 7 + L.nd; L.nf = 7 + L.nd + L.ns;
  L.npad = (L.nf + 15) / 16 * 16;
  return true;
}

// ---------------------------------------------------------------------------
// Gathers.  Cell coordinates in double exactly as the reference
// (lib/DepthMapTransform.cpp:751-764, :868-881, :1257-1271, :1293-1308): explicit
// _rn intrinsics so that no FMA contraction can change an index.
// ---------------------------------------------------------------------------
struct Gather { int n; int idx[16]; double w[16]; };

__device__ __forceinline__ void cell_coord(float loc, int g, int& i, double& r) {
  const double gm1 = (double)(g - 1);
  const double maxc = nextafter(gm1, 0.0);
  double s = __ddiv_rn(__dmul_rn(__dadd_rn((double)loc, 1.0), gm1), 2.0);
  s = fmin(fmax(s, 0.0), maxc);
  i = (int)s;
  r = __dsub_rn(s, (double)i);
}
// cubicSpline, lib/DepthMapTransform.cpp:671-678
__device__ __forceinline__ void cubic_spline(double w[4], double t) {
  const double t2 = __dmul_rn(t, t), t3 = __dmul_rn(t2, t);
  w[0] = __dsub_rn(__dadd_rn(__dmul_rn(-0.5, t3), t2), __dmul_rn(0.5, t));
  w[1] = __dadd_rn(__dsub_rn(__dmul_rn(1.5, t3), __dmul_rn(2.5, t2)), 1.0);
  w[2] = __dadd_rn(__dadd_rn(__dmul_rn(-1.5, t3), __dmul_rn(2.0, t2)), __dmul_rn(0.5, t));
  w[3] = __dsub_rn(__dmul_rn(0.5, t3), __dmul_rn(0.5, t2));
}
// linearGather spatial branch (:822-840) and bilinearSpatialGridGather (:1253-1286)
__device__ __forceinline__ void gather_bilinear(float lx, float ly, int gx, int gy, Gather& g) {
  int ix, iy; double rx, ry;
  cell_coord(lx, gx, ix, rx); cell_coord(ly, gy, iy, ry);
  g.n = 4;
  g.idx[0] = ix + iy * gx; g.idx[1] = ix + 1 + iy * gx; g.idx[2] = ix + (iy + 1) * gx; g.idx[3] = ix + 1 + (iy + 1) * gx;
  const double ox = __dsub_rn(1.0, rx), oy = __dsub_rn(1.0, ry);
  g.w[0] = __dmul_rn(ox, oy); g.w[1] = __dmul_rn(rx, oy); g.w[2] = __dmul_rn(ox, ry); g.w[3] = __dmul_rn(rx, ry);
}
// cubicGather (:853-948, gz == 1) and bicubicSpatialGridGather (:1288-1343): taps outside the
// grid are not created; their weight is folded onto the nearest in-range tap.
__device__ __forceinline__ void gather_bicubic(float lx, float ly, int gx, int gy, Gather& g) {
  int ix, iy; double rx, ry;
  cell_coord(lx, gx, ix, rx); cell_coord(ly, gy, iy, ry);
  double wx[4], wy[4];
  cubic_spline(wx, rx); cubic_spline(wy, ry);
  const int x0 = (ix == 0 ? 1 : 0), x1 = (ix == gx - 2 ? 3 : 4);
  const int y0 = (iy == 0 ? 1 : 0), y1 = (iy == gy - 2 ? 3 : 4);
  const int xs = x1 - x0, ys = y1 - y0;
  g.n = xs * ys;
#pragma unroll
  for (int i = 0; i < 16; ++i) { g.w[i] = 0.0; g.idx[i] = 0; }
  for (int y = y0; y < y1; ++y)
    for (int x = x0; x < x1; ++x) g.idx[(x - x0) + (y - y0) * xs] = (ix - 1 + x) + (iy - 1 + y) * gx;
  // accumulation order y-major then x, as the reference's loops (:936-947 / :1336-1342)
  for (int y = 0; y < 4; ++y)
    for (int x = 0; x < 4; ++x) {
      const int cx = min(max(x - x0, 0), xs - 1), cy = min(max(y - y0, 0), ys - 1);
      const int o = cx + cy * xs;
      g.w[o] = __dadd_rn(g.w[o], __dmul_rn(wx[x], wy[y]));
    }
}
__device__ __forceinline__ void gather_depth(const rcvd_config& c, float lx, float ly, Gather& g) {
  if (c.depth_type == RCVD_DEPTH_IDENTITY) { g.n = 0; }
  else if (c.depth_type == RCVD_DEPTH_GLOBAL) { g.n = 1; g.idx[0] = 0; g.w[0] = 1.0; }   // GlobalDepthFunctor :495-523
  else if (c.depth_cubic) gather_bicubic(lx, ly, c.depth_grid_x, c.depth_grid_y, g);
  else gather_bilinear(lx, ly, c.depth_grid_x, c.depth_grid_y, g);
}
__device__ __forceinline__ void gather_spatial(const rcvd_config& c, float lx, float ly, Gather& g) {
  switch (c.spatial_type) {
    case RCVD_SPATIAL_VERTICAL_LINEAR: {   // :1107-1114
      const double w0 = __dadd_rn(0.5, __dmul_rn(0.5, (double)ly));
      g.n = 2; g.idx[0] = 0; g.idx[1] = 1; g.w[0] = w0; g.w[1] = __dsub_rn(1.0, w0); break; }
    case RCVD_SPATIAL_CORNERS_BILINEAR: {  // :1181-1191
      const double wx = __dadd_rn(0.5, __dmul_rn(0.5, (double)lx)), wy = __dadd_rn(0.5, __dmul_rn(0.5, (double)ly));
      const double ox = __dsub_rn(1.0, wx), oy = __dsub_rn(1.0, wy);
      g.n = 4; g.idx[0] = 0; g.idx[1] = 1; g.idx[2] = 2; g.idx[3] = 3;
      g.w[0] = __dmul_rn(wx, wy); g.w[1] = __dmul_rn(ox, wy); g.w[2] = __dmul_rn(wx, oy); g.w[3] = __dmul_rn(ox, oy); break; }
    case RCVD_SPATIAL_BILINEAR_GRID: gather_bilinear(lx, ly, c.spatial_grid_x, c.spatial_grid_y, g); break;
    case RCVD_SPATIAL_BICUBIC_GRID: gather_bicubic(lx, ly, c.spatial_grid_x, c.spatial_grid_y, g); break;
    default: g.n = 0;
  }
}

// Depth functor value (lib/DepthMapTransform.cpp:457-523, :597-606; ValueXform lib/ValueTransform.h:57-94).
// pf: the frame's parameter vector.
__device__ __forceinline__ double depth_value(const rcvd_config& c, const Layout& L, const Gather& g, float src, const double* __restrict__ pf) {
  const double s = (double)src;
  if (c.depth_type == RCVD_DEPTH_IDENTITY) return s;
  double D = 0.0;
  for (int i = 0; i < g.n; ++i) {
    const double* q = pf + L.offD + g.idx[i] * L.k;
    const double v = (L.k == 2) ? s * q[0] + q[1] : s * q[0];
    D += v * g.w[i];
  }
  return D;
}
// Spatial functor value (:1036-1045, :1075-1085, :1146-1160, :1225-1233)
__device__ __forceinline__ void warp_value(const Layout& L, const Gather& g, const double* __restrict__ pf, double u[2]) {
  u[0] = 0.0; u[1] = 0.0;
  for (int i = 0; i < g.n; ++i) { u[0] += pf[L.offS + 2 * g.idx[i]] * g.w[i]; u[1] += pf[L.offS + 2 * g.idx[i] + 1] * g.w[i]; }
}

// ---------------------------------------------------------------------------
// ceres::AngleAxisRotatePoint (reference call sites lib/PoseOptimizer.cpp:185,:211) and
// its exact derivative w.r.t. the angle-axis vector, both branches.
// f = R(v) p ; R row-major ; dfdv[i*3+j] = d f_i / d v_j
// ---------------------------------------------------------------------------
template <bool JAC>
__device__ __forceinline__ void rotate_point(const double v[3], const double p[3], double f[3], double R[9], double dfdv[9]) {
  const double th2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
  if (th2 > DBL_EPSILON) {
    const double th = sqrt(th2);
    double s, c; sincos(th, &s, &c);
    const double ti = 1.0 / th;
    const double k0 = v[0] * ti, k1 = v[1] * ti, k2 = v[2] * ti;
    const double x0 = k1 * p[2] - k2 * p[1], x1 = k2 * p[0] - k0 * p[2], x2 = k0 * p[1] - k1 * p[0];
    const double kp = k0 * p[0] + k1 * p[1] + k2 * p[2];
    const double omc = 1.0 - c;
    f[0] = p[0] * c + x0 * s + k0 * kp * omc;
    f[1] = p[1] * c + x1 * s + k1 * kp * omc;
    f[2] = p[2] * c + x2 * s + k2 * kp * omc;
    if (JAC) {
      R[0] = c + omc * k0 * k0; R[1] = -s * k2 + omc * k0 * k1; R[2] = s * k1 + omc * k0 * k2;
      R[3] = s * k2 + omc * k1 * k0; R[4] = c + omc * k1 * k1; R[5] = -s * k0 + omc * k1 * k2;
      R[6] = -s * k1 + omc * k2 * k0; R[7] = s * k0 + omc * k2 * k1; R[8] = c + omc * k2 * k2;
      const double k[3] = {k0, k1, k2}, kx[3] = {x0, x1, x2};
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        double dk[3] = {-k0 * k[j] * ti, -k1 * k[j] * ti, -k2 * k[j] * ti};
        dk[j] += ti;
        const double d0 = dk[1] * p[2] - dk[2] * p[1], d1 = dk[2] * p[0] - dk[0] * p[2], d2 = dk[0] * p[1] - dk[1] * p[0];
        const double dkp = dk[0] * p[0] + dk[1] * p[1] + dk[2] * p[2];
        const double dc = -s * k[j], ds = c * k[j];
        const double dd[3] = {d0, d1, d2};
#pragma unroll
        for (int i = 0; i < 3; ++i)
          dfdv[i * 3 + j] = p[i] * dc + dd[i] * s + kx[i] * ds + dk[i] * kp * omc + k[i] * dkp * omc - k[i] * kp * dc;
      }
    }
  } else {
    f[0] = p[0] + (v[1] * p[2] - v[2] * p[1]);
    f[1] = p[1] + (v[2] * p[0] - v[0] * p[2]);
    f[2] = p[2] + (v[0] * p[1] - v[1] * p[0]);
    if (JAC) {
      R[0] = 1; R[1] = -v[2]; R[2] = v[1]; R[3] = v[2]; R[4] = 1; R[5] = -v[0]; R[6] = -v[1]; R[7] = v[0]; R[8] = 1;
      dfdv[0] = 0; dfdv[1] = p[2]; dfdv[2] = -p[1];
      dfdv[3] = -p[2]; dfdv[4] = 0; dfdv[5] = p[0];
      dfdv[6] = p[1]; dfdv[7] = -p[0]; dfdv[8] = 0;
    }
  }
}

// cameraToWorld (lib/PoseOptimizer.cpp:175-192): X = t + R(w) (pcx*phi*a, pcy*phi, -1) D.
// dX[i*10 + j]: derivative of X_i w.r.t. local variable j in (t0..2, w0..2, phi, D, ux, uy).
template <bool JAC>
__device__ __forceinline__ void camera_to_world(const double* pose, double phi, double a, double pcx, double pcy, double D,
                                                double X[3], double dX[30]) {
  const double p[3] = {pcx * phi * a, pcy * phi, -1.0};
  double w[3], R[9], dw[9];
  rotate_point<JAC>(pose + 3, p, w, R, dw);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    X[i] = pose[i] + w[i] * D;
    if (JAC) {
      double* row = dX + i * 10;
      row[0] = (i == 0); row[1] = (i == 1); row[2] = (i == 2);
      row[3] = D * dw[i * 3]; row[4] = D * dw[i * 3 + 1]; row[5] = D * dw[i * 3 + 2];
      row[6] = D * (R[i * 3] * pcx * a + R[i * 3 + 1] * pcy);
      row[7] = w[i];
      row[8] = D * R[i * 3] * phi * a;
      row[9] = D * R[i * 3 + 1] * phi;
    }
  }
}

struct ObsIn { float ndcx, ndcy, depth; };

// StaticSceneCost (lib/PoseOptimizer.cpp:237-308, with worldToCamera :196-221) in local
// variables.  r[3]; Jl[i*20 + j], j<10: frame 0 locals, j>=10: frame 1 locals.
template <bool JAC>
__device__ __forceinline__ void static_scene(const rcvd_config& c, const double* pose0, double phi0, double D0, const double u0[2],
                                             const double* pose1, double phi1, double D1, const double u1[2],
                                             const ObsIn& o0, const ObsIn& o1, double r[3], double* Jl) {
  const double a = c.aspect;
  double X0[3], dX0[30];
  camera_to_world<JAC>(pose0, phi0, a, (double)o0.ndcx + u0[0], (double)o0.ndcy + u0[1], D0, X0, dX0);
  const double pc1x = (double)o1.ndcx + u1[0], pc1y = (double)o1.ndcy + u1[1];
  if (c.static_loss_type == RCVD_LOSS_EUCLIDEAN) {   // :267-272 (no spatial/depth weights)
    double X1[3], dX1[30];
    camera_to_world<JAC>(pose1, phi1, a, pc1x, pc1y, D1, X1, dX1);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      r[i] = X1[i] - X0[i];
      if (JAC) {
#pragma unroll
        for (int j = 0; j < 10; ++j) { Jl[i * 20 + j] = -dX0[i * 10 + j]; Jl[i * 20 + 10 + j] = dX1[i * 10 + j]; }
      }
    }
    return;
  }
  const double rel[3] = {X0[0] - pose1[0], X0[1] - pose1[1], X0[2] - pose1[2]};
  const double v[3] = {-pose1[3], -pose1[4], -pose1[5]};
  double q[3], R1[9], dq[9];
  rotate_point<JAC>(v, rel, q, R1, dq);
  const double depth = -q[2];
  const double fx1 = phi1 * a, fy1 = phi1;
  const double id = 1.0 / depth;
  const double projx = q[0] * id / fx1, projy = q[1] * id / fy1;
  const double ws = c.static_spatial_weight, wd = c.static_depth_weight;
  r[0] = (projx - pc1x) * ws; r[1] = (projy - pc1y) * ws;
  double dA = 0.0, dB = 0.0;
  const double A = depth, B = D1;
  if (c.static_loss_type == RCVD_LOSS_REPRO_DISPARITY) {   // :287-292; max(x, eps) = (x < eps) ? eps : x
    const double eps = 1e-6;
    const bool ca = A < eps, cb = B < eps;
    r[2] = (1.0 / (ca ? eps : A) - 1.0 / (cb ? eps : B)) * wd;
    dA = ca ? 0.0 : -wd / (A * A);
    dB = cb ? 0.0 : wd / (B * B);
  } else {   // :294-300; max = (A<B)?B:A, min = (B<A)?B:A
    const bool mxB = (A < B), mnB = (B < A);
    const double mx = mxB ? B : A, mn = mnB ? B : A;
    const double mxA = mxB ? 0.0 : 1.0, mxBd = mxB ? 1.0 : 0.0, mnA = mnB ? 0.0 : 1.0, mnBd = mnB ? 1.0 : 0.0;
    if (c.static_loss_type == RCVD_LOSS_REPRO_DEPTH_RATIO) {
      r[2] = (mx / mn - 1.0) * wd;
      dA = wd * (mxA / mn - mx / (mn * mn) * mnA);
      dB = wd * (mxBd / mn - mx / (mn * mn) * mnBd);
    } else {
      r[2] = log(mn / mx) * wd;
      dA = wd * (mnA / mn - mxA / mx);
      dB = wd * (mnBd / mn - mxBd / mx);
    }
  }
  if (JAC) {
    const double ax = ws * id / fx1, ay = ws * id / fy1;          // d r0/d q0, d r1/d q1
    const double bx = ws * q[0] * id * id / fx1, by = ws * q[1] * id * id / fy1;  // d r0/d q2, d r1/d q2
#pragma unroll
    for (int j = 0; j < 20; ++j) {
      double Q0, Q1, Q2;
      if (j < 10) {
        Q0 = R1[0] * dX0[j] + R1[1] * dX0[10 + j] + R1[2] * dX0[20 + j];
        Q1 = R1[3] * dX0[j] + R1[4] * dX0[10 + j] + R1[5] * dX0[20 + j];
        Q2 = R1[6] * dX0[j] + R1[7] * dX0[10 + j] + R1[8] * dX0[20 + j];
      } else if (j < 13) { Q0 = -R1[j - 10]; Q1 = -R1[3 + j - 10]; Q2 = -R1[6 + j - 10]; }
      else if (j < 16) { Q0 = dq[j - 13]; Q1 = dq[3 + j - 13]; Q2 = dq[6 + j - 13]; }   // dq/dw1 = -dq/dv, v = -w1 => +
      else { Q0 = 0; Q1 = 0; Q2 = 0; }
      if (j >= 13 && j < 16) { Q0 = -Q0; Q1 = -Q1; Q2 = -Q2; }
      Jl[j] = ax * Q0 + bx * Q2;
      Jl[20 + j] = ay * Q1 + by * Q2;
      Jl[40 + j] = -dA * Q2;
    }
    Jl[16] += -r[0] / phi1 - ws * pc1x / phi1;      // d/dphi1 of ws*(projx - pc1x) = -ws*projx/phi1
    Jl[20 + 16] += -r[1] / phi1 - ws * pc1y / phi1;
    Jl[18] += -ws; Jl[20 + 19] += -ws;
    Jl[40 + 17] += dB;
  }
}

// worldToCamera (lib/PoseOptimizer.cpp:196-221) with derivatives: p = (x, y, depth); dpdX 3x3 (row-major),
// dpdP 3x6 w.r.t. (t1, w1) of the receiving camera, dpdphi 3 w.r.t. its focal.
template <bool JAC>
__device__ __forceinline__ void world_to_camera(const double* pose1, double phi1, double a, const double X[3], double p[3],
                                                double dpdX[9], double dpdP[18], double dpdphi[3]) {
  const double rel[3] = {X[0] - pose1[0], X[1] - pose1[1], X[2] - pose1[2]};
  const double v[3] = {-pose1[3], -pose1[4], -pose1[5]};
  double q[3], R1[9], dq[9];
  rotate_point<JAC>(v, rel, q, R1, dq);
  const double depth = -q[2], id = 1.0 / depth, fx = phi1 * a, fy = phi1;
  p[0] = q[0] * id / fx; p[1] = q[1] * id / fy; p[2] = depth;
  if (JAC) {
    const double g0[3] = {id / fx, 0.0, q[0] * id * id / fx}, g1[3] = {0.0, id / fy, q[1] * id * id / fy}, g2[3] = {0.0, 0.0, -1.0};
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      dpdX[j] = g0[0] * R1[j] + g0[2] * R1[6 + j];
      dpdX[3 + j] = g1[1] * R1[3 + j] + g1[2] * R1[6 + j];
      dpdX[6 + j] = g2[2] * R1[6 + j];
      dpdP[j] = -dpdX[j]; dpdP[6 + j] = -dpdX[3 + j]; dpdP[12 + j] = -dpdX[6 + j];
      // dq/dw1 = -dq/dv
      dpdP[3 + j] = -(g0[0] * dq[j] + g0[2] * dq[6 + j]);
      dpdP[9 + j] = -(g1[1] * dq[3 + j] + g1[2] * dq[6 + j]);
      dpdP[15 + j] = -(g2[2] * dq[6 + j]);
    }
    dpdphi[0] = -p[0] / phi1; dpdphi[1] = -p[1] / phi1; dpdphi[2] = 0.0;
  }
}

// SceneFlowSmoothnessLoss (lib/PoseOptimizer.cpp:332-413) in local variables of the three frames:
// r[3]; Jl[i*30 + j], j < 10 frame f-1, 10..19 frame f, 20..29 frame f+1 (t, w, phi, D, u per frame).
template <bool JAC>
__device__ __forceinline__ void smooth_scene(const rcvd_config& c, const double* const pose[3], const double phi[3], const double D[3],
                                             const double (*u)[2], const ObsIn o[3], double r[3], double* Jl) {
  const double a = c.aspect;
  double X0[3], dX0[30], X2[3], dX2[30];
  camera_to_world<JAC>(pose[0], phi[0], a, (double)o[0].ndcx + u[0][0], (double)o[0].ndcy + u[0][1], D[0], X0, dX0);
  camera_to_world<JAC>(pose[2], phi[2], a, (double)o[2].ndcx + u[2][0], (double)o[2].ndcy + u[2][1], D[2], X2, dX2);
  const double pc1x = (double)o[1].ndcx + u[1][0], pc1y = (double)o[1].ndcy + u[1][1];
  if (JAC) {
#pragma unroll
    for (int i = 0; i < 90; ++i) Jl[i] = 0.0;
  }
  if (c.smooth_loss_type == RCVD_SMOOTH_EUCLIDEAN_LAPLACIAN) {   // :364-373
    double X1[3], dX1[30];
    camera_to_world<JAC>(pose[1], phi[1], a, pc1x, pc1y, D[1], X1, dX1);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      r[i] = X0[i] + X2[i] - 2.0 * X1[i];
      if (JAC) {
#pragma unroll
        for (int j = 0; j < 10; ++j) { Jl[i * 30 + j] = dX0[i * 10 + j]; Jl[i * 30 + 10 + j] = -2.0 * dX1[i * 10 + j]; Jl[i * 30 + 20 + j] = dX2[i * 10 + j]; }
      }
    }
    return;
  }
  double p01[3], p21[3], A0[9], A2[9], B0[18], B2[18], f0[3], f2[3];
  world_to_camera<JAC>(pose[1], phi[1], a, X0, p01, A0, B0, f0);
  world_to_camera<JAC>(pose[1], phi[1], a, X2, p21, A2, B2, f2);
  const double ip = 1.0 / phi[1];
  r[0] = (p01[0] + p21[0] - 2.0 * pc1x) * ip;
  r[1] = (p01[1] + p21[1] - 2.0 * pc1y) * ip;
  const double za = p01[2], zc = p21[2], zb = D[1];
  double da, dc, db;   // d r2 / d(za, zc, zb)
  if (c.smooth_loss_type == RCVD_SMOOTH_REPRO_DISPARITY_LAPLACIAN) {   // :388-394
    const double eps = 1e-6;
    const bool ca = za < eps, cb = zb < eps, cc = zc < eps;
    r[2] = 1.0 / (ca ? eps : za) + 1.0 / (cc ? eps : zc) - 2.0 / (cb ? eps : zb);
    da = ca ? 0.0 : -1.0 / (za * za); dc = cc ? 0.0 : -1.0 / (zc * zc); db = cb ? 0.0 : 2.0 / (zb * zb);
  } else {   // :396-405: base = zb, other = za + zc - zb; max = (base<other)?other:base, min = (other<base)?other:base
    const double base = zb, other = za + zc - zb;
    const bool mxO = base < other, mnO = other < base;
    const double mx = mxO ? other : base, mn = mnO ? other : base;
    double dbase, dother;
    if (c.smooth_loss_type == RCVD_SMOOTH_REPRO_DEPTH_RATIO_CONSISTENCY) {
      r[2] = mx / mn - 1.0;
      dbase = (mxO ? 0.0 : 1.0) / mn - mx / (mn * mn) * (mnO ? 0.0 : 1.0);
      dother = (mxO ? 1.0 : 0.0) / mn - mx / (mn * mn) * (mnO ? 1.0 : 0.0);
    } else {
      r[2] = log(mn / mx);
      dbase = (mnO ? 0.0 : 1.0) / mn - (mxO ? 0.0 : 1.0) / mx;
      dother = (mnO ? 1.0 : 0.0) / mn - (mxO ? 1.0 : 0.0) / mx;
    }
    da = dother; dc = dother; db = dbase - dother;
  }
  if (JAC) {
    const double wr[3] = {ip, ip, 0.0};
#pragma unroll
    for (int row = 0; row < 3; ++row) {
      const double s0 = (row < 2) ? wr[row] : da, s2 = (row < 2) ? wr[row] : dc;
#pragma unroll
      for (int j = 0; j < 10; ++j) {
        Jl[row * 30 + j] = s0 * (A0[row * 3] * dX0[j] + A0[row * 3 + 1] * dX0[10 + j] + A0[row * 3 + 2] * dX0[20 + j]);
        Jl[row * 30 + 20 + j] = s2 * (A2[row * 3] * dX2[j] + A2[row * 3 + 1] * dX2[10 + j] + A2[row * 3 + 2] * dX2[20 + j]);
      }
#pragma unroll
      for (int j = 0; j < 6; ++j) Jl[row * 30 + 10 + j] = s0 * B0[row * 6 + j] + s2 * B2[row * 6 + j];
    }
    Jl[16] = (f0[0] + f2[0]) * ip - r[0] * ip;
    Jl[30 + 16] = (f0[1] + f2[1]) * ip - r[1] * ip;
    Jl[18] = -2.0 * ip; Jl[30 + 19] = -2.0 * ip;
    Jl[60 + 17] = db;
  }
}

// Robust loss rho(s) = {rho, rho', rho''}; CauchyLoss is the reference's
// (lib/PoseOptimizer.cpp:1219-1220); restated from ceres/loss_function.cc.
__device__ __forceinline__ void robust_loss(const rcvd_config& c, double s, double& rho0, double& rho1) {
  if (c.robust_type == RCVD_ROBUST_CAUCHY) {
    const double b = c.robustness * c.robustness, ci = 1.0 / b;
    const double sum = 1.0 + s * ci, inv = 1.0 / sum;
    rho0 = b * log(sum); rho1 = fmax(DBL_MIN, inv);
  } else if (c.robust_type == RCVD_ROBUST_HUBER) {
    const double a = c.robustness, b = a * a;
    if (s > b) { const double rr = sqrt(s); rho0 = 2.0 * a * rr - b; rho1 = fmax(DBL_MIN, a / rr); }
    else { rho0 = s; rho1 = 1.0; }
  } else { rho0 = s; rho1 = 1.0; }
}

__device__ __forceinline__ void red_add(double* addr, double v) {
  // RED.E.ADD.F64 (no return value): L2-resident atomic add
  asm volatile("red.global.add.f64 [%0], %1;" ::"l"(addr), "d"(v) : "memory");
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace rcvd
