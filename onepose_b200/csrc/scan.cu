// An annotated scan's object poses and crop geometry on the GPU: the arithmetic of parse_scanned_data.py's data_process_anno
// (:184-240) and parse_video (:129-181) once the scan's text files are read and its video decoded.
//   data_process_anno's loop over ARposes rows     quat2mat, the flip, T_oc, reproj, the skip rule, the kept rows' order   opb_scan_poses
//   parse_video's M and box after the two crops    inv(T2 @ T1), reproj with K_crop, min / max                           opb_scan_crop_geometry
// The crops themselves are opb_crop_resize_colour (csrc/crop.cu).  Everything is fp64 with every product and sum rounded on its
// own (__dmul_rn / __dadd_rn, no fused multiply-add) in numpy's index order; the model is tests/scan_reference.py.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/onepose_b200.h"
#include "block.cuh"
#include "host_util.cuh"

namespace opb {
namespace {

constexpr int kScanThreads = 256;

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dv(double a, double b) { return __ddiv_rn(a, b); }

// transforms3d.quaternions.quat2mat of q = (w, x, y, z), its non-normalising formula: s = 2 / |q|^2, the identity below float64
// eps.  The rotation of q / |q| for any q above that bound.
__device__ void quat2mat(const double* q, double R[3][3]) {
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  const double Nq = add(add(add(mul(w, w), mul(x, x)), mul(y, y)), mul(z, z));
  if (Nq < 2.220446049250313e-16) {
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) R[r][c] = r == c ? 1.0 : 0.0;
    return;
  }
  const double s = dv(2.0, Nq);
  const double X = mul(x, s), Y = mul(y, s), Z = mul(z, s);
  const double wX = mul(w, X), wY = mul(w, Y), wZ = mul(w, Z);
  const double xX = mul(x, X), xY = mul(x, Y), xZ = mul(x, Z);
  const double yY = mul(y, Y), yZ = mul(y, Z), zZ = mul(z, Z);
  R[0][0] = sub(1.0, add(yY, zZ)); R[0][1] = sub(xY, wZ);          R[0][2] = add(xZ, wY);
  R[1][0] = add(xY, wZ);          R[1][1] = sub(1.0, add(xX, zZ)); R[1][2] = sub(yZ, wX);
  R[2][0] = sub(xZ, wY);          R[2][1] = add(yZ, wX);          R[2][2] = sub(1.0, add(xX, yY));
}

// The inverse of the affine [A t; 0 1] (A 3x3): [A^-1, -A^-1 t], A^-1 as the adjugate over the determinant.  np.linalg.inv's LU
// gives the same matrix to a few ulps.
__device__ void affine_inverse3(const double A[3][3], const double* t, double Ai[3][3], double* ti) {
  const double c00 = sub(mul(A[1][1], A[2][2]), mul(A[1][2], A[2][1]));
  const double c01 = sub(mul(A[1][2], A[2][0]), mul(A[1][0], A[2][2]));
  const double c02 = sub(mul(A[1][0], A[2][1]), mul(A[1][1], A[2][0]));
  const double det = add(add(mul(A[0][0], c00), mul(A[0][1], c01)), mul(A[0][2], c02));
  Ai[0][0] = dv(c00, det);
  Ai[1][0] = dv(c01, det);
  Ai[2][0] = dv(c02, det);
  Ai[0][1] = dv(sub(mul(A[0][2], A[2][1]), mul(A[0][1], A[2][2])), det);
  Ai[1][1] = dv(sub(mul(A[0][0], A[2][2]), mul(A[0][2], A[2][0])), det);
  Ai[2][1] = dv(sub(mul(A[0][1], A[2][0]), mul(A[0][0], A[2][1])), det);
  Ai[0][2] = dv(sub(mul(A[0][1], A[1][2]), mul(A[0][2], A[1][1])), det);
  Ai[1][2] = dv(sub(mul(A[0][2], A[1][0]), mul(A[0][0], A[1][2])), det);
  Ai[2][2] = dv(sub(mul(A[0][0], A[1][1]), mul(A[0][1], A[1][0])), det);
  for (int r = 0; r < 3; ++r) ti[r] = -add(add(mul(Ai[r][0], t[0]), mul(Ai[r][1], t[1])), mul(Ai[r][2], t[2]));
}

// data_process_anno's T_oc of ARposes row `a` = (timestamp, position, quaternion w-first) and the object's T_ow [4][4]:
// R = quat2mat(q) @ diag(1, -1, -1) (a sign flip of columns 1 and 2, exact), T_cw = [R p; 0 1], T_oc = inv(T_cw) @ T_ow.
// Rows 0..2 of T_oc; its last row is T_ow's.
__device__ void object_pose(const double* a, const double* T_ow, double T[3][4]) {
  double R[3][3];
  quat2mat(a + 4, R);
  for (int r = 0; r < 3; ++r) { R[r][1] = -R[r][1]; R[r][2] = -R[r][2]; }
  double Ri[3][3], ti[3];
  affine_inverse3(R, a + 1, Ri, ti);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c)
      T[r][c] = add(add(add(mul(Ri[r][0], T_ow[c]), mul(Ri[r][1], T_ow[4 + c])), mul(Ri[r][2], T_ow[8 + c])), mul(ti[r], T_ow[12 + c]));
}

// P = K @ T[:3] (3x4): reproj's K_homo @ pose, whose fourth K_homo column is zero
__device__ void camera_matrix(const double* K, const double T[3][4], double P[3][4]) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) P[r][c] = add(add(mul(K[r * 3], T[0][c]), mul(K[r * 3 + 1], T[1][c])), mul(K[r * 3 + 2], T[2][c]));
}

// reproj of corner X under P: (P @ [X; 1])[:2] / (P @ [X; 1])[2]
__device__ __forceinline__ void project(const double P[3][4], const double* X, double* uv) {
  double p[3];
  for (int r = 0; r < 3; ++r) p[r] = add(add(add(mul(P[r][0], X[0]), mul(P[r][1], X[1])), mul(P[r][2], X[2])), P[r][3]);
  uv[0] = dv(p[0], p[2]);
  uv[1] = dv(p[1], p[2]);
}

// numpy's min / max over the corners, NaN propagating: ext = [x0, y0, x1, y1]
__device__ void corner_extent(const double P[3][4], const double* corners, int n, double* ext) {
  ext[0] = ext[1] = INFINITY;
  ext[2] = ext[3] = -INFINITY;
  for (int i = 0; i < n; ++i) {
    double uv[2];
    project(P, corners + (size_t)i * 3, uv);
    for (int a = 0; a < 2; ++a) {
      if (!isnan(ext[a]) && (isnan(uv[a]) || uv[a] < ext[a])) ext[a] = uv[a];
      if (!isnan(ext[2 + a]) && (isnan(uv[a]) || uv[a] > ext[2 + a])) ext[2 + a] = uv[a];
    }
  }
}

// One block walks the rows in order, kScanThreads at a time: each thread computes its row's pose and the extent of its
// projected corners, the skip rule decides keep, and a block scan gives each kept row its slot, the number of kept rows before
// it.  Slots below n_out get the pose, projections, box and source row; slots from the kept count to n_out are cleared.
__global__ void __launch_bounds__(kScanThreads) scan_poses_kernel(const double* __restrict__ K, const double* __restrict__ rows, int n_rows,
                                                                  const double* __restrict__ T_ow, const double* __restrict__ corners, int n_corners,
                                                                  int n_out, double* __restrict__ pose, double* __restrict__ proj,
                                                                  int32_t* __restrict__ box, int32_t* __restrict__ row_of, int32_t* __restrict__ keep,
                                                                  int32_t* __restrict__ count) {
  __shared__ int sh[kScanThreads / 32];
  double Tow[16], Kc[9];
  for (int i = 0; i < 16; ++i) Tow[i] = T_ow[i];
  for (int i = 0; i < 9; ++i) Kc[i] = K[i];
  int base = 0;
  for (int start = 0; start < n_rows; start += kScanThreads) {
    const int r = start + (int)threadIdx.x;
    double T[3][4], P[3][4], ext[4];
    bool kept = false;
    if (r < n_rows) {
      object_pose(rows + (size_t)r * 8, Tow, T);
      camera_matrix(Kc, T, P);
      corner_extent(P, corners, n_corners, ext);
      kept = !(ext[0] < -1000.0 || ext[1] < -1000.0 || ext[2] > 3000.0 || ext[3] > 3000.0);   // NaN compares false: kept
      if (keep) keep[r] = kept ? 1 : 0;
    }
    int total;
    const int slot = base + block_rank(kept, sh, &total);
    if (kept && slot < n_out) {
      double* Po = pose + (size_t)slot * 16;
      for (int rr = 0; rr < 3; ++rr)
        for (int c = 0; c < 4; ++c) Po[rr * 4 + c] = T[rr][c];
      for (int c = 0; c < 4; ++c) Po[12 + c] = Tow[12 + c];
      if (proj)
        for (int i = 0; i < n_corners; ++i) project(P, corners + (size_t)i * 3, proj + ((size_t)slot * n_corners + i) * 2);
      bool finite = true;
      for (int a = 0; a < 4; ++a) finite = finite && ext[a] > -2147483649.0 && ext[a] < 2147483648.0;   // false for NaN
      for (int a = 0; a < 4; ++a) box[(size_t)slot * 4 + a] = finite ? (int32_t)ext[a] : 0;
      if (row_of) row_of[slot] = r;
    }
    base += total;
  }
  for (int s = base + (int)threadIdx.x; s < n_out; s += kScanThreads) {
    for (int i = 0; i < 16; ++i) pose[(size_t)s * 16 + i] = 0.0;
    if (proj)
      for (int i = 0; i < n_corners * 2; ++i) proj[(size_t)s * n_corners * 2 + i] = 0.0;
    for (int a = 0; a < 4; ++a) box[(size_t)s * 4 + a] = 0;
    if (row_of) row_of[s] = -1;
  }
  if (threadIdx.x == 0) *count = base;
}

// One thread per frame: parse_video's M = inv(T2_homo @ T1_homo) and box_new, the extent of reproj(K_crop_homo, pose, corners).
__global__ void scan_crop_geometry_kernel(const double* __restrict__ trans, const double* __restrict__ K_crop, const double* __restrict__ pose,
                                          const double* __restrict__ corners, int n_corners, const int32_t* __restrict__ status, int F,
                                          double* __restrict__ M, double* __restrict__ box_crop) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  double* Mo = M + (size_t)f * 9;
  double* bo = box_crop + (size_t)f * 4;
  if (!status[f]) {
    for (int i = 0; i < 9; ++i) Mo[i] = 0.0;
    for (int i = 0; i < 4; ++i) bo[i] = 0.0;
    return;
  }
  const double* T1 = trans + (size_t)f * 12;
  const double* T2 = T1 + 6;
  double A[2][3];            // (T2_homo @ T1_homo)[:2]; its last row is (0, 0, 1)
  for (int r = 0; r < 2; ++r)
    for (int c = 0; c < 3; ++c) A[r][c] = add(add(mul(T2[r * 3], T1[c]), mul(T2[r * 3 + 1], T1[3 + c])), mul(T2[r * 3 + 2], c == 2 ? 1.0 : 0.0));
  // its inverse as an affine of the plane: the 2x2 block's adjugate over its determinant, then -A^-1 t
  const double det = sub(mul(A[0][0], A[1][1]), mul(A[0][1], A[1][0]));
  const double i00 = dv(A[1][1], det), i01 = dv(-A[0][1], det), i10 = dv(-A[1][0], det), i11 = dv(A[0][0], det);
  Mo[0] = i00; Mo[1] = i01; Mo[2] = -add(mul(i00, A[0][2]), mul(i01, A[1][2]));
  Mo[3] = i10; Mo[4] = i11; Mo[5] = -add(mul(i10, A[0][2]), mul(i11, A[1][2]));
  Mo[6] = 0.0; Mo[7] = 0.0; Mo[8] = 1.0;
  double T[3][4], P[3][4];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) T[r][c] = pose[(size_t)f * 16 + r * 4 + c];
  camera_matrix(K_crop + (size_t)f * 9, T, P);
  corner_extent(P, corners, n_corners, bo);
}

}  // namespace
}  // namespace opb

extern "C" int opb_scan_poses(const double* K, const double* arposes, int32_t n_rows, const double* T_ow, const double* corners, int32_t n_corners,
                              int32_t n_out, double* pose, double* proj, int32_t* box, int32_t* row, int32_t* keep, int32_t* count, void* stream) {
  REQUIRE(__func__, K && arposes && T_ow && corners && pose && box && count);
  REQUIRE(__func__, n_rows > 0 && n_corners > 0 && n_corners <= 1024 && n_out > 0);
  LAUNCH_NH(__func__, opb::scan_poses_kernel, 1, opb::kScanThreads, 0, (cudaStream_t)stream, K, arposes, n_rows, T_ow, corners, n_corners, n_out, pose,
            proj, box, row, keep, count);
  return OPB_OK;
}

extern "C" int opb_scan_crop_geometry(const double* trans, const double* K_crop, const double* pose, const double* corners, int32_t n_corners,
                                      const int32_t* status, int32_t F, double* M, double* box_crop, void* stream) {
  REQUIRE(__func__, trans && K_crop && pose && corners && status && M && box_crop);
  REQUIRE(__func__, F > 0 && n_corners > 0 && n_corners <= 1024);
  LAUNCH_NH(__func__, opb::scan_crop_geometry_kernel, (unsigned)((F + 127) / 128), 128, 0, (cudaStream_t)stream, trans, K_crop, pose, corners,
            n_corners, status, F, M, box_crop);
  return OPB_OK;
}
