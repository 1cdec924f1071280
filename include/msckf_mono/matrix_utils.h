// include/msckf_mono/matrix_utils.h -- drop-in for the reference's include/msckf_mono/matrix_utils.h (":N" = its line N):
// the small host helpers the reference's callers reach through this header (src/corner_detector.cpp via
// corner_detector.h:24).  Inside the GPU filter none of them is on the numeric path any more -- the skew / Omega
// products live in k_propagate / k_augment and the covariance slicing of the prune functions is k_gather
// (msckf_mono_b200/csrc/state_kernels.cuh) -- so these are plain host functions over the boundary types of types.h,
// compiled against Eigen when it is present and against the stand-ins of pod_linalg.h otherwise.
#pragma once

#include <msckf_mono/types.h>

namespace msckf_mono {
// :8-17  skew-symmetric form of a 3-vector
template <typename _Scalar>
inline Matrix3<_Scalar> vectorToSkewSymmetric(const Vector3<_Scalar>& Vec) {
  Matrix3<_Scalar> M;
  M << 0, -Vec(2), Vec(1),
       Vec(2), 0, -Vec(0),
       -Vec(1), Vec(0), 0;
  return M;
}

// :20-30  Omega(w) = [[-skew(w), w], [-w^T, 0]]
template <typename _Scalar>
inline Matrix4<_Scalar> omegaMat(const Vector3<_Scalar>& omega) {
  Matrix4<_Scalar> bigOmega;
  bigOmega.setZero();
  const Matrix3<_Scalar> sk = vectorToSkewSymmetric(omega);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) bigOmega(i, j) = -sk(i, j);
    bigOmega(i, 3) = omega(i);
    bigOmega(3, i) = -omega(i);
  }
  return bigOmega;
}

// :33-40  (the reference writes Vec(3), one past the end of a 3-vector; nothing calls it -- restated with the index it means)
template <typename _Scalar>
inline Vector3<_Scalar> skewSymmetricToVector(const Matrix3<_Scalar>& Skew) {
  Vector3<_Scalar> Vec;
  Vec(0) = Skew(2, 1);
  Vec(1) = Skew(0, 2);
  Vec(2) = Skew(1, 0);
  return Vec;
}

#ifdef MSCKF_B200_HAVE_EIGEN
// :43-51  condition number through the singular values (needs Eigen's JacobiSVD; unused by the filter and its callers)
template <typename _Scalar>
_Scalar cond(const MatrixX<_Scalar>& M) {
  Eigen::JacobiSVD<MatrixX<_Scalar>> svd(M);
  return svd.singularValues()(0) / svd.singularValues()(svd.singularValues().size() - 1);
}
#endif

// :58-68  out = in(inds, inds)
template <typename _Scalar>
inline void square_slice(const MatrixX<_Scalar>& in, const IndexVector& inds, MatrixX<_Scalar>& out) {
  const int inds_size = (int)inds.rows();
  out.resize(inds_size, inds_size);
  for (int i = 0; i < inds_size; i++)
    for (int j = 0; j < inds_size; j++) out(i, j) = in(inds(i), inds(j));
}

// :76-87  out = in(:, inds)
template <typename _Scalar, int _Rows>
inline void column_slice(const FixedMatrix<_Scalar, _Rows, DynamicSize>& in, const IndexVector& inds,
                         FixedMatrix<_Scalar, _Rows, DynamicSize>& out) {
  const int inds_size = (int)inds.rows();
  const int rows = (int)in.rows();
  out.resize(rows, inds_size);
  for (int i = 0; i < rows; i++)
    for (int j = 0; j < inds_size; j++) out(i, j) = in(i, inds(j));
}
}  // namespace msckf_mono
