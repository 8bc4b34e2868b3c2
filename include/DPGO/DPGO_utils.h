// DPGO_utils.h -- host utilities either side of the hot path (reader, Laplacian assembly, initial guesses,
// projections, single-pose averaging).  Signature-compatible with the reference's
// include/DPGO/DPGO_utils.h:26-208; one-shot setup work stays on the host as in the reference.
#ifndef DPGO_B200_UTILS_H
#define DPGO_B200_UTILS_H

#include <DPGO/DPGO_types.h>
#include <DPGO/RelativeSEMeasurement.h>

namespace DPGO {

void writeMatrixToFile(const Matrix &M, const std::string &filename);
void writeSparseMatrixToFile(const SparseMatrix &M, const std::string &filename);

// .g2o reader (EDGE_SE2 / EDGE_SE3:QUAT); ref src/DPGO_utils.cpp:64-197
std::vector<RelativeSEMeasurement> read_g2o_file(const std::string &filename, size_t &num_poses);

// Q = A Omega A^T of the pose graph; ref src/DPGO_utils.cpp:199-271
void constructOrientedConnectionIncidenceMatrixSE(const std::vector<RelativeSEMeasurement> &measurements,
                                                  SparseMatrix &AT, DiagonalMatrix &OmegaT);
SparseMatrix constructConnectionLaplacianSE(const std::vector<RelativeSEMeasurement> &measurements);

// initial guesses; ref src/DPGO_utils.cpp:362-461
Matrix chordalInitialization(size_t dimension, size_t num_poses, const std::vector<RelativeSEMeasurement> &measurements);
// GPU extension: the same two least-squares problems solved on the GPU (conjugate gradients over the block-CSR product
// kernel, dpgo_chordal_initialization); device < 0: env DPGO_DEVICE or 0.  Throws std::runtime_error on failure.
Matrix chordalInitializationGPU(size_t dimension, size_t num_poses, const std::vector<RelativeSEMeasurement> &measurements,
                                int device = -1, double tol = 1e-11);
// GPU extension: marginal covariances of the poses of trajectory T (d x (d+1)n, e.g. DeviceRBCD::trajectory()) under the
// Gauss-Newton information of the measurements (weights honoured), pose `anchor` fixed (dpgo_pose_covariances; the model
// is in dpgo_b200.h).  pose[p]: b x b, b = 6 (3D: rotation then translation) or 3 (2D: angle then translation), the
// anchor's block 0; pair[q]: the cross block Sigma[x_i, x_j] of pairs[q] = (i, j).  device < 0: env DPGO_DEVICE or 0.
// Throws std::runtime_error on failure.
struct PoseCovariances {
  std::vector<Matrix> pose, pair;
};
PoseCovariances poseCovariancesGPU(size_t dimension, size_t num_poses, const std::vector<RelativeSEMeasurement> &measurements,
                                   const Matrix &T, size_t anchor = 0,
                                   const std::vector<std::pair<size_t, size_t>> &pairs = {}, int device = -1);
Matrix odometryInitialization(size_t dimension, size_t num_poses, const std::vector<RelativeSEMeasurement> &odometry);

// projections; ref src/DPGO_utils.cpp:463-492
Matrix projectToRotationGroup(const Matrix &M);
Matrix projectToStiefelManifold(const Matrix &M);
Matrix fixedStiefelVariable(unsigned d, unsigned r);

double computeMeasurementError(const RelativeSEMeasurement &m, const Matrix &R1, const Matrix &t1, const Matrix &R2,
                               const Matrix &t2);
double chi2inv(double quantile, size_t dof);
double angular2ChordalSO3(double rad);
void checkRotationMatrix(const Matrix &R);

// single-pose averaging used by the cross-robot frame alignment; ref src/DPGO_utils.cpp:518-711
void singleTranslationAveraging(Vector &tOpt, const std::vector<Vector> &tVec, const Vector &tau = Vector::Ones(0));
void singleRotationAveraging(Matrix &ROpt, const std::vector<Matrix> &RVec, const Vector &kappa = Vector::Ones(0));
void singlePoseAveraging(Matrix &ROpt, Vector &tOpt, const std::vector<Matrix> &RVec, const std::vector<Vector> &tVec,
                         const Vector &kappa = Vector::Ones(0), const Vector &tau = Vector::Ones(0));
void robustSingleRotationAveraging(Matrix &ROpt, std::vector<size_t> &inlierIndices, const std::vector<Matrix> &RVec,
                                   const Vector &kappa = Vector::Ones(0), double errorThreshold = 0.1);
void robustSinglePoseAveraging(Matrix &ROpt, Vector &tOpt, std::vector<size_t> &inlierIndices,
                               const std::vector<Matrix> &RVec, const std::vector<Vector> &tVec,
                               const Vector &kappa = Vector::Ones(0), const Vector &tau = Vector::Ones(0),
                               double errorThreshold = 0.1);

// thin SVD of a small dense matrix (one-sided Jacobi): M = U diag(s) V^T, U is rows x cols
void smallSVD(const Matrix &M, Matrix &U, Vector &s, Matrix &V);

}  // namespace DPGO
#endif
