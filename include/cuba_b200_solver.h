/*
 * cuba_b200_solver.h -- the linear solver of the drop-in class cuba::CudaBundleAdjustment (include/cuda_bundle_adjustment.h).
 *
 * g2o users pick the solver of the reduced camera system when they build the optimizer (LinearSolverDense, LinearSolverEigen,
 * LinearSolverCholmod); Ceres offers DENSE_SCHUR beside ITERATIVE_SCHUR.  PCG (the default) is the engine's preconditioned conjugate
 * gradient family; DENSE_CHOLESKY factors the reduced camera system as a dense fp64 matrix (include/cuba_b200.h:
 * cuba_engine_set_linear_solver), an exact step like the reference's Cholesky, for local-BA windows, densely covisible graphs and
 * graphs the PCG refuses, up to 2730 free poses.  The class must stay method-for-method the reference's (a drop-in shares its
 * vtable), so the choice is a free function on the object create() returned.
 *
 * The choice takes effect at the next optimize() (which then uploads the problem again); edge levels and robust kernels are kept.
 * ORB-SLAM2's local BA with LinearSolverDense semantics:
 *     auto ba = cuba::CudaBundleAdjustment::create();
 *     cuba::setLinearSolver(*ba, cuba::LinearSolverType::DENSE_CHOLESKY);
 */
#ifndef CUBA_B200_SOLVER_H
#define CUBA_B200_SOLVER_H

#include "cuda_bundle_adjustment.h"

namespace cuba
{

enum class LinearSolverType
{
	PCG,              // CUBA_SOLVER_PCG
	DENSE_CHOLESKY    // CUBA_SOLVER_DENSE_CHOLESKY
};

/** Selects the solver of the reduced camera system from the next optimize() on.  std::invalid_argument for an object not made by
 *  cuba::CudaBundleAdjustment::create().  optimize() throws std::runtime_error when the dense solver meets more than 2730 free poses
 *  and free landmarks; the choice stays pending, so a later optimize() tries the upload again. */
void setLinearSolver(CudaBundleAdjustment& ba, LinearSolverType type);
/** The solver the next optimize() uses. */
LinearSolverType linearSolver(const CudaBundleAdjustment& ba);

} // namespace cuba

#endif
