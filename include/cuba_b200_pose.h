/*
 * cuba_b200_pose.h -- pose optimisation of many frames for the drop-in class cuba::CudaBundleAdjustment.
 *
 * ORB-SLAM2's Optimizer::PoseOptimization refines one frame's pose against fixed map points in four rounds of optimize(10), with an
 * outlier test and re-inclusion after each.  optimizePoses() runs that schedule for any number of frames at once, in one kernel
 * launch on the GPU of the optimizer (one CTA per frame).  Each frame's result is what the optimizer would compute for the frame on
 * its own: the pose as the only free vertex, its edges' landmarks fixed, every edge at level 0 to start with, and per round the
 * robust kernels, a reset to the frame's pose when `restart` is set, optimize(iterations) and classifyEdges() (cuba_b200_levels.h).
 * Always in double precision.
 *
 * These are free functions, so that the class keeps the reference's vtable.  The optimizer's graph is neither read nor changed:
 * frames need not be added to it, and its next initialize() / optimize() give what they would have given without the call.
 */
#ifndef CUBA_B200_POSE_H
#define CUBA_B200_POSE_H

#include <cstddef>
#include <vector>

#include "cuda_bundle_adjustment.h"
#include "cuba_b200_levels.h"

namespace cuba
{

/** One frame: a pose and its edges (MonoEdge / StereoEdge, each with poseVertex() == pose).  The edges' landmarks are read, not
 *  changed; the pose's `fixed` flag is ignored (the pose is what gets optimised). */
struct PoseFrame
{
	PoseVertex* pose = nullptr;
	std::vector<BaseEdge*> edges;
};

/** One round: optimize(iterations) under the robust kernels, from the frame's input pose when restart is set (ORB-SLAM2 calls
 *  setEstimate(mTcw) at the top of every round), then `test` on the result. */
struct PoseRound
{
	int iterations = 10;
	RobustKernelType kernelMono = RobustKernelType::NONE, kernelStereo = RobustKernelType::NONE;
	double deltaMono = 0, deltaStereo = 0;
	bool restart = true;
	OutlierTest test;
};

/** ORB-SLAM2's schedule: four rounds of 10 iterations from the frame's pose; Huber with delta sqrt(5.991) / sqrt(7.815) in rounds 0-1,
 *  no robust kernel in rounds 2-3; chi2 test at 5.991 / 7.815 with re-inclusion and without the depth test after each round. */
std::vector<PoseRound> orbSlam2PoseSchedule();

struct PoseResult
{
	std::vector<int> levels;                 // 0 / 1 per edge after the last round, in the frame's edge order
	size_t inliers = 0;                      // edges at level 0 after the last round (PoseOptimization's return value)
	std::vector<BatchStatistics> rounds;     // the iterations each round ran (none for a round without an edge at level 0)
};

/** Runs `schedule` (1 to 8 rounds) on every frame in one launch and writes the refined q / t into each frame's PoseVertex.
 *  std::invalid_argument for a null pose or edge, an edge whose poseVertex() is not the frame's pose, an edge without a landmark, a
 *  non-finite information value or robust-kernel delta, or a schedule the engine refuses; std::runtime_error when the GPU fails. */
std::vector<PoseResult> optimizePoses(CudaBundleAdjustment& ba, const std::vector<PoseFrame>& frames,
	const std::vector<PoseRound>& schedule = orbSlam2PoseSchedule());

} // namespace cuba

#endif
