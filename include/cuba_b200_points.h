/*
 * cuba_b200_points.h -- structure-only refinement of many map points for the drop-in class cuba::CudaBundleAdjustment.
 *
 * A SLAM or SfM back end refines points against keyframes it holds fixed: newly triangulated points against every keyframe that
 * observes them (ORB-SLAM2's CreateNewMapPoints triangulates from two keyframes and never refines), or the points of a map after its
 * keyframes moved (g2o's StructureOnlySolver).  optimizePoints() runs a round schedule for any number of points at once, in one
 * kernel launch on the GPU of the optimizer (one warp per point).  Each point's result is what the optimizer would compute for the
 * point on its own: the landmark as the only free vertex, its edges' poses fixed, every edge at level 0 to start with, and per round
 * the robust kernels, a reset to the point's input position when `restart` is set, optimize(iterations) and classifyEdges()
 * (cuba_b200_levels.h).  Always in double precision.
 *
 * These are free functions, so that the class keeps the reference's vtable.  The optimizer's graph is neither read nor changed:
 * points need not be added to it, and its next initialize() / optimize() give what they would have given without the call.
 */
#ifndef CUBA_B200_POINTS_H
#define CUBA_B200_POINTS_H

#include <cstddef>
#include <vector>

#include "cuda_bundle_adjustment.h"
#include "cuba_b200_levels.h"
#include "cuba_b200_pose.h"

namespace cuba
{

/** One point: a landmark and its edges (MonoEdge / StereoEdge, each with landmarkVertex() == landmark).  The edges' poses are read,
 *  not changed, and shared by pointer between points; the landmark's `fixed` flag is ignored (the landmark is what gets refined). */
struct PointProblem
{
	LandmarkVertex* landmark = nullptr;
	std::vector<BaseEdge*> edges;
};

struct PointResult
{
	std::vector<int> levels;                 // 0 / 1 per edge after the last round, in the point's edge order
	size_t inliers = 0;                      // edges at level 0 after the last round
	std::vector<BatchStatistics> rounds;     // the iterations each round ran (none for a round without an edge at level 0)
};

/** Runs `schedule` (1 to 8 rounds of PoseRound; restart = from the point's input position) on every point in one launch and writes the
 *  refined Xw into each point's LandmarkVertex.  There is no default schedule: ORB-SLAM2 has no structure-only one.
 *  std::invalid_argument for a null landmark or edge, an edge whose landmarkVertex() is not the point's landmark, an edge without a
 *  pose, a non-finite information value or robust-kernel delta, or a schedule the engine refuses; std::runtime_error when the GPU
 *  fails. */
std::vector<PointResult> optimizePoints(CudaBundleAdjustment& ba, const std::vector<PointProblem>& points,
	const std::vector<PoseRound>& schedule);

/** Structure-only refinement of the optimizer's own landmarks in place: the free landmarks of the graph the last initialize() uploaded
 *  (every one, or those listed) against its poses as they stand, held fixed, on the GPU that holds the graph, without a new upload.
 *  Each edge starts at its current level (setEdgeLevel(), classifyEdges()) and each round ends with the outlier test of
 *  classifyEdges() on the refined landmarks' edges, which writes their levels (edgeLevel() shows them).  The refined Xw goes into
 *  each vertex, chiSquared() reports the new estimate, and the next optimize() continues from it; poses and the other landmarks are
 *  not changed.  The fp32 build (USE_FLOAT32) is refused.  Returns the counts of each round over the refined landmarks' edges.
 *  std::logic_error without an optimize() since the last initialize(); std::invalid_argument for a listed vertex that is not a free
 *  landmark of the uploaded graph (null, fixed, added since, or listed twice), or a schedule the engine refuses. */
std::vector<OutlierCounts> optimizeLandmarks(CudaBundleAdjustment& ba, const std::vector<PoseRound>& schedule);
std::vector<OutlierCounts> optimizeLandmarks(CudaBundleAdjustment& ba, const std::vector<PoseRound>& schedule,
	const std::vector<LandmarkVertex*>& landmarks);

} // namespace cuba

#endif
