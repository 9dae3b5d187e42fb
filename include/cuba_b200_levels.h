/*
 * cuba_b200_levels.h -- edge levels for the drop-in class cuba::CudaBundleAdjustment (include/cuda_bundle_adjustment.h).
 *
 * g2o's `edge->setLevel(1); optimizer.initializeOptimization(0);` keeps an edge in the graph but leaves it out of the objective and
 * the normal equations.  ORB-SLAM2's local BA and pose optimisation run their outlier rounds this way.  The class itself must stay
 * method-for-method the reference's (a drop-in shares its vtable), so levels are free functions on the object create() returned.
 *
 * A level belongs to an edge inside the optimizer: it survives initialize() and optimize(); removeEdge() forgets it and an edge added
 * again starts at 0; an edge with both ends fixed, which initialize() leaves out of the problem, keeps its level for when it comes
 * back.  optimize() applies the levels current when it is called (no initialize() needed).  chiSquared(e) of an edge at level 1 is
 * its omega*|r|^2 with its own information after the last optimize().  With every edge at level 1, optimize() leaves the estimate
 * alone and appends nothing to batchStatistics().
 */
#ifndef CUBA_B200_LEVELS_H
#define CUBA_B200_LEVELS_H

#include <cstddef>

#include "cuda_bundle_adjustment.h"

namespace cuba
{

/** g2o e->setLevel(level): level != 0 excludes the edge.  std::out_of_range for an edge the optimizer does not hold. */
void setEdgeLevel(CudaBundleAdjustment& ba, BaseEdge* e, int level);
/** 0 or 1; after classifyEdges() the device's decision.  std::out_of_range for an edge the optimizer does not hold. */
int edgeLevel(const CudaBundleAdjustment& ba, const BaseEdge* e);

/** ORB-SLAM2's outlier test: an edge fails when chi2 > chi2Mono / chi2Stereo (non-robust omega*|r|^2, the value chiSquared()
 *  returns) or, with requirePositiveDepth, when its landmark is not in front of the camera.  Failing edges go to level 1; with
 *  reinclude, an edge that passes goes back to level 0 (pose optimisation), otherwise levels only go 0 -> 1 (local BA). */
struct OutlierTest
{
	double chi2Mono = 5.991, chi2Stereo = 7.815;
	bool requirePositiveDepth = true;
	bool reinclude = false;
};
struct OutlierCounts
{
	size_t includedMono = 0, includedStereo = 0, excluded = 0, reincluded = 0;   // excluded / reincluded: levels this call changed
};
/** Runs the test on the GPU at the estimate of the last optimize(), on the problem that optimize() solved (edges added or removed
 *  since are not seen), and calls no initialize().  std::logic_error before the first optimize() after an initialize(). */
OutlierCounts classifyEdges(CudaBundleAdjustment& ba, const OutlierTest& test);

} // namespace cuba

#endif
