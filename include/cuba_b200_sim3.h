/*
 * cuba_b200_sim3.h -- Sim(3) alignment of many keyframe pairs for the drop-in class cuba::CudaBundleAdjustment.
 *
 * ORB-SLAM2's Optimizer::OptimizeSim3 refines the similarity S12 between two keyframes from matched map points during loop closing:
 * optimize(5), a chi2 test that drops the failing matches, optimize(10) (optimize(5) when no match was dropped) and the test again;
 * its return value is the number of inliers.  optimizeSim3() runs that procedure for any number of keyframe pairs at once, in one
 * kernel launch on the GPU of the optimizer (one CTA per pair of keyframes): a loop detector can refine every candidate whose RANSAC
 * succeeded and still accept them in its own order, since each result depends on its own problem only.  Always in double precision.
 *
 * A free function, so that the class keeps the reference's vtable.  The optimizer's graph is neither read nor changed: its next
 * initialize() / optimize() give what they would have given without the call.
 */
#ifndef CUBA_B200_SIM3_H
#define CUBA_B200_SIM3_H

#include <cstddef>
#include <vector>

#include "cuda_bundle_adjustment.h"

namespace cuba
{

/** One matched pair: X1 is the point of keyframe 1 in camera-1 coordinates, X2 its match in camera-2 coordinates; obs1 / obs2 the
 *  keypoints in keyframes 1 / 2 and information1 / information2 their scalar informations (ORB-SLAM2: invSigma2 of the octave). */
struct Sim3Match
{
	Array<double, 3> X1, X2;
	Array<double, 2> obs1, obs2;
	double information1 = 1, information2 = 1;
};

/** S12 maps camera-2 coordinates into camera 1: S12 X = s R(q) X + t.  Two monocular edges per match, pi1(S12 X2) against obs1 and
 *  pi2(S12^-1 X1) against obs2; the cameras' bf is not used. */
struct Sim3Problem
{
	Eigen::Quaterniond q;
	Array<double, 3> t;
	double s = 1;
	CameraParams camera1, camera2;
	bool fixScale = false;
	std::vector<Sim3Match> matches;
};

/** OptimizeSim3's parameters: th2 (the chi2 threshold of the test, and the square of the Huber delta), the iterations of the first
 *  optimize, of the second one when the first test dropped a match / when it did not, and the fewest matches the second optimize
 *  needs (with fewer, the result is 0 inliers and the input S12). */
struct Sim3Options
{
	double chi2 = 10;
	int iterations = 5;
	int iterationsBad = 10;
	int iterationsGood = 5;
	int minPairs = 10;
};

struct Sim3Result
{
	Eigen::Quaterniond q;                    // the refined S12 (the input S12 when inliers == 0 for lack of matches)
	Array<double, 3> t;
	double s = 1;
	size_t inliers = 0;                      // OptimizeSim3's return value
	std::vector<int> levels;                 // 0 (inlier) / 1 (dropped) per match, in the problem's order
	std::vector<BatchStatistics> rounds;     // the iterations of the first and of the second optimize
};

/** Runs OptimizeSim3 on every problem in one launch.  std::invalid_argument for a non-finite input, s <= 0 or options the engine
 *  refuses; std::runtime_error when the GPU fails. */
std::vector<Sim3Result> optimizeSim3(CudaBundleAdjustment& ba, const std::vector<Sim3Problem>& problems, const Sim3Options& options = {});

} // namespace cuba

#endif
