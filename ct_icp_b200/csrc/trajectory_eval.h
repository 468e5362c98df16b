// trajectory_eval.h — kitti::EvaluatePoses and ComputeTrajectoryMetrics (include/SlamCore/eval.h, src/SlamCore/eval.cxx of
// the reference) on one device: B estimates against one ground truth per call. Semantics and refusals: include/cticp.h.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "../../include/cticp.h"
#include "trajectory.h"

namespace cticp {

// The argument checks of each entry point; throw std::invalid_argument before anything touches a device.
void CheckKittiArgs(const cticp_pose *gt, size_t n, const cticp_pose *est, size_t num_estimates, const double *lengths,
                    size_t num_lengths, const cticp_kitti_errors *out);
void CheckKittiTrajectoryArgs(const cticp_pose *gt, size_t n, const double *lengths, size_t num_lengths,
                              const cticp_kitti_errors *out);
void CheckMetricsArgs(const cticp_pose *gt, size_t n, const cticp_pose *est, size_t num_estimates,
                      double segment_length, const cticp_traj_metrics *out);
void CheckDistancesArgs(const cticp_pose *gt, size_t n, int kind, const double *out);

// The evaluations proper, on the current device (set by the caller), synchronous; return the pair / segment count.
int64_t KittiEvaluate(const cticp_pose *gt, size_t n, const cticp_pose *est, size_t num_estimates, const double *lengths,
                      size_t num_lengths, cticp_kitti_errors *out, double *tab_errors, size_t cap);
int64_t KittiEvaluateTrajectory(ContinuousTrajectory &t, const cticp_pose *gt, size_t n, const double *lengths,
                                size_t num_lengths, cticp_kitti_errors *out, double *tab_errors, size_t cap);
int64_t TrajectoryMetrics(const cticp_pose *gt, size_t n, const cticp_pose *est, size_t num_estimates,
                          double segment_length, cticp_traj_metrics *out, cticp_traj_segment *segments, size_t cap);
void TrajectoryDistances(const cticp_pose *gt, size_t n, int kind, double *out);

}  // namespace cticp
