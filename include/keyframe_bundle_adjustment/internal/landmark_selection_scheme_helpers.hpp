// internal/landmark_selection_scheme_helpers.hpp -- ranking helpers of the near / middle / far bins (reference:
// internal/landmark_selection_scheme_helpers.hpp:49-71, src/landmark_selection_scheme_helpers.cpp:14-231).
#pragma once
#include <map>
#include <vector>

#include "../keyframe.hpp"
#include "definitions.hpp"

namespace keyframe_bundle_adjustment {

namespace landmark_helpers {
// near bin: the max_num_lms ids with the largest optical flow (ids without a flow value are dropped first)
std::vector<LandmarkId> chooseNearLmIds(size_t max_num_lms, const std::vector<LandmarkId>& near_ids,
                                        const std::map<LandmarkId, double>& map_flow);
// middle bin: a random subset (std::random_shuffle of the reference, i.e. driven by std::rand())
std::vector<LandmarkId> chooseMiddleLmIds(size_t max_num, const std::vector<LandmarkId>& middle_ids);
// far bin: the ids observed from the most keyframes
std::vector<LandmarkId> chooseFarLmIds(size_t max_num, const std::vector<LandmarkId>& ids_far,
                                       const std::map<KeyframeId, Keyframe::ConstPtr>& keyframes);
// ... the same ranking from the number of keyframes observing each of them (from the device-resident store, say)
std::vector<LandmarkId> chooseFarLmIds(size_t max_num, const std::vector<LandmarkId>& ids_far,
                                       const std::map<LandmarkId, unsigned int>& seen);
// per landmark and camera: pixel flow summed (use_mean: averaged) over consecutive keyframes that both see it; the
// landmark's value is the maximum over the cameras.  Landmarks seen only once have no entry.
std::map<LandmarkId, double> calcFlow(const std::vector<LandmarkId>& landmarks,
                                      const std::vector<Keyframe::ConstPtr>& sorted_keyframes, bool use_mean = true);
std::map<LandmarkId, double> calcFlow(const std::vector<LandmarkId>& landmarks,
                                      const std::map<KeyframeId, Keyframe::ConstPtr>& keyframes, bool use_mean = true);
}  // namespace landmark_helpers

namespace keyframe_helpers {
// active keyframes, newest first (helpers.cpp:212-229)
std::vector<Keyframe::ConstPtr> getSortedKeyframes(const std::map<KeyframeId, Keyframe::ConstPtr>& keyframes);
}  // namespace keyframe_helpers

}  // namespace keyframe_bundle_adjustment
