// internal/keyframe_selection_scheme_pose.hpp -- select a frame whose rotation differs enough from the newest selected
// keyframe's, so that curves keep enough keyframes (reference: internal/keyframe_selection_scheme_pose.hpp,
// src/keyframe_selection_scheme_pose.cpp:18-37).
#pragma once
#include "keyframe_schemes_base.hpp"

namespace keyframe_bundle_adjustment {

class KeyframeSelectionSchemePose : public KeyframeSelectionSchemeBase {
public:
    explicit KeyframeSelectionSchemePose(double critical_quaternion_difference);
    // empty last_frames: false (an empty buffer would otherwise take every frame); else calcQuaternionDiff(new, newest) > critical
    bool isUsable(const Keyframe::Ptr& new_frame, const std::map<KeyframeId, Keyframe::Ptr>& last_frames) const override;
    static ConstPtr createConst(double critical_quaternion_difference);
    static Ptr create(double critical_quaternion_difference);

private:
    double critical_quaternion_diff_;
};

}  // namespace keyframe_bundle_adjustment
