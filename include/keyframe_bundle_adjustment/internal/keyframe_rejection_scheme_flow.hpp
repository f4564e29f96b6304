// internal/keyframe_rejection_scheme_flow.hpp -- reject a frame whose pixels moved too little against the newest selected
// keyframe, e.g. while the vehicle stands still (reference: internal/keyframe_rejection_scheme_flow.hpp,
// src/keyframe_rejection_scheme_flow.cpp:17-74).  The quantity is the squared mean, not the median, of the flow over the
// (landmark, camera) pairs both frames measure; the reference keeps the name min_median_flow.  For a track user the same
// quantity comes from the store: kba_track_frame_flow (include/kba_b200.h).
#pragma once
#include "keyframe_schemes_base.hpp"

namespace keyframe_bundle_adjustment {

class KeyframeRejectionSchemeFlow : public KeyframeRejectionSchemeBase {
public:
    struct Flow {                  // what isUsable computes before its verdict
        int n_matched = 0;         // pairs of new_frame that last_keyframe also measures
        double flow_sum = 0.;      // sum of their pixel distances, in measurements_ order
        double mean_flow_sq = 0.;  // (flow_sum / n_matched)^2, NaN without a match
    };
    explicit KeyframeRejectionSchemeFlow(double min_median_flow);
    // empty last_frames: true; new_frame without measurements: false; else flow(...).mean_flow_sq > min_median_flow^2 against
    // the frame of last_frames with the largest time stamp
    bool isUsable(const Keyframe::Ptr& new_frame, const std::map<KeyframeId, Keyframe::Ptr>& last_frames) const override;
    static Flow flow(const Keyframe& new_frame, const Keyframe& last_keyframe);
    static ConstPtr createConst(double min_median_flow);
    static Ptr create(double min_median_flow);

    double min_median_flow_squared_;
};

}  // namespace keyframe_bundle_adjustment
