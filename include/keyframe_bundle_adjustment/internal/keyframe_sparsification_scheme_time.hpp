// internal/keyframe_sparsification_scheme_time.hpp -- keep a frame only when enough time has passed since the newest selected
// keyframe (reference: internal/keyframe_sparsification_scheme_time.hpp, src/keyframe_sparsification_scheme_time.cpp:13-27).
#pragma once
#include "keyframe_schemes_base.hpp"

namespace keyframe_bundle_adjustment {

class KeyframeSparsificationSchemeTime : public KeyframeSparsificationSchemeBase {
public:
    using DurationNSec = unsigned long;
    // the threshold is convert(time_difference_sec): ts * 1e9, truncated
    explicit KeyframeSparsificationSchemeTime(double time_difference_sec) : time_difference_nano_sec_(convert(time_difference_sec)) {}
    // empty last_frames: true; else new.timestamp_ - newest.timestamp_ > threshold in unsigned 64-bit arithmetic, so a frame
    // older than the newest one wraps around and is usable
    bool isUsable(const Keyframe::Ptr& new_frame, const std::map<KeyframeId, Keyframe::Ptr>& last_frames) const override;
    static ConstPtr createConst(double time_difference_sec);
    static Ptr create(double time_difference_sec);

    DurationNSec time_difference_nano_sec_;
};

}  // namespace keyframe_bundle_adjustment
