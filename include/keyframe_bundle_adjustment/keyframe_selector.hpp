// keyframe_selector.hpp -- which of the new frames become keyframes (reference: keyframe_selector.hpp,
// src/keyframe_selector.cpp:14-133).  limo calls select({cur_frame}, getActiveKeyframePtrs()) on every frame between
// adjustPoseOnly and push (mono_lidar.cpp:219-220, mono_standalone.cpp:144-145).  Host code, as in the reference; a track user
// gets the flow scheme's quantity from the store with kba_track_frame_flow and composes the verdicts the same way.
#pragma once
#include <map>
#include <set>
#include <vector>

#include "keyframe.hpp"
#include "keyframe_selection_schemes.hpp"

namespace keyframe_bundle_adjustment {

class KeyframeSelector {
public:
    using Keyframes = std::set<Keyframe::Ptr>;

    void addScheme(KeyframeSelectionSchemeBase::ConstPtr scheme);
    void addScheme(KeyframeRejectionSchemeBase::ConstPtr scheme);
    void addScheme(KeyframeSparsificationSchemeBase::ConstPtr scheme);

    // A frame is kept when no rejection scheme rejects it and either some selection scheme selects it or no sparsification
    // scheme drops it; every test is made against buffer_selected_frames and against the frames the same pass accepted before
    // it.  The erasure that combines the passes compares the passes' own counters, not frames (see keyframe_selector.cpp).
    Keyframes select(const Keyframes& frames, std::map<KeyframeId, Keyframe::Ptr> buffer_selected_frames);

    std::vector<KeyframeSchemeBase::ConstPtr> selection_schemes_;
    std::vector<KeyframeSchemeBase::ConstPtr> rejection_schemes_;
    std::vector<KeyframeSchemeBase::ConstPtr> sparsification_schemes_;
};

}  // namespace keyframe_bundle_adjustment
