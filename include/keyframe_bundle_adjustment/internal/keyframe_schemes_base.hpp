// internal/keyframe_schemes_base.hpp -- the three kinds of keyframe schemes KeyframeSelector composes (reference:
// internal/keyframe_schemes_base.hpp): rejection (a frame that would make the estimate unstable), selection (a frame the
// estimate needs) and sparsification (a frame that adds little).  A scheme judges one new frame against a map of frames
// selected before it.
#pragma once
#include <map>
#include <memory>

#include "../keyframe.hpp"
#include "definitions.hpp"

namespace keyframe_bundle_adjustment {

class KeyframeSchemeBase {
public:
    using Ptr = std::shared_ptr<KeyframeSchemeBase>;
    using ConstPtr = std::shared_ptr<const KeyframeSchemeBase>;
    virtual ~KeyframeSchemeBase() = default;
    // true: the scheme accepts new_frame given the frames in last_selected_keyframes
    virtual bool isUsable(const Keyframe::Ptr& new_frame, const std::map<KeyframeId, Keyframe::Ptr>& last_selected_keyframes) const = 0;
};
class KeyframeSelectionSchemeBase : public KeyframeSchemeBase {
public:
    using Ptr = std::shared_ptr<KeyframeSelectionSchemeBase>;
    using ConstPtr = std::shared_ptr<const KeyframeSelectionSchemeBase>;
};
class KeyframeRejectionSchemeBase : public KeyframeSchemeBase {
public:
    using Ptr = std::shared_ptr<KeyframeRejectionSchemeBase>;
    using ConstPtr = std::shared_ptr<const KeyframeRejectionSchemeBase>;
};
class KeyframeSparsificationSchemeBase : public KeyframeSchemeBase {
public:
    using Ptr = std::shared_ptr<KeyframeSparsificationSchemeBase>;
    using ConstPtr = std::shared_ptr<const KeyframeSparsificationSchemeBase>;
};

}  // namespace keyframe_bundle_adjustment
