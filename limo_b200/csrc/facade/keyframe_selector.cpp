// keyframe_selector.cpp -- KeyframeSelector and the three keyframe schemes limo configures (reference: src/keyframe_selector.cpp,
// src/keyframe_rejection_scheme_flow.cpp, src/keyframe_selection_scheme_pose.cpp, src/keyframe_sparsification_scheme_time.cpp).
// Host code; the reference's console messages are not restated.
#include <algorithm>
#include <cmath>

#include "keyframe_bundle_adjustment/keyframe_selector.hpp"

namespace keyframe_bundle_adjustment {

namespace {
// the frame with the largest time stamp (the first of equal ones); last_frames is not empty
const Keyframe::Ptr& newest(const std::map<KeyframeId, Keyframe::Ptr>& last_frames) {
    auto it = last_frames.cbegin();
    for (auto jt = std::next(it); jt != last_frames.cend(); ++jt)
        if (it->second->timestamp_ < jt->second->timestamp_) it = jt;
    return it->second;
}
}  // namespace

// ---- flow (keyframe_rejection_scheme_flow.cpp:17-74) ------------------------------------------------------------------------
KeyframeRejectionSchemeFlow::KeyframeRejectionSchemeFlow(double min_median_flow)
        : min_median_flow_squared_(min_median_flow * min_median_flow) {}

KeyframeRejectionSchemeFlow::Flow KeyframeRejectionSchemeFlow::flow(const Keyframe& new_frame, const Keyframe& last_keyframe) {
    Flow f;
    for (const auto& lm : new_frame.measurements_) {
        for (const auto& cm : lm.second) {
            if (!last_keyframe.hasMeasurement(lm.first, cm.first)) continue;
            const Measurement& last = last_keyframe.getMeasurement(lm.first, cm.first);
            const double dx = double(cm.second.u) - double(last.u), dy = double(cm.second.v) - double(last.v);
            f.flow_sum += std::sqrt(dx * dx + dy * dy);
            ++f.n_matched;
        }
    }
    double s = f.flow_sum;
    s /= static_cast<double>(f.n_matched);
    f.mean_flow_sq = s * s;
    return f;
}

bool KeyframeRejectionSchemeFlow::isUsable(const Keyframe::Ptr& new_frame, const std::map<KeyframeId, Keyframe::Ptr>& last_frames) const {
    if (last_frames.empty()) return true;
    if (new_frame->measurements_.empty()) return false;
    return flow(*new_frame, *newest(last_frames)).mean_flow_sq > min_median_flow_squared_;
}

KeyframeRejectionSchemeBase::ConstPtr KeyframeRejectionSchemeFlow::createConst(double min_median_flow) {
    return std::make_shared<const KeyframeRejectionSchemeFlow>(min_median_flow);
}
KeyframeRejectionSchemeBase::Ptr KeyframeRejectionSchemeFlow::create(double min_median_flow) {
    return std::make_shared<KeyframeRejectionSchemeFlow>(min_median_flow);
}

// ---- pose (keyframe_selection_scheme_pose.cpp:18-37) ------------------------------------------------------------------------
KeyframeSelectionSchemePose::KeyframeSelectionSchemePose(double critical_quaternion_difference)
        : critical_quaternion_diff_(critical_quaternion_difference) {}

bool KeyframeSelectionSchemePose::isUsable(const Keyframe::Ptr& new_frame, const std::map<KeyframeId, Keyframe::Ptr>& last_frames) const {
    if (last_frames.empty()) return false;
    return calcQuaternionDiff(new_frame->pose_, newest(last_frames)->pose_) > critical_quaternion_diff_;
}

KeyframeSelectionSchemeBase::ConstPtr KeyframeSelectionSchemePose::createConst(double critical_quaternion_difference) {
    return std::make_shared<const KeyframeSelectionSchemePose>(critical_quaternion_difference);
}
KeyframeSelectionSchemeBase::Ptr KeyframeSelectionSchemePose::create(double critical_quaternion_difference) {
    return std::make_shared<KeyframeSelectionSchemePose>(critical_quaternion_difference);
}

// ---- time (keyframe_sparsification_scheme_time.cpp:13-27) -------------------------------------------------------------------
bool KeyframeSparsificationSchemeTime::isUsable(const Keyframe::Ptr& new_frame, const std::map<KeyframeId, Keyframe::Ptr>& last_frames) const {
    if (last_frames.empty()) return true;
    const TimestampNSec max_ts = newest(last_frames)->timestamp_;
    return (new_frame->timestamp_ - max_ts) > time_difference_nano_sec_;  // unsigned: an older frame wraps
}

KeyframeSparsificationSchemeBase::ConstPtr KeyframeSparsificationSchemeTime::createConst(double time_difference_sec) {
    return std::make_shared<const KeyframeSparsificationSchemeTime>(time_difference_sec);
}
KeyframeSparsificationSchemeBase::Ptr KeyframeSparsificationSchemeTime::create(double time_difference_sec) {
    return std::make_shared<KeyframeSparsificationSchemeTime>(time_difference_sec);
}

// ---- the selector (keyframe_selector.cpp:14-133) ----------------------------------------------------------------------------
void KeyframeSelector::addScheme(KeyframeSelectionSchemeBase::ConstPtr scheme) { selection_schemes_.push_back(scheme); }
void KeyframeSelector::addScheme(KeyframeRejectionSchemeBase::ConstPtr scheme) { rejection_schemes_.push_back(scheme); }
void KeyframeSelector::addScheme(KeyframeSparsificationSchemeBase::ConstPtr scheme) { sparsification_schemes_.push_back(scheme); }

namespace {
using KeyframeMap = std::map<KeyframeId, Keyframe::Ptr>;

// the frames no scheme turns down, numbered 0, 1, ... in the order of `frames`; each frame is tested against the buffer and
// against the frames this pass accepted before it (cpp:33-56)
KeyframeMap passAll(const KeyframeSelector::Keyframes& frames, const KeyframeMap& buffer,
                    const std::vector<KeyframeSchemeBase::ConstPtr>& schemes) {
    KeyframeMap out;
    KeyframeId n = 0;
    for (const auto& frame : frames) {
        const bool turned_down = std::any_of(schemes.begin(), schemes.end(), [&](const KeyframeSchemeBase::ConstPtr& s) {
            return !s->isUsable(frame, buffer) || !s->isUsable(frame, out);
        });
        if (!turned_down) out[n++] = frame;
    }
    return out;
}

// the frames some scheme takes, against the buffer or against the frames this pass took before (cpp:66-84)
KeyframeMap passAny(const KeyframeSelector::Keyframes& frames, const KeyframeMap& buffer,
                    const std::vector<KeyframeSchemeBase::ConstPtr>& schemes) {
    KeyframeMap out;
    KeyframeId n = 0;
    for (const auto& frame : frames) {
        for (const auto& s : schemes) {
            if (s->isUsable(frame, buffer) || s->isUsable(frame, out)) {
                out[n++] = frame;
                break;
            }
        }
    }
    return out;
}

// cpp:85-104: drops the entries of `cur` whose KEY is not a key of `kept`.  The keys are each pass's own counters, so this
// compares positions, not frames.  As in the reference, the entry after an erased one is not examined: the loop advances past
// the iterator erase() returns.  When that iterator is end(), the reference's advance is undefined; here the loop stops.
void eraseRejected(KeyframeMap& cur, const KeyframeMap& kept) {
    if (kept.empty()) cur.clear();
    if (cur.empty()) return;
    for (auto it = cur.begin(); it != cur.end(); ++it) {
        if (kept.count(it->first)) continue;
        it = cur.erase(it);
        if (it == cur.end()) break;
    }
}
}  // namespace

KeyframeSelector::Keyframes KeyframeSelector::select(const Keyframes& frames, std::map<KeyframeId, Keyframe::Ptr> buffer_selected_frames) {
    const KeyframeMap kept = passAll(frames, buffer_selected_frames, rejection_schemes_);
    KeyframeMap selected = passAny(frames, buffer_selected_frames, selection_schemes_);
    eraseRejected(selected, kept);
    KeyframeMap sparse = passAll(frames, buffer_selected_frames, sparsification_schemes_);
    eraseRejected(sparse, kept);
    Keyframes out;
    for (const auto& el : selected) out.insert(el.second);
    for (const auto& el : sparse) out.insert(el.second);
    return out;
}

}  // namespace keyframe_bundle_adjustment
