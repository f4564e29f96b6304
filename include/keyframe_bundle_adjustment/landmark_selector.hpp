// landmark_selector.hpp -- chains the landmark schemes in front of solve() (reference: keyframe_bundle_adjustment/include/
// keyframe_bundle_adjustment/landmark_selector.hpp:40-345): outliers out, rejection schemes narrow the set, selection
// schemes name landmarks that are taken in any case, sparsification schemes thin out the rest; landmarks that were not
// selected age in a counter that forgets after 10 s.
#pragma once
#include <cstdint>
#include <map>
#include <memory>
#include <set>
#include <vector>

#include "internal/landmark_categorization_interface.hpp"
#include "keyframe.hpp"
#include "landmark_selection_schemes.hpp"

namespace keyframe_bundle_adjustment {

class LandmarkSelector {
public:
    EIGEN_MAKE_ALIGNED_OPERATOR_NEW
    LandmarkSelector() = default;
    virtual ~LandmarkSelector() = default;

    void addScheme(LandmarkSelectionSchemeBase::ConstPtr scheme) { selection_schemes_.push_back(scheme); }
    void addScheme(LandmarkSparsificationSchemeBase::ConstPtr scheme) { sparsification_schemes_.push_back(scheme); }
    void addScheme(LandmarkRejectionSchemeBase::ConstPtr scheme) { rejection_schemes_.push_back(scheme); }

    // landmark_selector.hpp:118-253
    std::set<LandmarkId> select(const std::map<LandmarkId, Landmark::ConstPtr>& landmarks,
                                const std::map<KeyframeId, Keyframe::ConstPtr>& kfs);

    // Not in the reference: the per-landmark quantities of the cheirality + voxel chain, computed outside the selector
    // (kba_track_select_landmarks on the device-resident store, include/kba_b200.h).  candidates: the landmarks given to select()
    // minus the outliers, ascending id; the other vectors by candidate, as kba_select_out describes them.
    struct ChainQuantities {
        std::vector<LandmarkId> candidates;
        std::vector<uint8_t> cheiral;
        std::vector<int8_t> bin;
        std::vector<int32_t> near_order;  // the near bin, candidate indices in ascending voxel index
        std::vector<double> flow;         // NaN: no flow value
        std::vector<int32_t> seen;
    };
    // The voxel scheme of a chain such quantities stand for -- exactly one rejection scheme, the cheirality one, exactly one
    // sparsification scheme, the voxel one, and any selection schemes (they run on the host over the cheirality survivors) --
    // or nullptr for any other chain.
    const LandmarkSparsificationSchemeVoxel* quantitiesChainVoxel() const;
    // select() with q in place of the chain's own loops over keyframes and measurements: the ranking (std::rand included), the
    // categories, the aging of unselected landmarks and the result are those of select(landmarks, kfs) on the same state.
    // Throws std::invalid_argument if the chain is not one quantitiesChainVoxel() accepts or q.candidates are not the candidates.
    std::set<LandmarkId> select(const std::map<LandmarkId, Landmark::ConstPtr>& landmarks,
                                const std::map<KeyframeId, Keyframe::ConstPtr>& kfs, const ChainQuantities& q);

    void markUnselected(LandmarkId lm_id, TimestampNSec last_time_seen) {
        unselected_lms_[lm_id] += 1;
        last_time_seen_[lm_id] = last_time_seen;
    }
    void clean(TimestampNSec oldest_ts);  // forget counters of landmarks last unselected before oldest_ts
    const std::map<LandmarkId, unsigned int>& getUnselectedLandmarks() const { return unselected_lms_; }
    // categories of the last scheme that implements LandmarkCategorizatonInterface (empty if none ran)
    const std::map<LandmarkId, LandmarkCategorizatonInterface::Category>& getLandmarkCategories() const { return landmark_categories_; }
    std::set<LandmarkId> getLastSelection() const { return last_selected_lms_; }
    void clearOutliers() { outlier_ids_.clear(); }
    const std::set<LandmarkId>& getOutliers() const { return outlier_ids_; }
    void setOutlier(LandmarkId id) { outlier_ids_.insert(id); }
    void setOutlier(const std::set<LandmarkId>& ids) { for (const auto& el : ids) setOutlier(el); }

    std::vector<LandmarkSelectionSchemeBase::ConstPtr> selection_schemes_;
    std::vector<LandmarkSparsificationSchemeBase::ConstPtr> sparsification_schemes_;
    std::vector<LandmarkRejectionSchemeBase::ConstPtr> rejection_schemes_;
    std::set<LandmarkId> outlier_ids_;

private:
    std::set<LandmarkId> selectImpl(const std::map<LandmarkId, Landmark::ConstPtr>& landmarks,
                                    const std::map<KeyframeId, Keyframe::ConstPtr>& kfs, const ChainQuantities* q);
    std::set<LandmarkId> runScheme(const LandmarkSchemeBase& scheme, const std::map<LandmarkId, Landmark::ConstPtr>& lms,
                                   const std::map<KeyframeId, Keyframe::ConstPtr>& kfs);
    std::map<LandmarkId, unsigned int> unselected_lms_;
    std::map<LandmarkId, TimestampNSec> last_time_seen_;
    std::set<LandmarkId> last_selected_lms_;
    std::map<LandmarkId, LandmarkCategorizatonInterface::Category> landmark_categories_;
};

}  // namespace keyframe_bundle_adjustment
