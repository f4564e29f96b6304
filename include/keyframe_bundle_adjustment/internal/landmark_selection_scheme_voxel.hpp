// internal/landmark_selection_scheme_voxel.hpp -- voxel-grid sparsification with near / middle / far bins (reference:
// internal/landmark_selection_scheme_voxel.hpp:22-81, src/landmark_selection_scheme_voxel.cpp:116-234).  The reference
// runs it on PCL (PassThrough, VoxelGrid<PointXYZL>) and boost::geometry (point-to-path distance); this is a
// dependency-free restatement of exactly those steps, single precision where PCL is single precision:
//   1. landmarks into the frame of the newest keyframe, as float points labelled by their position in id order;
//   2. keep z in [-20, 100];
//   3. far bin = points further than roi_far_xyz[0] from the polyline of keyframe positions;
//   4. voxel grid (leaf = voxel_size_xyz) over the rest: one point per voxel = centroid, labelled by the SMALLEST label
//      in the voxel (PCL >= 1.8 CentroidPoint: most frequent label, ties to the first in std::map order);
//   5. middle bin = voxel points further than roi_middle_xyz[0] from the path, near bin = the others;
//   6. near: largest accumulated pixel flow first, middle: random subset, far: most observations first; each bin capped.
#pragma once
#include <array>

#include "landmark_categorization_interface.hpp"
#include "landmark_selection_scheme_base.hpp"

namespace keyframe_bundle_adjustment {

class LandmarkSparsificationSchemeVoxel : public LandmarkSparsificationSchemeBase, public LandmarkCategorizatonInterface {
public:
    struct Parameters {
        Parameters() {}
        std::array<double, 3> voxel_size_xyz{{1.0, 1.0, 0.5}};    // metres
        std::array<double, 3> roi_far_xyz{{50., 50., 50.}};       // only [0] is used: distance to the trajectory
        std::array<double, 3> roi_middle_xyz{{25., 25., 25.}};    // only [0] is used
        unsigned int max_num_landmarks_near{300};
        unsigned int max_num_landmarks_middle{300};
        unsigned int max_num_landmarks_far{300};
    };
    explicit LandmarkSparsificationSchemeVoxel(Parameters p) : params_(p) { identifier = "voxel"; }
    std::set<LandmarkId> getSelection(const LandmarkMap& landmarks, const KeyframeMap& keyframes) const override;
    std::map<LandmarkId, LandmarkCategorizatonInterface::Category> getCategorizedSelection(
        const LandmarkMap& landmarks, const KeyframeMap& keyframes) const override;
    // step 6 alone: the capped ranking of the bins from the per-landmark quantities of steps 1-5 (ids_near in ascending voxel
    // index, ids_middle / ids_far ascending; flow of the near landmarks that have one, seen counts of the far ones).
    // getCategorizedSelection ends in it; LandmarkSelector feeds it the quantities the device-resident store computed.
    std::map<LandmarkId, LandmarkCategorizatonInterface::Category> rankBins(const std::vector<LandmarkId>& ids_near,
                                                                            const std::map<LandmarkId, double>& flow,
                                                                            const std::vector<LandmarkId>& ids_middle,
                                                                            const std::vector<LandmarkId>& ids_far,
                                                                            const std::map<LandmarkId, unsigned int>& seen) const;
    static ConstPtr createConst(Parameters p = Parameters()) { return ConstPtr(new LandmarkSparsificationSchemeVoxel(p)); }
    static Ptr create(Parameters p = Parameters()) { return Ptr(new LandmarkSparsificationSchemeVoxel(p)); }
    Parameters params_;
};

}  // namespace keyframe_bundle_adjustment
