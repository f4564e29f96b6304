// keyframe_selection_schemes.hpp -- every keyframe scheme of this interface (reference: keyframe_selection_schemes.hpp): the
// three that both limo nodes configure (mono_lidar.cpp:447-453, mono_standalone.cpp:327-333).
#pragma once
#include "internal/keyframe_rejection_scheme_flow.hpp"
#include "internal/keyframe_schemes_base.hpp"
#include "internal/keyframe_selection_scheme_pose.hpp"
#include "internal/keyframe_sparsification_scheme_time.hpp"
