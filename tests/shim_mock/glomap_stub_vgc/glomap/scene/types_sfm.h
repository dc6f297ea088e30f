// TEST STUB (tests only, never shipped): the glomap stub of tests/shim_mock/glomap_stub_pairs with glomap::Camera as
// glomap/scene/camera.h:12-33 declares it on top of colmap::Camera: has_refined_focal_length, Focal(), PrincipalPoint()
// and FocalLengthIdxs() (colmap returns a span of size_t), for type-checking the shim's ViewGraphCalibrator branch that is
// compiled inside a glomap build.
#pragma once
#define Camera CameraOfThePairsStub_
#include "../../../glomap_stub_pairs/glomap/scene/types_sfm.h"
#undef Camera

namespace glomap {
struct Camera : public CameraOfThePairsStub_ {
  bool has_refined_focal_length = false;
  double Focal() const { return params.empty() ? 0.0 : params[0]; }
  Eigen::Vector2d PrincipalPoint() const { return Eigen::Vector2d(); }
  std::vector<size_t> FocalLengthIdxs() const { return {0}; }
};
}  // namespace glomap
