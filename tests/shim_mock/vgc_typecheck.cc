// TEST (tests only): the shim's ViewGraphCalibrator in its -DB200SFM_WITH_GLOMAP form, instantiated with the glomap types
// of tests/shim_mock/glomap_stub_vgc -- compiled with -fsyntax-only by tests/test_view_graph_calibration_cpu.py.
#include "estimators_shim.h"

bool Run(glomap::ViewGraph& vg, std::unordered_map<glomap::camera_t, glomap::Camera>& cameras,
         std::unordered_map<glomap::image_t, glomap::Image>& images) {
  b200sfm_shim::ViewGraphCalibratorOptions options;
  b200sfm_shim::ViewGraphCalibrator calibrator(options);
  return calibrator.Solve(vg, cameras, images);
}
