// TEST STUB (tests only, never shipped): the glomap stub of tests/shim_mock/glomap_stub (Image::features /
// features_undist, Frame::HasPose / RigPtr, colmap::Rig with NonRefSensors / SetSensorFromRig, Track::xyz) beside
// colmap/geometry/sim3.h of this directory, for type-checking the shim's TrackFilter, UndistortImages and
// NormalizeReconstruction in the form compiled inside a glomap build.
#pragma once
#include "../../../glomap_stub/glomap/scene/types_sfm.h"
