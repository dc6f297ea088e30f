// TEST STUB (tests only, never shipped): the glomap stub of tests/shim_mock/glomap_stub_vgc with glomap::Frame carrying
// cluster_id as glomap/scene/frame.h:35 declares it, for type-checking the shim's PruneWeaklyConnectedImages branch that
// is compiled inside a glomap build.
#pragma once
#define Frame FrameOfTheVgcStub_
#include "../../../glomap_stub_vgc/glomap/scene/types_sfm.h"
#undef Frame

namespace glomap {
struct Frame : public FrameOfTheVgcStub_ {
  int cluster_id = -1;
};
}  // namespace glomap
