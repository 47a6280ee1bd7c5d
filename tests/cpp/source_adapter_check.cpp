// Compiles B200Backend with its source-output constructor argument and accessors against the stub headers and links it
// to libvp_b200.so.  Without a GPU (or with a missing checkpoint) the constructor keeps the reference's error contract:
// it throws std::runtime_error.  With argv = <scene_seg.vpw> <scene_3d.vpw> and a GPU, one 1080p frame through each
// model: the mask / depth come back at the frame's size.
#include <cstdio>
#include <memory>
#include "cv_stub.hpp"
#include "../../adapters/b200_backend.hpp"

using autoware_pov::vision::B200Backend;

int main(int argc, char** argv) {
  if (argc < 3) {
    int thrown = 0;
    try { B200Backend b("/nonexistent.vpw", "fp16", 0, VP_SCENE_SEG, true); } catch (const std::runtime_error& e) { ++thrown; std::printf("ctor threw: %s\n", e.what()); }
    try { B200Backend b("/nonexistent.vpw", "fp16", 0, VP_SCENE_3D, true); } catch (const std::runtime_error& e) { ++thrown; std::printf("ctor threw: %s\n", e.what()); }
    std::printf("SOURCE_ADAPTER_CTOR_THROWS %d\n", thrown);
    return thrown == 2 ? 0 : 1;
  }
  cv::Mat frame(1080, 1920, 0);
  for (size_t i = 0; i < frame.store.size(); ++i) frame.store[i] = static_cast<unsigned char>((i * 2654435761u) >> 24);
  B200Backend seg(argv[1], "fp16", 0, VP_SCENE_SEG, true);
  B200Backend plain(argv[1], "fp16", 0, VP_SCENE_SEG);
  B200Backend depth(argv[2], "fp16", 0, VP_SCENE_3D, true);
  if (seg.getSourceMask() || depth.getSourceDepth()) return 2;              // before the first inference
  if (!seg.doInference(frame) || !plain.doInference(frame) || !depth.doInference(frame)) return 3;
  const uint8_t* m = seg.getSourceMask();
  const float* d = depth.getSourceDepth();
  if (!m || !d || seg.getSourceDepth() || depth.getSourceMask() || plain.getSourceMask()) return 4;
  long n255 = 0;
  for (long i = 0; i < 1080L * 1920; ++i) { if (m[i] != 0 && m[i] != 255) return 5; n255 += m[i] == 255; }
  std::printf("SOURCE_ADAPTER_OK mask255=%ld depth[last]=%f\n", n255, d[1080L * 1920 - 1]);
  return 0;
}
