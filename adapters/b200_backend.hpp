// b200_backend.hpp — header-only adapter: the reference's C++ backend interface on top of the
// C-ABI of libvp_b200.so (include/vp_b200.h).
//
// Drop-in for (reference, VisionPilot/middleware_recipes/common):
//   class InferenceBackend            include/inference_backend_base.hpp:14-27  (5 pure virtuals)
//   class TensorRTBackend             include/tensorrt_backend.hpp:19-57, backends/tensorrt_backend.cpp
// selected by string at ROS2/models/src/run_model_node.cpp:39-46 and Zenoh/models/run_model.cpp:108-113
// (add a third value "b200" next to "onnxruntime" / "tensorrt", see INTEGRATION.md).
//
// Behaviour kept from TensorRTBackend:
//   * ctor (model_path, precision, gpu_id) throws std::runtime_error on failure (tensorrt_backend.cpp:16,58,117)
//   * doInference(const cv::Mat& bgr) is synchronous, returns false on failure (:179-202)
//   * getRawTensorData() throws before the first inference (:206-211); the pointer is a host buffer owned
//     by the backend and valid until the next doInference (tensorrt_backend.hpp:47)
//   * getTensorShape() = {1, C, H, W}; getModelInputHeight/Width() = 320 / 640
//   * pre-process convention P0b: cv::resize INTER_LINEAR on BGR, no channel swap, BGR-ordered ImageNet
//     stats (:160-177) — done on the GPU, bit-exact at the uint8 stage.
// `model_path` is the .vpw converted from the .pth checkpoint (python -m autoware_vision_pilot_b200.convert),
// the role the ONNX file plays for TensorRTBackend.  model kind: segmentation with 3 classes = SceneSeg,
// 1 class = DomainSeg, "depth" = Scene3D (run_model_node.cpp:29-36 `model_type`).
//
// Only needs <opencv2/core.hpp> for cv::Mat; include this header after inference_backend_base.hpp.
#pragma once
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "../include/vp_b200.h"

namespace autoware_pov::vision
{

class B200Backend : public InferenceBackend
{
public:
  // model_kind: VP_SCENE_SEG / VP_SCENE_3D / VP_DOMAIN_SEG / VP_EGO_LANES
  // source_outputs: every doInference also makes the result at the input image's own size on the GPU (the resize-back
  // run_model_node.cpp:96-104,177 does on the CPU): getSourceMask() / getSourceDepth()
  B200Backend(const std::string & model_path, const std::string & precision, int gpu_id,
              int model_kind = VP_SCENE_SEG, bool source_outputs = false)
  : source_kind_(source_outputs ? (model_kind == VP_SCENE_3D ? VP_SRC_DEPTH : VP_SRC_MASK) : 0)
  {
    vp_engine_config cfg{};
    cfg.gpu_id = gpu_id;
    // "fp16" (reference default) / "bf16": 16-bit operands, fp32 accumulate; "fp32" (tensorrt_backend.cpp:129-131 builds
    // an FP32 engine): the split-fp16 fp32-grade mode; anything else is rejected like an unknown TensorRT precision
    if (precision != "fp16" && precision != "bf16" && precision != "fp32")
      throw std::runtime_error("B200Backend: unsupported precision '" + precision + "' (fp16 | bf16 | fp32)");
    cfg.dtype = (precision == "bf16") ? VPB_BF16 : VPB_F16;
    cfg.precision = (precision == "fp32") ? VP_PREC_SPLIT : VP_PREC_16;
    cfg.resize_mode = VPB_RESIZE_CV_LINEAR;
    cfg.convention = VPB_CONV_BGR_NOSWAP;
    cfg.n_models = 1;
    cfg.kinds[0] = model_kind;
    cfg.weights[0] = model_path.c_str();
    cfg.fetch_raw = 1;
    cfg.use_graph = 1;
    cfg.source_outputs = source_kind_;
    if (vp_engine_create(&cfg, &engine_) != VPB_OK) {
      throw std::runtime_error(std::string("B200Backend: ") + vp_last_error());
    }
  }
  ~B200Backend() override { vp_engine_destroy(engine_); }
  B200Backend(const B200Backend &) = delete;
  B200Backend & operator=(const B200Backend &) = delete;

  bool doInference(const cv::Mat & input_image) override
  {
    if (input_image.empty() || input_image.channels() != 3 || input_image.depth() != 0 /*CV_8U*/) return false;
    if (vp_engine_infer(engine_, input_image.data, input_image.rows, input_image.cols,
                        static_cast<int>(input_image.step)) != VPB_OK) {
      return false;
    }
    ran_ = true;
    if (source_kind_ && vp_engine_source_output(engine_, 0, 0, source_kind_, &src_) != VPB_OK) return false;
    return vp_engine_output(engine_, 0, &out_) == VPB_OK;
  }

  const float * getRawTensorData() const override
  {
    if (!ran_) throw std::runtime_error("Inference has not been run yet. Call doInference() first.");
    return out_.raw_host;
  }
  std::vector<int64_t> getTensorShape() const override
  {
    return {1, static_cast<int64_t>(out_.channels), static_cast<int64_t>(out_.height), static_cast<int64_t>(out_.width)};
  }
  int getModelInputHeight() const override { return 320; }
  int getModelInputWidth() const override { return 640; }

  // Extension: the class / threshold map the last convolution's epilogue already produced on the GPU
  // (what createMaskKernel computes from the raw tensor, cuda_visualization_kernels.cu:13-42, after a
  // D2H+H2D round trip in the reference).  SceneSeg: class id {0,1,2}; DomainSeg: {0,1}; nullptr for depth.
  const uint8_t * getClassMap() const { return ran_ ? out_.cls_host : nullptr; }

  // Extension (constructed with source_outputs = true): the result at the input image's rows x cols, host memory owned
  // by the backend and valid until the next doInference.  getSourceMask: SceneSeg / DomainSeg mask 255 / 0 (the
  // argmax / > 0 rule, run_model_node.cpp:148-172), EgoLanes ids {0,1,2,255}, INTER_NEAREST; getSourceDepth: Scene3D
  // depth, INTER_LINEAR.  nullptr when that output was not requested or before the first inference.
  const uint8_t * getSourceMask() const
  {
    return ran_ && source_kind_ == VP_SRC_MASK ? static_cast<const uint8_t *>(src_.host) : nullptr;
  }
  const float * getSourceDepth() const
  {
    return ran_ && source_kind_ == VP_SRC_DEPTH ? static_cast<const float *>(src_.host) : nullptr;
  }

private:
  vp_engine * engine_{nullptr};
  vp_output out_{};
  int source_kind_{0};
  vp_source_output src_{};
  bool ran_{false};
};

}  // namespace autoware_pov::vision
