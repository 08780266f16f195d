// io::OutlierRemovingPointsProcessor (io/outlier_removing_points_processor.h/.cc) over the
// csm_outlier_remover entry points, on device 0 like the other adapter defaults: the same
// constructor, action name, Process / Flush state machine and CHECK, with the voxel map on the
// device.  Every count and kept point is bit for bit the reference's.  In a checkout this class
// replaces the processor's header and body; the pipeline builder
// (points_processor_pipeline_builder.cc) registers it by kConfigurationFileActionName and
// FromDictionary as before (INTEGRATION.md §3).
#ifndef CSM_ADAPTER_POINTS_PROCESSOR_B200_H_
#define CSM_ADAPTER_POINTS_PROCESSOR_B200_H_

#include <cstdio>
#include <cstdlib>
#include <memory>
#include <vector>

#include "../../include/csm_abi.h"

#if defined(__has_include) && __has_include("cartographer/io/points_processor.h")
#include "absl/container/flat_hash_set.h"
#include "absl/memory/memory.h"
#include "cartographer/common/lua_parameter_dictionary.h"
#include "cartographer/io/points_batch.h"
#include "cartographer/io/points_processor.h"
#define CSM_B200_IO_CHECKOUT 1
#else
#include "compat.h"
#define CSM_B200_IO_CHECKOUT 0
#endif

namespace cartographer {
namespace io {

// Passes on only the points in voxels that are not seen through too often: three passes over
// the stream count hits per voxel, then rays through voxels with hits, then filter.
class OutlierRemovingPointsProcessor : public PointsProcessor {
 public:
  constexpr static const char* kConfigurationFileActionName =
      "voxel_filter_and_remove_moving_objects";

  OutlierRemovingPointsProcessor(const double voxel_size, const double miss_per_hit_limit,
                                 PointsProcessor* const next)
      : next_(next) {
    Check(csm_outlier_remover_create(voxel_size, miss_per_hit_limit, 0, &remover_));
  }

#if CSM_B200_IO_CHECKOUT
  static std::unique_ptr<OutlierRemovingPointsProcessor> FromDictionary(
      common::LuaParameterDictionary* const dictionary, PointsProcessor* const next) {
    const double miss_per_hit_limit = dictionary->HasKey("miss_per_hit_limit")
                                          ? dictionary->GetDouble("miss_per_hit_limit")
                                          : 3.;
    return absl::make_unique<OutlierRemovingPointsProcessor>(dictionary->GetDouble("voxel_size"),
                                                             miss_per_hit_limit, next);
  }
#endif

  ~OutlierRemovingPointsProcessor() override { csm_outlier_remover_destroy(remover_); }

  OutlierRemovingPointsProcessor(const OutlierRemovingPointsProcessor&) = delete;
  OutlierRemovingPointsProcessor& operator=(const OutlierRemovingPointsProcessor&) = delete;

  void Process(std::unique_ptr<PointsBatch> batch) override {
    const int32_t n = static_cast<int32_t>(batch->points.size());
    std::vector<float> xyz;
    xyz.reserve(3 * static_cast<size_t>(n));
    for (const auto& p : batch->points) {
      xyz.push_back(p.position.x());
      xyz.push_back(p.position.y());
      xyz.push_back(p.position.z());
    }
    const float* batches[1] = {xyz.data()};
    switch (state_) {
      case State::kPhase1:
        Check(csm_outlier_remover_add_hits(remover_, batches, &n, 1, nullptr));
        break;
      case State::kPhase2: {
        const float origin[3] = {batch->origin.x(), batch->origin.y(), batch->origin.z()};
        Check(csm_outlier_remover_count_rays(remover_, origin, batches, &n, 1, nullptr));
        break;
      }
      case State::kPhase3: {
        std::vector<int32_t> kept(n > 0 ? n : 1);
        int32_t num_kept = 0;
        Check(csm_outlier_remover_filter(remover_, batches, &n, 1, kept.data(), &num_kept,
                                         nullptr));
        absl::flat_hash_set<int> to_remove;
        for (int32_t i = 0, j = 0; i < n; ++i) {
          if (j < num_kept && kept[j] == i) {
            ++j;
          } else {
            to_remove.insert(i);
          }
        }
        RemovePoints(to_remove, batch.get());
        next_->Process(std::move(batch));
        break;
      }
    }
  }

  FlushResult Flush() override {
    switch (state_) {
      case State::kPhase1:
        state_ = State::kPhase2;
        return FlushResult::kRestartStream;
      case State::kPhase2:
        state_ = State::kPhase3;
        return FlushResult::kRestartStream;
      case State::kPhase3:
        if (next_->Flush() != FlushResult::kFinished) {
          std::fprintf(stderr,
                       "Voxel filtering and outlier removal must be configured to occur after "
                       "any stages that require multiple passes.\n");
          std::abort();
        }
        return FlushResult::kFinished;
    }
    std::abort();
  }

 private:
  enum class State { kPhase1, kPhase2, kPhase3 };

  // Refusals and CUDA failures keep the reference's CHECK semantics (abort with the message).
  static void Check(csm_status s) {
    if (s != CSM_OK) {
      std::fprintf(stderr, "libcsm_b200: %s\n", csm_last_error_string());
      std::abort();
    }
  }

  PointsProcessor* const next_;
  State state_ = State::kPhase1;
  csm_outlier_remover* remover_ = nullptr;
};

}  // namespace io
}  // namespace cartographer

#endif  // CSM_ADAPTER_POINTS_PROCESSOR_B200_H_
