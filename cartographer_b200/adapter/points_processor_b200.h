// io::OutlierRemovingPointsProcessor (io/outlier_removing_points_processor.h/.cc) over the
// csm_outlier_remover entry points, io::XRayPointsProcessor (io/xray_points_processor.h/.cc)
// over the csm_xray entry points, and the map writers io::ProbabilityGridPointsProcessor
// (io/probability_grid_points_processor.h/.cc) and io::HybridGridPointsProcessor
// (io/hybrid_grid_points_processor.h/.cc) over the device grids and range data inserters, on
// device 0 like the other adapter defaults: the same constructors, action names, Process / Flush
// and CHECKs, with the voxel maps and grids on the device.  Every count, kept point, pixel and
// serialised byte is bit for bit the reference's.  In a checkout these classes replace the
// processors' headers and bodies; the pipeline builder
// (points_processor_pipeline_builder.cc) registers them by kConfigurationFileActionName and
// FromDictionary as before (INTEGRATION.md §3).
#ifndef CSM_ADAPTER_POINTS_PROCESSOR_B200_H_
#define CSM_ADAPTER_POINTS_PROCESSOR_B200_H_

#include <cstdio>
#include <cstdlib>
#include <memory>
#include <string>
#include <vector>

#include "../../include/csm_abi.h"

#if defined(__has_include) && __has_include("cartographer/io/points_processor.h")
#include "absl/container/flat_hash_set.h"
#include "absl/memory/memory.h"
#include "cartographer/common/lua_parameter_dictionary.h"
#include "cartographer/io/points_batch.h"
#include "cartographer/io/points_processor.h"
#include "absl/strings/str_cat.h"
#include "cartographer/common/math.h"
#include "cartographer/io/color.h"
#include "cartographer/io/draw_trajectories.h"
#include "cartographer/io/file_writer.h"
#include "cartographer/io/image.h"
#include "cartographer/mapping/2d/map_limits.h"
#include "cartographer/mapping/2d/probability_grid_range_data_inserter_2d.h"
#include "cartographer/mapping/3d/range_data_inserter_3d.h"
#include "cartographer/mapping/detect_floors.h"
#include "cartographer/mapping/proto/trajectory.pb.h"
#include "cartographer/transform/rigid_transform.h"
#include "cartographer/transform/transform.h"
#include "glog/logging.h"
#define CSM_B200_IO_CHECKOUT 1
#else
#include "compat.h"
#define CSM_B200_IO_CHECKOUT 0
#endif
#include "scan_matchers_b200.h"

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

// Creates X-ray cuts through the points with pixels being 'voxel_size' big: per floor (or one)
// aggregation the voxels and column colour sums live on the device, and Flush draws each image
// there.
class XRayPointsProcessor : public PointsProcessor {
 public:
  constexpr static const char* kConfigurationFileActionName = "write_xray_image";
  enum class DrawTrajectories { kNo, kYes };

  XRayPointsProcessor(double voxel_size, double saturation_factor,
                      const transform::Rigid3f& transform,
                      const std::vector<mapping::Floor>& floors,
                      const DrawTrajectories& draw_trajectories,
                      const std::string& output_filename,
                      const std::vector<mapping::proto::Trajectory>& trajectories,
                      FileWriterFactory file_writer_factory, PointsProcessor* const next)
      : draw_trajectories_(draw_trajectories),
        trajectories_(trajectories),
        file_writer_factory_(file_writer_factory),
        next_(next),
        floors_(floors),
        output_filename_(output_filename),
        transform_(transform),
        resolution_(static_cast<float>(voxel_size)) {
    const float t[7] = {transform.translation().x(), transform.translation().y(),
                        transform.translation().z(), transform.rotation().w(),
                        transform.rotation().x(),    transform.rotation().y(),
                        transform.rotation().z()};
    const int32_t num_aggregations = floors_.empty() ? 1 : static_cast<int32_t>(floors_.size());
    Check(csm_xray_create(voxel_size, saturation_factor, t, num_aggregations, 0, &xray_));
  }

#if CSM_B200_IO_CHECKOUT
  static std::unique_ptr<XRayPointsProcessor> FromDictionary(
      const std::vector<mapping::proto::Trajectory>& trajectories,
      FileWriterFactory file_writer_factory, common::LuaParameterDictionary* const dictionary,
      PointsProcessor* const next) {
    std::vector<mapping::Floor> floors;
    const bool separate_floor =
        dictionary->HasKey("separate_floors") && dictionary->GetBool("separate_floors");
    const auto draw_trajectories =
        (!dictionary->HasKey("draw_trajectories") || dictionary->GetBool("draw_trajectories"))
            ? DrawTrajectories::kYes
            : DrawTrajectories::kNo;
    const double saturation_factor =
        dictionary->HasKey("saturation_factor") ? dictionary->GetDouble("saturation_factor") : 1.;
    if (separate_floor) {
      CHECK_EQ(trajectories.size(), 1) << "Can only detect floors with a single trajectory.";
      floors = mapping::DetectFloors(trajectories.at(0));
    }
    return absl::make_unique<XRayPointsProcessor>(
        dictionary->GetDouble("voxel_size"), saturation_factor,
        transform::FromDictionary(dictionary->GetDictionary("transform").get()).cast<float>(),
        floors, draw_trajectories, dictionary->GetString("filename"), trajectories,
        file_writer_factory, next);
  }
#endif

  ~XRayPointsProcessor() override { csm_xray_destroy(xray_); }

  XRayPointsProcessor(const XRayPointsProcessor&) = delete;
  XRayPointsProcessor& operator=(const XRayPointsProcessor&) = delete;

  void Process(std::unique_ptr<PointsBatch> batch) override {
    if (floors_.empty()) {
      Insert(*batch, 0);
    } else {
      for (size_t i = 0; i < floors_.size(); ++i) {
        if (!ContainedIn(batch->start_time, floors_[i].timespans)) continue;
        Insert(*batch, static_cast<int32_t>(i));
      }
    }
    next_->Process(std::move(batch));
  }

  FlushResult Flush() override {
    if (floors_.empty()) {
      WriteVoxels(0, file_writer_factory_(output_filename_ + ".png").get());
    } else {
      for (size_t i = 0; i < floors_.size(); ++i) {
        WriteVoxels(static_cast<int32_t>(i),
                    file_writer_factory_(output_filename_ + std::to_string(i) + ".png").get());
      }
    }
    switch (next_->Flush()) {
      case FlushResult::kRestartStream:
        std::fprintf(stderr,
                     "X-Ray generation must be configured to occur after any stages that "
                     "require multiple passes.\n");
        std::abort();
      case FlushResult::kFinished:
        return FlushResult::kFinished;
    }
    std::abort();
  }

  // The shared box of cell indices as {empty, min, max} (the reference returns an
  // Eigen::AlignedBox3i, empty until the first point).
  struct Box {
    bool empty;
    int32_t min[3], max[3];
  };
  Box bounding_box() const {
    Box box;
    int32_t empty = 0;
    Check(csm_xray_bounding_box(xray_, box.min, box.max, &empty));
    box.empty = empty != 0;
    return box;
  }

 private:
  static bool ContainedIn(const common::Time& time,
                          const std::vector<mapping::Timespan>& timespans) {
    for (const mapping::Timespan& timespan : timespans) {
      if (timespan.start <= time && time <= timespan.end) return true;
    }
    return false;
  }

  void Insert(const PointsBatch& batch, int32_t aggregation) {
    const int32_t n = static_cast<int32_t>(batch.points.size());
    std::vector<float> xyz, rgb;
    xyz.reserve(3 * static_cast<size_t>(n));
    for (const auto& p : batch.points) {
      xyz.push_back(p.position.x());
      xyz.push_back(p.position.y());
      xyz.push_back(p.position.z());
    }
    for (size_t i = 0; i < batch.colors.size(); ++i) {
      for (int c = 0; c < 3; ++c) rgb.push_back(batch.colors.at(i)[c]);
    }
    const float* points[1] = {xyz.data()};
    const float* colors[1] = {batch.colors.empty() ? nullptr : rgb.data()};
    Check(csm_xray_insert(xray_, aggregation, points, colors, &n, 1, nullptr));
  }

  void WriteVoxels(int32_t aggregation, FileWriter* const file_writer) {
    int32_t width = 0, height = 0;
    Check(csm_xray_draw(xray_, aggregation, nullptr, 0, &width, &height, nullptr));
    if (width == 0) {
      std::fprintf(stderr, "Not writing output: bounding box is empty.\n");
      return;
    }
    std::vector<uint32_t> pixels(static_cast<size_t>(width) * height);
    Check(csm_xray_draw(xray_, aggregation, pixels.data(), static_cast<int64_t>(pixels.size()),
                        &width, &height, nullptr));
    Image image(width, height);
    for (int y = 0; y < height; ++y) {
      for (int x = 0; x < width; ++x) {
        const uint32_t word = pixels[static_cast<size_t>(y) * width + x];
        image.SetPixel(x, y, {{static_cast<uint8_t>(word >> 16), static_cast<uint8_t>(word >> 8),
                               static_cast<uint8_t>(word)}});
      }
    }
#if CSM_B200_IO_CHECKOUT
    if (draw_trajectories_ == DrawTrajectories::kYes) {
      const Box box = bounding_box();
      // voxel_index_to_pixel of the cell of the pose's transformed translation
      const auto pose_to_pixel = [&box, this](const transform::Rigid3d& pose) -> Eigen::Array2i {
        const Eigen::Vector3f p = (transform_ * pose.cast<float>()).translation();
        return Eigen::Array2i(box.max[1] - common::RoundToInt(p.y() / resolution_),
                              box.max[2] - common::RoundToInt(p.z() / resolution_));
      };
      for (size_t i = 0; i < trajectories_.size(); ++i) {
        DrawTrajectory(trajectories_[i], GetColor(i), pose_to_pixel,
                       image.GetCairoSurface().get());
      }
    }
#endif
    image.WritePng(file_writer);
    if (!file_writer->Close()) {
      std::fprintf(stderr, "Check failed: file_writer->Close()\n");
      std::abort();
    }
  }

  // Refusals and CUDA failures keep the reference's CHECK semantics (abort with the message).
  static void Check(csm_status s) {
    if (s != CSM_OK) {
      std::fprintf(stderr, "libcsm_b200: %s\n", csm_last_error_string());
      std::abort();
    }
  }

  const DrawTrajectories draw_trajectories_;
  const std::vector<mapping::proto::Trajectory> trajectories_;
  FileWriterFactory file_writer_factory_;
  PointsProcessor* const next_;
  // If empty, we do not separate into floors.
  const std::vector<mapping::Floor> floors_;
  const std::string output_filename_;
  const transform::Rigid3f transform_;
  const float resolution_;
  csm_xray* xray_ = nullptr;
};

namespace points_processor_b200_internal {
// Refusals and CUDA failures keep the reference's CHECK semantics (abort with the message).
inline void Check(csm_status s) {
  if (s != CSM_OK) {
    std::fprintf(stderr, "libcsm_b200: %s\n", csm_last_error_string());
    std::abort();
  }
}
inline void CheckClose(FileWriter* const file_writer) {
  if (!file_writer->Close()) {
    std::fprintf(stderr, "Check failed: file_writer->Close()\n");
    std::abort();
  }
}
// A batch's points as n x {x, y, z}.
inline std::vector<float> Flatten(const PointsBatch& batch) {
  std::vector<float> xyz;
  xyz.reserve(3 * batch.points.size());
  for (const auto& p : batch.points) {
    xyz.push_back(p.position.x());
    xyz.push_back(p.position.y());
    xyz.push_back(p.position.z());
  }
  return xyz;
}
}  // namespace points_processor_b200_internal

// Draws the device grid into an image (csm_rt_grid2d_draw) and fills in 'offset' with the
// cropped map limits.  A grid without known cells draws one unknown pixel at offset (0, 0), as
// the reference's ComputeCroppedLimits gives 1 x 1 cells there, so this never returns nullptr.
inline std::unique_ptr<Image> DrawProbabilityGrid(
    const mapping::scan_matching::DeviceGrid2D& probability_grid, Eigen::Array2i* offset) {
  using points_processor_b200_internal::Check;
  int32_t width = 0, height = 0, cropped_offset[2] = {0, 0};
  Check(csm_rt_grid2d_draw(probability_grid.handle(), nullptr, 0, &width, &height,
                           cropped_offset, nullptr));
  std::vector<uint32_t> pixels(static_cast<size_t>(width) * height);
  Check(csm_rt_grid2d_draw(probability_grid.handle(), pixels.data(),
                           static_cast<int64_t>(pixels.size()), &width, &height, cropped_offset,
                           nullptr));
  *offset = Eigen::Array2i(cropped_offset[0], cropped_offset[1]);
  std::unique_ptr<Image> image(new Image(width, height));
  for (int y = 0; y < height; ++y) {
    for (int x = 0; x < width; ++x) {
      const uint8_t value = static_cast<uint8_t>(pixels[static_cast<size_t>(y) * width + x]);
      image->SetPixel(x, y, {{value, value, value}});
    }
  }
  return image;
}

// An initially empty probability grid with 'resolution' and a small size (100 x 100 cells,
// max = 0.5 * 100 * resolution on both axes), suitable for a PointsBatchProcessor, on the device.
inline std::unique_ptr<mapping::scan_matching::DeviceGrid2D> CreateProbabilityGrid(
    const double resolution, const int device = 0) {
  constexpr int kInitialProbabilityGridSize = 100;
  const double max = 0.5 * kInitialProbabilityGridSize * resolution;
#if CSM_B200_IO_CHECKOUT
  const mapping::MapLimits limits(
      resolution, Eigen::Vector2d(max, max),
      mapping::CellLimits(kInitialProbabilityGridSize, kInitialProbabilityGridSize));
#else
  const mapping::MapLimits limits(
      resolution, max, max,
      mapping::CellLimits{kInitialProbabilityGridSize, kInitialProbabilityGridSize});
#endif
  return std::unique_ptr<mapping::scan_matching::DeviceGrid2D>(
      new mapping::scan_matching::DeviceGrid2D(limits, device));
}

// Creates a probability grid with the specified 'resolution' on the device.  As all points are
// projected into the x-y plane the z component of the data is ignored.  The grid refuses (and
// the processor CHECK-fails) an insert that would grow it to 30 000 cells per axis.
class ProbabilityGridPointsProcessor : public PointsProcessor {
 public:
  constexpr static const char* kConfigurationFileActionName = "write_probability_grid";
  enum class DrawTrajectories { kNo, kYes };
  enum class OutputType { kPng, kPb };

  ProbabilityGridPointsProcessor(
      double resolution,
      const mapping::proto::ProbabilityGridRangeDataInserterOptions2D&
          probability_grid_range_data_inserter_options,
      const DrawTrajectories& draw_trajectories, const OutputType& output_type,
      std::unique_ptr<FileWriter> file_writer,
      const std::vector<mapping::proto::Trajectory>& trajectories, PointsProcessor* next)
      : draw_trajectories_(draw_trajectories),
        output_type_(output_type),
        trajectories_(trajectories),
        file_writer_(std::move(file_writer)),
        next_(next),
        probability_grid_(CreateProbabilityGrid(resolution)) {
    csm_range_inserter_options2d o{};
    o.hit_probability = probability_grid_range_data_inserter_options.hit_probability();
    o.miss_probability = probability_grid_range_data_inserter_options.miss_probability();
    o.insert_free_space =
        probability_grid_range_data_inserter_options.insert_free_space() ? 1 : 0;
    points_processor_b200_internal::Check(csm_range_inserter2d_create(&o, 0, &inserter_));
    if (output_type == OutputType::kPb && draw_trajectories_ == DrawTrajectories::kYes) {
      std::fprintf(stderr,
                   "Drawing the trajectories is not supported when writing the probability "
                   "grid as protobuf.\n");
    }
  }

#if CSM_B200_IO_CHECKOUT
  static std::unique_ptr<ProbabilityGridPointsProcessor> FromDictionary(
      const std::vector<mapping::proto::Trajectory>& trajectories,
      const FileWriterFactory& file_writer_factory,
      common::LuaParameterDictionary* const dictionary, PointsProcessor* const next) {
    const auto draw_trajectories =
        (!dictionary->HasKey("draw_trajectories") || dictionary->GetBool("draw_trajectories"))
            ? DrawTrajectories::kYes
            : DrawTrajectories::kNo;
    OutputType output_type = OutputType::kPng;
    if (dictionary->HasKey("output_type")) {
      const std::string name = dictionary->GetString("output_type");
      if (name == "pb") {
        output_type = OutputType::kPb;
      } else if (name != "png") {
        LOG(FATAL) << "OutputType " << name << " does not exist!";
      }
    }
    return absl::make_unique<ProbabilityGridPointsProcessor>(
        dictionary->GetDouble("resolution"),
        mapping::CreateProbabilityGridRangeDataInserterOptions2D(
            dictionary->GetDictionary("range_data_inserter").get()),
        draw_trajectories, output_type,
        file_writer_factory(dictionary->GetString("filename") +
                            (output_type == OutputType::kPng ? ".png" : ".pb")),
        trajectories, next);
  }
#endif

  ~ProbabilityGridPointsProcessor() override { csm_range_inserter2d_destroy(inserter_); }

  ProbabilityGridPointsProcessor(const ProbabilityGridPointsProcessor&) = delete;
  ProbabilityGridPointsProcessor& operator=(const ProbabilityGridPointsProcessor&) = delete;

  void Process(std::unique_ptr<PointsBatch> batch) override {
    // range_data_inserter_.Insert({batch->origin, sensor::PointCloud(batch->points), {}}, ...)
    const std::vector<float> returns = points_processor_b200_internal::Flatten(*batch);
    const float origin[3] = {batch->origin.x(), batch->origin.y(), batch->origin.z()};
    points_processor_b200_internal::Check(csm_range_inserter2d_insert(
        inserter_, origin, returns.data(), static_cast<int32_t>(batch->points.size()), nullptr,
        0, probability_grid_->mutable_handle(), nullptr));
    next_->Process(std::move(batch));
  }

  FlushResult Flush() override {
    if (output_type_ == OutputType::kPng) {
      Eigen::Array2i offset;
      std::unique_ptr<Image> image = DrawProbabilityGrid(*probability_grid_, &offset);
#if CSM_B200_IO_CHECKOUT
      if (draw_trajectories_ == DrawTrajectories::kYes) {
        double resolution = 0., max_x = 0., max_y = 0.;
        int32_t num_x_cells = 0, num_y_cells = 0;
        points_processor_b200_internal::Check(csm_rt_grid2d_limits(
            probability_grid_->handle(), &resolution, &max_x, &max_y, &num_x_cells,
            &num_y_cells));
        const mapping::MapLimits limits(resolution, Eigen::Vector2d(max_x, max_y),
                                        mapping::CellLimits(num_x_cells, num_y_cells));
        for (size_t i = 0; i < trajectories_.size(); ++i) {
          DrawTrajectory(
              trajectories_[i], GetColor(i),
              [&limits, &offset](const transform::Rigid3d& pose) -> Eigen::Array2i {
                return limits.GetCellIndex(pose.cast<float>().translation().head<2>()) - offset;
              },
              image->GetCairoSurface().get());
        }
      }
#endif
      image->WritePng(file_writer_.get());
    } else {
      const std::string serialized = mapping::scan_matching::b200_internal::Serialize(
          csm_rt_grid2d_to_proto, probability_grid_->handle());
      file_writer_->Write(serialized.data(), serialized.size());
    }
    points_processor_b200_internal::CheckClose(file_writer_.get());
    switch (next_->Flush()) {
      case FlushResult::kRestartStream:
        std::fprintf(stderr,
                     "ProbabilityGrid generation must be configured to occur after any stages "
                     "that require multiple passes.\n");
        std::abort();
      case FlushResult::kFinished:
        return FlushResult::kFinished;
    }
    std::abort();
  }

  // The device grid the batches went into.
  const mapping::scan_matching::DeviceGrid2D& probability_grid() const {
    return *probability_grid_;
  }

 private:
  const DrawTrajectories draw_trajectories_;
  const OutputType output_type_;
  const std::vector<mapping::proto::Trajectory> trajectories_;
  std::unique_ptr<FileWriter> file_writer_;
  PointsProcessor* const next_;
  csm_range_inserter2d* inserter_ = nullptr;
  std::unique_ptr<mapping::scan_matching::DeviceGrid2D> probability_grid_;
};

// Creates a hybrid grid of the points with voxels being 'voxel_size' big, on the device (the
// dense csm_grid3d box: a cell outside [-8192, 8192)^3, or a box the device cannot hold,
// CHECK-fails).  'range_data_inserter' options configure the ray tracing through the grid.
class HybridGridPointsProcessor : public PointsProcessor {
 public:
  constexpr static const char* kConfigurationFileActionName = "write_hybrid_grid";

  HybridGridPointsProcessor(
      double voxel_size, const mapping::proto::RangeDataInserterOptions3D& range_data_inserter_options,
      std::unique_ptr<FileWriter> file_writer, PointsProcessor* next)
      : next_(next),
        hybrid_grid_(static_cast<float>(voxel_size), 0),
        file_writer_(std::move(file_writer)) {
    csm_range_inserter_options3d o{};
    o.hit_probability = range_data_inserter_options.hit_probability();
    o.miss_probability = range_data_inserter_options.miss_probability();
    o.num_free_space_voxels = range_data_inserter_options.num_free_space_voxels();
    o.intensity_threshold = range_data_inserter_options.intensity_threshold();
    points_processor_b200_internal::Check(csm_range_inserter3d_create(&o, 0, &inserter_));
  }

#if CSM_B200_IO_CHECKOUT
  static std::unique_ptr<HybridGridPointsProcessor> FromDictionary(
      const FileWriterFactory& file_writer_factory,
      common::LuaParameterDictionary* const dictionary, PointsProcessor* const next) {
    return absl::make_unique<HybridGridPointsProcessor>(
        dictionary->GetDouble("voxel_size"),
        mapping::CreateRangeDataInserterOptions3D(
            dictionary->GetDictionary("range_data_inserter").get()),
        file_writer_factory(dictionary->GetString("filename")), next);
  }
#endif

  ~HybridGridPointsProcessor() override { csm_range_inserter3d_destroy(inserter_); }

  HybridGridPointsProcessor(const HybridGridPointsProcessor&) = delete;
  HybridGridPointsProcessor& operator=(const HybridGridPointsProcessor&) = delete;

  void Process(std::unique_ptr<PointsBatch> batch) override {
    // range_data_inserter_.Insert({batch->origin, sensor::PointCloud(batch->points), {}},
    // &hybrid_grid_, /*intensity_hybrid_grid=*/nullptr)
    const std::vector<float> returns = points_processor_b200_internal::Flatten(*batch);
    const float origin[3] = {batch->origin.x(), batch->origin.y(), batch->origin.z()};
    points_processor_b200_internal::Check(csm_range_inserter3d_insert(
        inserter_, origin, returns.data(), nullptr, static_cast<int32_t>(batch->points.size()),
        hybrid_grid_.mutable_handle(), nullptr, nullptr));
    next_->Process(std::move(batch));
  }

  FlushResult Flush() override {
    const std::string serialized = mapping::scan_matching::b200_internal::Serialize(
        csm_grid3d_to_proto, hybrid_grid_.handle());
    file_writer_->Write(serialized.data(), serialized.size());
    points_processor_b200_internal::CheckClose(file_writer_.get());
    switch (next_->Flush()) {
      case FlushResult::kRestartStream:
        std::fprintf(stderr,
                     "Hybrid grid generation must be configured to occur after any stages that "
                     "require multiple passes.\n");
        std::abort();
      case FlushResult::kFinished:
        return FlushResult::kFinished;
    }
    std::abort();
  }

 private:
  PointsProcessor* const next_;
  csm_range_inserter3d* inserter_ = nullptr;
  mapping::scan_matching::DeviceHybridGrid hybrid_grid_;
  std::unique_ptr<FileWriter> file_writer_;
};

}  // namespace io
}  // namespace cartographer

#endif  // CSM_ADAPTER_POINTS_PROCESSOR_B200_H_
