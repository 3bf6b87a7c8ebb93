// map_eval_b200.hpp — C++ host side of the drop-in: MapEval's config / CLI / metric-output surface re-hosted on the
// C-ABI of libmapeval_b200.so.  Names, argument meaning and error behaviour follow the reference
// (map_eval/src/map_eval.h, map_eval.cpp, map_eval_main.cpp) for the path this repository replaces:
//
//   reference                                           here
//   ------------------------------------------------    ---------------------------------------------------------
//   struct Param                       map_eval.h:60     struct Param (same fields and defaults)
//   loadParametersFromYAML   map_eval_main.cpp:120-208    loadParametersFromYAML (same keys, same required/optional split)
//   MapEval::MapEval(Param&)        map_eval.h:123-189    MapEvalB200::MapEvalB200 (results folder + header lines)
//   MapEval::process()               map_eval.cpp:4-102    MapEvalB200::process (same sequence, same return codes)
//   computeMME(cloud, gt)           map_eval.cpp:149-189   computeMME            -> me_eval_mme
//   calculateMetricsWithInitialMatrix    :1204-1260       calculateMetricsWithInitialMatrix -> me_transform + me_eval_nn
//   calculateVMD                          :240-390        calculateVMD          -> me_eval_awd (+ the two text files)
//   saveMmeResults / saveRegistrationResults :392-482     same line formats in map_results.txt
//
//   VoxelDownSample                  map_eval.cpp:38-39    me_voxel_downsample (§8f N1)
//   performRegistration / performICPRegistration :191-237, 1366-1394   performRegistration -> me_icp (§8f N2: point-to-point,
//                                                         point-to-plane and generalized ICP) + calculateMetrics(reg)
//   rendered clouds                  :485-499, 568-736    render.hpp (§8f N3): entropy maps, raw / inlier NN-distance maps
// Normals: on path B (evaluate_using_initial: false) with point-to-plane or generalized ICP (registration_methods: 1 / 2)
// the normals that either FILE carries are read and handed to every context before VoxelDownSample, which averages them
// as Open3D does; generalized ICP builds a cloud's covariances from them and estimates normals (KNN 20) only for a cloud
// without any.  Point-to-plane ICP needs them in the ground-truth file, as in the reference (Open3D raises without them).
// Path A and point-to-point ICP never read normals.
#pragma once
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <ctime>
#include <filesystem>
#include <fstream>
#include <iomanip>
#include <iostream>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/mapeval_b200.h"
#include "cloud_io.hpp"
#include "gpu_group.hpp"
#include "render.hpp"
#include "yaml_lite.hpp"

namespace fs = std::filesystem;

struct Param {   // map_eval.h:60-116
  std::string evaluation_map_pcd_path_ = "/data/map_evaluation/canteen/";
  std::string map_gt_path_ = "/data/map_evaluation/canteen/merged_scan.pcd";
  std::string result_path_ = "/home/hts/workspace/dataset/eva_results/";
  std::string pcd_file_name_ = "map.pcd";
  std::string name_;
  int evaluation_method_ = 2;
  double voxel_size_ = 1.0;
  double icp_max_distance_ = 2.5;
  double nn_radius_ = 0.2;
  bool save_immediate_result_ = false;
  bool evaluate_mme_ = true;
  bool evaluate_gt_mme_ = true;
  bool evaluate_using_initial_ = true;
  bool evaluate_noised_gt_ = false;
  bool use_visualization = false;
  bool enable_debug = false;
  bool use_tbb_mme = true;
  double trunc_dist_[5] = {0, 0, 0, 0, 0};   // the reference leaves it uninitialised when accuracy_level is absent
  bool trunc_dist_set_ = false;
  double initial_matrix_[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  double noise_std_dev_ = 0.1;
  double vmd_voxel_size_ = 3.0;
  double downsample_size = 0.01;
  // additions of this implementation (absent keys keep the reference behaviour)
  int gpu_device_ = 0;
  int n_gpus_ = 1;                      // GPUs gpu_device_ .. gpu_device_ + n_gpus_ - 1 share the sweeps (NCCL all-reduce)
  bool geometric_gt_pairing_ = false;   // false = reproduce map_eval.cpp:1233/:1241 verbatim
  // evaluate_noised_gt: the degradation of the ground truth that stands in for the estimate (map_eval.cpp:1745-1829); the
  // operators run in the order deformation -> density -> noise -> outliers, every draw a function of simulation_seed_
  uint64_t simulation_seed_ = 20250002;   // synth.EST_SEED
  bool density_set_ = false;            // density is applied when density_region_size is given
  double density_sparse_ratio_ = 0.5, density_dense_ratio_ = 1.0, density_region_size_ = 0.0;
  double outlier_ratio_ = 0.0, outlier_range_ = 1.0;   // applied when outlier_ratio > 0
  double deform_radius_ = 0.0, deform_strength_ = 0.0; // applied when deform_radius > 0
  double deform_center_[3] = {0, 0, 0};
  // global_registration: the initial pose from the maps themselves (me_global_registration, FPFH + RANSAC on the GPU); its T
  // replaces initial_matrix on both paths
  bool global_registration_ = false;
  double global_registration_voxel_size_ = 0.5;
  uint64_t global_registration_seed_ = 0;
  int64_t global_registration_hypotheses_ = 100000;
  // accuracy curve: AC / COM / CD / F1 / IoU at tau_k = (accuracy_curve_max * k) / accuracy_curve_steps, k = 1..steps, written to
  // accuracy_curve.txt (me_nn_curve*: no new sweep); 0 = off.  accuracy_curve_max defaults to the largest accuracy_level
  int accuracy_curve_steps_ = 0;
  double accuracy_curve_max_ = 0.0;
  // exact distance quantiles at these probabilities and the Hausdorff distance, written to distance_quantiles.txt
  // (me_nn_quantile*: no new sweep); absent or empty = off
  std::vector<double> distance_quantiles_;
  // AC / COM / CD / F1 / IoU per region floor(x / region_size), written to region_errors.txt (me_nn_region*: no new sweep);
  // absent or 0 = off.  region_size = vmd_voxel_size lines the rows up with voxel_errors.txt
  double region_size_ = 0.0;
  // drift per region: every region floor(x / drift_region_size) of the estimate aligned to the ground truth on its own
  // (me_drift*: point-to-point ICP per region, R = icp_max_distance, ICP's criteria), written to region_drift.txt; absent or 0 = off
  double drift_region_size_ = 0.0;
  // point-to-plane AC / COM / CD / F1 / IoU and normal consistency, written to surface_metrics.txt (me_nn_surface*: no new
  // sweep); the clouds' normals where the files carry them, else working k-NN normals with surface_normals_knn neighbours
  bool surface_metrics_ = false;
  int surface_normals_knn_ = 20;
  // local consistency without a ground truth: MME and the mean plane variance of MME's neighbourhoods (r = nn_radius; the
  // est cloud with min_neighbors 10, the gt cloud with 5 when evaluate_gt_mme), whole map and per region
  // floor(x / consistency_region_size) (0 = whole map only), written to map_consistency.txt (me_consistency*)
  bool evaluate_consistency_ = false;
  double consistency_region_size_ = 0.0;
  // the mutually orthogonal metric without a ground truth (me_mom*, r = nn_radius; est with min_neighbors 10, gt with 5 when
  // evaluate_gt_mme), written to map_mom.txt
  bool evaluate_mom_ = false;
  double mom_angle_deg_ = 10.0, mom_planarity_ = 0.5;
  int64_t mom_min_family_ = 100;
  // the MOM call of each cloud per region floor(x / mom_region_size) (0 = off), written to map_mom_regions.txt (me_mom_region*)
  double mom_region_size_ = 0.0;
  // the estimate alone: gt_map_path is neither read nor required; MME, local consistency and MOM run on the est cloud
  bool evaluate_without_gt_ = false;
  // the Gaussian 2-Wasserstein distance per voxel at vmd_voxel_size (me_eval_w2, after calculateVMD): offset and shape terms,
  // their means and SCS over W2, written to map_w2.txt and voxel_w2.txt; pairs need w2_min_points (>= 2) in each cloud
  bool evaluate_w2_ = false;
  int w2_min_points_ = 100;
};

// map_eval_main.cpp:120-208
inline Param loadParametersFromYAML(const std::string &yaml_file_path) {
  try {
    yaml_lite::Document config = yaml_lite::Document::LoadFile(yaml_file_path);
    Param param;
    param.evaluation_method_ = config["registration_methods"].as<int>();
    param.icp_max_distance_ = config["icp_max_distance"].as<double>();
    if (config["accuracy_level"] && config["accuracy_level"].size() >= 5) {
      for (int i = 0; i < 5; ++i) param.trunc_dist_[i] = config["accuracy_level"][i].as<double>();
      param.trunc_dist_set_ = true;
    }
    if (config["initial_matrix"] && config["initial_matrix"].size() >= 4) {
      for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) param.initial_matrix_[i * 4 + j] = config["initial_matrix"][i][j].as<double>();
    }
    param.save_immediate_result_ = config["save_immediate_result"].as<bool>();
    param.evaluate_mme_ = config["evaluate_mme"].as<bool>();
    param.evaluate_gt_mme_ = config["evaluate_gt_mme"].as<bool>();
    param.evaluate_using_initial_ = config["evaluate_using_initial"].as<bool>();
    param.nn_radius_ = config["nn_radius"].as<double>();
    param.vmd_voxel_size_ = config["vmd_voxel_size"].as<double>();
    param.downsample_size = config["downsample_size"].as<double>();
    param.evaluation_map_pcd_path_ = config["estimate_map_path"].as<std::string>();
    if (config["evaluate_without_gt"]) param.evaluate_without_gt_ = config["evaluate_without_gt"].as<bool>();
    if (!param.evaluate_without_gt_ || config["gt_map_path"]) param.map_gt_path_ = config["gt_map_path"].as<std::string>();
    else param.map_gt_path_.clear();
    param.name_ = config["scene_name"].as<std::string>();
    if (!param.evaluation_map_pcd_path_.empty() && param.evaluation_map_pcd_path_.back() != '/')
      param.evaluation_map_pcd_path_ += '/';
    param.result_path_ = param.evaluation_map_pcd_path_ + "map_results/";
    if (config["pcd_file_name"]) param.pcd_file_name_ = config["pcd_file_name"].as<std::string>();
    if (config["evaluate_noised_gt"]) param.evaluate_noised_gt_ = config["evaluate_noised_gt"].as<bool>();
    if (config["noise_std_dev"]) param.noise_std_dev_ = config["noise_std_dev"].as<double>();
    if (config["voxel_size"]) param.voxel_size_ = config["voxel_size"].as<double>();
    if (config["use_visualization"]) param.use_visualization = config["use_visualization"].as<bool>();
    param.enable_debug = config["enable_debug"].as<bool>();
    if (config["use_tbb_mme"]) param.use_tbb_mme = config["use_tbb_mme"].as<bool>();
    if (config["gpu_device"]) param.gpu_device_ = config["gpu_device"].as<int>();
    if (config["n_gpus"]) param.n_gpus_ = config["n_gpus"].as<int>();
    if (config["geometric_gt_pairing"]) param.geometric_gt_pairing_ = config["geometric_gt_pairing"].as<bool>();
    if (config["simulation_seed"]) param.simulation_seed_ = config["simulation_seed"].as<uint64_t>();
    if (config["density_sparse_ratio"]) param.density_sparse_ratio_ = config["density_sparse_ratio"].as<double>();
    if (config["density_dense_ratio"]) param.density_dense_ratio_ = config["density_dense_ratio"].as<double>();
    if (config["density_region_size"]) {
      param.density_region_size_ = config["density_region_size"].as<double>();
      param.density_set_ = true;
    }
    if (config["outlier_ratio"]) param.outlier_ratio_ = config["outlier_ratio"].as<double>();
    if (config["outlier_range"]) param.outlier_range_ = config["outlier_range"].as<double>();
    if (config["deform_radius"]) param.deform_radius_ = config["deform_radius"].as<double>();
    if (config["deform_strength"]) param.deform_strength_ = config["deform_strength"].as<double>();
    if (config["global_registration"]) param.global_registration_ = config["global_registration"].as<bool>();
    if (config["global_registration_voxel_size"])
      param.global_registration_voxel_size_ = config["global_registration_voxel_size"].as<double>();
    if (config["global_registration_seed"]) param.global_registration_seed_ = config["global_registration_seed"].as<uint64_t>();
    if (config["global_registration_hypotheses"])
      param.global_registration_hypotheses_ = (int64_t)config["global_registration_hypotheses"].as<uint64_t>();
    if (config["deform_center"] && config["deform_center"].size() >= 3)
      for (int a = 0; a < 3; ++a) param.deform_center_[a] = config["deform_center"][a].as<double>();
    if (config["accuracy_curve_steps"]) param.accuracy_curve_steps_ = config["accuracy_curve_steps"].as<int>();
    param.accuracy_curve_max_ = config["accuracy_curve_max"] ? config["accuracy_curve_max"].as<double>()
                                                             : *std::max_element(param.trunc_dist_, param.trunc_dist_ + 5);
    if (config["distance_quantiles"])
      for (size_t i = 0; i < config["distance_quantiles"].size(); ++i)
        param.distance_quantiles_.push_back(config["distance_quantiles"][i].as<double>());
    if (config["region_size"]) {
      param.region_size_ = config["region_size"].as<double>();
      if (!(std::isfinite(param.region_size_) && param.region_size_ >= 0.0))
        throw std::runtime_error("region_size must be finite and >= 0 (0 = off), not " + config["region_size"].as<std::string>());
    }
    if (config["drift_region_size"]) {
      param.drift_region_size_ = config["drift_region_size"].as<double>();
      if (!(std::isfinite(param.drift_region_size_) && param.drift_region_size_ >= 0.0))
        throw std::runtime_error("drift_region_size must be finite and >= 0 (0 = off), not " +
                                 config["drift_region_size"].as<std::string>());
    }
    if (config["surface_metrics"]) param.surface_metrics_ = config["surface_metrics"].as<bool>();
    if (config["surface_normals_knn"]) {
      param.surface_normals_knn_ = config["surface_normals_knn"].as<int>();
      if (param.surface_normals_knn_ < 1 || param.surface_normals_knn_ > 64)
        throw std::runtime_error("surface_normals_knn must be in 1..64, not " + config["surface_normals_knn"].as<std::string>());
    }
    if (config["evaluate_consistency"]) param.evaluate_consistency_ = config["evaluate_consistency"].as<bool>();
    if (config["consistency_region_size"]) {
      param.consistency_region_size_ = config["consistency_region_size"].as<double>();
      if (!(std::isfinite(param.consistency_region_size_) && param.consistency_region_size_ >= 0.0))
        throw std::runtime_error("consistency_region_size must be finite and >= 0 (0 = the whole map only), not " +
                                 config["consistency_region_size"].as<std::string>());
    }
    if (config["evaluate_mom"]) param.evaluate_mom_ = config["evaluate_mom"].as<bool>();
    if (config["mom_angle_deg"]) {
      param.mom_angle_deg_ = config["mom_angle_deg"].as<double>();
      if (!(param.mom_angle_deg_ > 0.0 && param.mom_angle_deg_ <= 30.0))
        throw std::runtime_error("mom_angle_deg must be in (0, 30], not " + config["mom_angle_deg"].as<std::string>());
    }
    if (config["mom_planarity"]) {
      param.mom_planarity_ = config["mom_planarity"].as<double>();
      if (!(param.mom_planarity_ > 0.0 && param.mom_planarity_ <= 1.0))
        throw std::runtime_error("mom_planarity must be in (0, 1], not " + config["mom_planarity"].as<std::string>());
    }
    if (config["mom_min_family"]) {
      const double mf = config["mom_min_family"].as<double>();
      if (!(mf >= 1.0 && mf <= 9.0e18 && mf == std::floor(mf)))
        throw std::runtime_error("mom_min_family must be an integer >= 1, not " + config["mom_min_family"].as<std::string>());
      param.mom_min_family_ = (int64_t)mf;
    }
    if (config["mom_region_size"]) {
      param.mom_region_size_ = config["mom_region_size"].as<double>();
      if (!(std::isfinite(param.mom_region_size_) && param.mom_region_size_ >= 0.0))
        throw std::runtime_error("mom_region_size must be finite and >= 0 (0 = off), not " + config["mom_region_size"].as<std::string>());
      if (param.mom_region_size_ > 0.0 && !param.evaluate_mom_)
        throw std::runtime_error("mom_region_size needs evaluate_mom: true (it breaks the MOM call down by region)");
    }
    if (config["evaluate_w2"]) param.evaluate_w2_ = config["evaluate_w2"].as<bool>();
    if (config["w2_min_points"]) {
      const double mp = config["w2_min_points"].as<double>();
      if (!(mp >= 2.0 && mp <= 2147483647.0 && mp == std::floor(mp)))
        throw std::runtime_error("w2_min_points must be an integer >= 2, not " + config["w2_min_points"].as<std::string>());
      param.w2_min_points_ = (int)mp;
    }
    return param;
  } catch (const std::exception &e) {
    std::cerr << "Error loading parameters: " << e.what() << std::endl;
    throw std::runtime_error("Failed to parse YAML file: " + yaml_file_path);
  }
}

inline void dumpParam(const Param &p, std::ostream &os) {
  os << std::setprecision(17);
  os << "registration_methods=" << p.evaluation_method_ << "\nicp_max_distance=" << p.icp_max_distance_ << "\naccuracy_level=";
  for (int i = 0; i < 5; ++i) os << (i ? "," : "") << p.trunc_dist_[i];
  os << "\naccuracy_level_set=" << p.trunc_dist_set_ << "\ninitial_matrix=";
  for (int i = 0; i < 16; ++i) os << (i ? "," : "") << p.initial_matrix_[i];
  os << "\nsave_immediate_result=" << p.save_immediate_result_ << "\nevaluate_mme=" << p.evaluate_mme_
     << "\nevaluate_gt_mme=" << p.evaluate_gt_mme_ << "\nevaluate_using_initial=" << p.evaluate_using_initial_
     << "\nnn_radius=" << p.nn_radius_ << "\nvmd_voxel_size=" << p.vmd_voxel_size_ << "\ndownsample_size=" << p.downsample_size
     << "\nestimate_map_path=" << p.evaluation_map_pcd_path_ << "\ngt_map_path=" << p.map_gt_path_ << "\nscene_name=" << p.name_
     << "\nresult_path=" << p.result_path_ << "\npcd_file_name=" << p.pcd_file_name_ << "\nevaluate_noised_gt=" << p.evaluate_noised_gt_
     << "\nnoise_std_dev=" << p.noise_std_dev_ << "\nvoxel_size=" << p.voxel_size_ << "\nuse_visualization=" << p.use_visualization
     << "\nenable_debug=" << p.enable_debug << "\nuse_tbb_mme=" << p.use_tbb_mme << "\nsimulation_seed=" << p.simulation_seed_
     << "\ndensity_sparse_ratio=" << p.density_sparse_ratio_ << "\ndensity_dense_ratio=" << p.density_dense_ratio_
     << "\ndensity_region_size=" << p.density_region_size_ << "\ndensity_set=" << p.density_set_ << "\noutlier_ratio=" << p.outlier_ratio_
     << "\noutlier_range=" << p.outlier_range_ << "\ndeform_radius=" << p.deform_radius_ << "\ndeform_strength=" << p.deform_strength_
     << "\ndeform_center=" << p.deform_center_[0] << "," << p.deform_center_[1] << "," << p.deform_center_[2]
     << "\nglobal_registration=" << p.global_registration_ << "\nglobal_registration_voxel_size=" << p.global_registration_voxel_size_
     << "\nglobal_registration_seed=" << p.global_registration_seed_
     << "\nglobal_registration_hypotheses=" << p.global_registration_hypotheses_
     << "\naccuracy_curve_steps=" << p.accuracy_curve_steps_ << "\naccuracy_curve_max=" << p.accuracy_curve_max_
     << "\ndistance_quantiles=";
  for (size_t i = 0; i < p.distance_quantiles_.size(); ++i) os << (i ? "," : "") << p.distance_quantiles_[i];
  os << "\nregion_size=" << p.region_size_ << "\ndrift_region_size=" << p.drift_region_size_ << "\nsurface_metrics=" << p.surface_metrics_
     << "\nsurface_normals_knn=" << p.surface_normals_knn_ << "\nevaluate_consistency=" << p.evaluate_consistency_
     << "\nconsistency_region_size=" << p.consistency_region_size_ << "\nevaluate_mom=" << p.evaluate_mom_
     << "\nmom_angle_deg=" << p.mom_angle_deg_ << "\nmom_planarity=" << p.mom_planarity_ << "\nmom_min_family=" << p.mom_min_family_
     << "\nmom_region_size=" << p.mom_region_size_ << "\nevaluate_w2=" << p.evaluate_w2_ << "\nw2_min_points=" << p.w2_min_points_
     << "\nevaluate_without_gt=" << p.evaluate_without_gt_ << "\n";
}

// Eigen's default IOFormat for `vec.transpose()`: coefficients right-aligned to a common width, one space apart
// Eigen's operator<< for a 4x4 matrix: rows on separate lines, every coefficient right-aligned to the widest one
inline std::string eigenMatrix4(const double *T, int precision) {
  std::string cell[16];
  size_t w = 0;
  for (int i = 0; i < 16; ++i) {
    std::ostringstream os;
    os << std::fixed << std::setprecision(precision) << T[i];
    cell[i] = os.str();
    w = std::max(w, cell[i].size());
  }
  std::string out;
  for (int r = 0; r < 4; ++r) {
    if (r) out += "\n";
    for (int c = 0; c < 4; ++c) {
      if (c) out += " ";
      out += std::string(w - cell[r * 4 + c].size(), ' ') + cell[r * 4 + c];
    }
  }
  return out;
}

inline std::string eigenRow(const double *v, int n, int precision) {
  std::vector<std::string> s(n);
  size_t w = 0;
  for (int i = 0; i < n; ++i) {
    std::ostringstream os;
    os << std::fixed << std::setprecision(precision) << v[i];
    s[i] = os.str();
    w = std::max(w, s[i].size());
  }
  std::string out;
  for (int i = 0; i < n; ++i) {
    if (i) out += " ";
    out += std::string(w - s[i].size(), ' ') + s[i];
  }
  return out;
}

class TicToc {   // include/tic_toc.h:10-25 (milliseconds, system_clock)
 public:
  TicToc() { tic(); }
  void tic() { start = std::chrono::system_clock::now(); }
  double toc() { return std::chrono::duration<double>(std::chrono::system_clock::now() - start).count() * 1000; }
 private:
  std::chrono::time_point<std::chrono::system_clock> start;
};

class MapEvalB200 {
 public:
  // Configurations this driver cannot run, reported BEFORE map_results.txt is opened (no partial record is left behind).
  static bool validate(const Param &p, std::string *why) {
    if (p.accuracy_curve_steps_ < 0 || p.accuracy_curve_steps_ > ME_CURVE_MAX_LEVELS) {
      *why = "accuracy_curve_steps: " + std::to_string(p.accuracy_curve_steps_) + " is outside 0 .. " + std::to_string(ME_CURVE_MAX_LEVELS);
      return false;
    }
    if (p.accuracy_curve_steps_ > 0 && !(std::isfinite(p.accuracy_curve_max_) && p.accuracy_curve_max_ >= 0.0)) {
      *why = "accuracy_curve_max must be finite and >= 0";
      return false;
    }
    if (p.distance_quantiles_.size() > ME_QUANTILE_MAX_PROBS) {
      *why = "distance_quantiles: " + std::to_string(p.distance_quantiles_.size()) + " probabilities, at most " +
             std::to_string(ME_QUANTILE_MAX_PROBS);
      return false;
    }
    for (double q : p.distance_quantiles_)
      if (!(std::isfinite(q) && q >= 0.0 && q <= 1.0)) {
        *why = "distance_quantiles: every probability must be finite and in [0, 1]";
        return false;
      }
    if (p.evaluate_without_gt_) {      // the keys that need a ground truth
      const char *key = p.evaluate_noised_gt_ ? "evaluate_noised_gt"
                        : p.global_registration_ ? "global_registration"
                        : p.accuracy_curve_steps_ > 0 ? "accuracy_curve_steps"
                        : !p.distance_quantiles_.empty() ? "distance_quantiles"
                        : p.region_size_ > 0.0 ? "region_size"
                        : p.drift_region_size_ > 0.0 ? "drift_region_size"
                        : p.surface_metrics_ ? "surface_metrics"
                        : p.evaluate_w2_ ? "evaluate_w2" : nullptr;
      if (key) {
        *why = std::string(key) + " needs a ground truth; evaluate_without_gt evaluates the estimate alone";
        return false;
      }
      if (!p.evaluate_mme_ && !p.evaluate_consistency_ && !p.evaluate_mom_) {
        *why = "evaluate_without_gt: nothing to do (evaluate_mme, evaluate_consistency and evaluate_mom are all off)";
        return false;
      }
      return true;
    }
    if (p.evaluate_using_initial_) return true;
    if (p.evaluation_method_ < 0 || p.evaluation_method_ > 2) {
      *why = "Invalid registration type specified (registration_methods: " + std::to_string(p.evaluation_method_) +
             "; 0 = point-to-point, 1 = point-to-plane, 2 = generalized ICP, map_eval.cpp:1368-1390)";
      return false;
    }
    return true;
  }

  explicit MapEvalB200(Param &param) : param_(param) {   // map_eval.h:123-189
    t1 = t2 = t3 = t4 = t5 = t6 = t7 = 0.0;
    if (param_.pcd_file_name_ == "merged_maps_all_trans.pcd") subfolder = "merged_maps_all_results/";
    else if (param_.pcd_file_name_ == "merged_maps_s0_trans.pcd") subfolder = "merged_maps_s0_results/";
    else if (param_.pcd_file_name_ == "merged_maps_s1_trans.pcd") subfolder = "merged_maps_s1_results/";
    else if (param_.pcd_file_name_ == "global_pcd_lidar.pcd") subfolder = "map_results/";
    else {
      subfolder = "map_results/";
      std::cerr << "ERROR: Invalid PCD file name: " << param_.pcd_file_name_ << std::endl;   // as the reference (map.pcd lands here too)
    }
    results_subfolder = param_.evaluation_map_pcd_path_ + subfolder;
    std::cout << "INFO: Saving results to: " << results_subfolder << std::endl;
    if (!fs::exists(results_subfolder)) fs::create_directory(results_subfolder);
    results_file_path = results_subfolder + "map_results.txt";
    file_result.open(results_file_path, std::ios::app);
    if (!file_result.is_open()) std::cerr << "ERROR: Failed to open results file at " << results_file_path << std::endl;
    auto now = std::chrono::system_clock::now();
    std::time_t now_c = std::chrono::system_clock::to_time_t(now);
    std::stringstream time_stream;
    time_stream << std::put_time(std::localtime(&now_c), "%Y-%m-%d %X");
    file_result << param_.name_ << " ===================== " << time_stream.str() << " ===================== " << std::endl;
    file_result << "Ground Truth Path: " << param_.map_gt_path_ << std::endl;
    file_result << "Evaluation Map Path: " << param_.evaluation_map_pcd_path_ + param_.pcd_file_name_ << std::endl;
    std::cout << "INFO: Evaluation details saved to " << results_file_path << std::endl;
  }
  ~MapEvalB200() {
    file_result.close();
    gpus_.destroy();
  }

  int process();                                   // map_eval.cpp:4-102
  int computeMME();                                // map_eval.cpp:149-189
  int calculateMetricsWithInitialMatrix();         // map_eval.cpp:1204-1260
  int performRegistration();                       // map_eval.cpp:191-237, 1366-1394 (all three registration methods), 1147-1202
  int calculateVMD();                              // map_eval.cpp:240-390
  void saveMmeResults();                           // map_eval.cpp:392-421 (result line + the rendered entropy clouds)
  void saveRegistrationResults();                  // map_eval.cpp:424-482 (text lines only)

  Param param_;
  // results, named as the reference's members (map_eval.h:319-361)
  me_nn_result nn_{};
  me_mme_result mme_est_res_{}, mme_gt_res_{};
  me_awd_result awd_{};
  double mme_est = 0.0, mme_gt = 0.0, max_abs_entropy = 0.0, min_abs_entropy = 0.0;
  double vmd = 0.0, scs_overall = 0.0, full_chamfer_dist = 0.0;

 private:
  int fail(const char *what) {
    std::cerr << "ERROR: " << what << ": "
              << (!gpus_.error().empty() ? gpus_.error().c_str() : (ctx_ ? me_last_error(ctx_) : me_last_error(nullptr))) << std::endl;
    return -1;
  }
  render::ColoredCloud map_3d_entropy_, gt_3d_entropy_, map_3d_render_raw_, map_3d_render_inlier_;   // map_eval.h:341-347
  int simulateEstimate(me_ctx *c, int64_t *n);
  int globalRegistration();                        // global_registration: T from the maps replaces initial_matrix     // evaluate_noised_gt: estimate := degraded copy of the ground truth
  std::string simulationSummary() const;
  int renderEntropy(int which, int64_t n, render::ColoredCloud *out);
  int renderDistances(bool cutoff_strict);
  int accuracyCurve(const me_nn_params &p, const me_nn_accum &e2g, const me_nn_accum &g2e);
  int distanceQuantiles();
  int regionErrors();
  int surfaceMetrics();
  int localConsistency();
  int mom();
  int voxelW2();
  int processWithoutGt();
  bool gt_mme() const { return param_.evaluate_gt_mme_ && !param_.evaluate_without_gt_; }
  int regionDrift();
  GpuGroup gpus_;            // one context per GPU; rank r evaluates the r-th shard of every sweep's query range
  me_ctx *ctx_ = nullptr;    // = gpus_.ctx(0): the voxel stage and the single-GPU calls
  std::vector<double> map_3d_, gt_3d_;   // N x 3 fp64, the layout of open3d PointCloud::points_ (as loaded)
  std::vector<double> map_normals_, gt_normals_;   // PointCloud::normals_ as loaded (path B, point-to-plane / generalized ICP)
  int64_t n_est_ = 0, n_gt_ = 0;         // point counts after VoxelDownSample (the clouds the metrics see)
  double t1, t2, t3, t4, t5, t6, t7, t_fcd = 0.0, t_acc = 0.0;
  double t_vmd = 0.0, t_v = 0.0, t_cdf = 0.0, t_scs = 0.0;
  std::string subfolder, results_subfolder, results_file_path;
  std::ofstream file_result;
};

inline int MapEvalB200::process() {
  TicToc tic_toc;
  std::string err;
  if (!validate(param_, &err)) {
    std::cerr << "ERROR: " << err << std::endl;
    return -1;
  }
  if (param_.evaluate_without_gt_) return processWithoutGt();
  // point-to-plane ICP needs normals on the target cloud, which can only come from the ground-truth file; generalized ICP
  // uses the normals of either file when it carries them (InitializePointCloudForGeneralizedICP); the surface metrics use them
  // on either path
  const bool load_normals =
      (!param_.evaluate_using_initial_ && (param_.evaluation_method_ == 1 || param_.evaluation_method_ == 2)) || param_.surface_metrics_;
  std::string file_extension = param_.map_gt_path_.substr(param_.map_gt_path_.find_last_of(".") + 1);
  bool gt_ok = false;
  if (file_extension == "pcd") gt_ok = cloud_io::read_pcd(param_.map_gt_path_, gt_3d_, &err, load_normals ? &gt_normals_ : nullptr);
  else if (file_extension == "ply") gt_ok = cloud_io::read_ply(param_.map_gt_path_, gt_3d_, &err, load_normals ? &gt_normals_ : nullptr);
  else {
    std::cerr << "ERROR: Unsupported ground truth file format: " << param_.map_gt_path_ << std::endl;
    return -1;
  }
  if (!gt_ok && param_.enable_debug) std::cerr << "WARNING: " << err << std::endl;   // the reference ignores this return value
  // evaluate_noised_gt (config.yaml:55-59): the estimate file is not read; every GPU degrades a copy of the ground truth
  const bool simulate = param_.evaluate_noised_gt_;
  if (!simulate) {
    bool success = cloud_io::read_pcd(param_.evaluation_map_pcd_path_ + param_.pcd_file_name_, map_3d_, &err,
                                      load_normals ? &map_normals_ : nullptr);
    if (param_.enable_debug)
      std::cout << "INFO: Loading map point cloud from: " << param_.evaluation_map_pcd_path_ + param_.pcd_file_name_ << std::endl;
    if (!success) {
      std::cerr << "ERROR: Failed to load point cloud from the specified path." << std::endl;
      return -1;
    }
  }
  if ((!simulate && map_3d_.empty()) || gt_3d_.empty()) {
    std::cerr << "ERROR: One or both point clouds are empty!" << std::endl;
    return -1;
  }
  if (load_normals && param_.evaluation_method_ == 1 && gt_normals_.size() != gt_3d_.size()) {
    std::cerr << "ERROR: TransformationEstimationPointToPlane requires pre-computed normal vectors for the target PointCloud: "
              << param_.map_gt_path_ << " carries none (registration_methods: 1)." << std::endl;
    return -1;
  }
  if (!gpus_.create(std::max(1, param_.n_gpus_), param_.gpu_device_, param_.vmd_voxel_size_)) return fail("cannot create the GPU context(s)");
  ctx_ = gpus_.ctx(0);
  if (gpus_.size() > 1) std::cout << "INFO: sharding the sweeps over " << gpus_.size() << " GPUs (NCCL all-reduce of the accumulators)" << std::endl;
  // every GPU holds both clouds (the lattices are replicated); VoxelDownSample (map_eval.cpp:38-39) runs on each of them.
  // The reference calls it unconditionally (Open3D raises for voxel_size <= 0); a non-positive value skips the step here.
  // Normals loaded from a file go with their cloud, so that VoxelDownSample averages them.
  std::vector<int64_t> ne(gpus_.size(), (int64_t)(map_3d_.size() / 3)), ng(gpus_.size(), (int64_t)(gt_3d_.size() / 3));
  const bool map_has_normals = !map_normals_.empty() && map_normals_.size() == map_3d_.size();
  const bool gt_has_normals = !gt_normals_.empty() && gt_normals_.size() == gt_3d_.size();
  if (simulate) std::cout << "INFO: " << simulationSummary() << std::endl;
  if (gpus_.for_each([&](int r, me_ctx *c) {
        int rc = simulate ? ME_OK : me_set_cloud(c, ME_CLOUD_EST, map_3d_.data(), (int64_t)(map_3d_.size() / 3));
        if (rc == ME_OK) rc = me_set_cloud(c, ME_CLOUD_GT, gt_3d_.data(), (int64_t)(gt_3d_.size() / 3));
        if (rc == ME_OK && map_has_normals) rc = me_set_normals(c, ME_CLOUD_EST, map_normals_.data(), (int64_t)(map_normals_.size() / 3));
        if (rc == ME_OK && gt_has_normals) rc = me_set_normals(c, ME_CLOUD_GT, gt_normals_.data(), (int64_t)(gt_normals_.size() / 3));
        if (rc == ME_OK && simulate) rc = simulateEstimate(c, &ne[r]);
        if (rc == ME_OK && param_.downsample_size > 0) {
          rc = me_voxel_downsample(c, ME_CLOUD_EST, param_.downsample_size, &ne[r]);
          if (rc == ME_OK) rc = me_voxel_downsample(c, ME_CLOUD_GT, param_.downsample_size, &ng[r]);
        }
        return rc;
      }) != ME_OK)
    return fail("uploading / down-sampling the clouds");
  if (!(param_.downsample_size > 0)) std::cout << "INFO: downsample_size <= 0: clouds are evaluated as loaded." << std::endl;
  const int64_t n_est = ne[0], n_gt = ng[0];
  n_est_ = n_est; n_gt_ = n_gt;

  file_result << std::fixed << std::setprecision(15) << "Estimated-Ground Truth point count: " << n_est << " / " << n_gt
              << std::endl;
  if (param_.enable_debug)
    std::cout << "INFO: Loaded point clouds: " << n_est << " points (Map), " << n_gt << " points (Ground Truth)."
              << std::endl;

  if (param_.global_registration_ && globalRegistration() != 0) return -1;

  if (param_.evaluate_mme_) {
    if (param_.enable_debug) std::cout << "INFO: Starting MME calculation..." << std::endl;
    if (computeMME() != 0) return -1;
    if (param_.enable_debug) std::cout << "INFO: MME calculation completed. Saving results." << std::endl;
    if (param_.save_immediate_result_) saveMmeResults();
    t2 = tic_toc.toc();
    if (param_.enable_debug) std::cout << "INFO: MME calculation completed in: " << (t2 - t1) / 1000.0 << " seconds." << std::endl;
  }
  if (param_.enable_debug) std::cout << "INFO: Starting registration..." << std::endl;
  if (param_.evaluate_using_initial_) {
    if (param_.enable_debug) std::cout << "INFO: Using initial matrix without registration." << std::endl;
    if (calculateMetricsWithInitialMatrix() != 0) return -1;
  } else {
    // map_eval.cpp:81 -> performRegistration() -> performICPRegistration() (:1366-1394) -> calculateMetrics(reg) (:1147-1202)
    if (performRegistration() != 0) return -1;
  }
  if (calculateVMD() != 0) return -1;
  if (param_.enable_debug) std::cout << "INFO: VMD calculation completed." << std::endl;
  // on the lattices calculateVMD left aligned with vmd_voxel_size
  if (param_.evaluate_w2_ && voxelW2() != 0) return -1;
  // after every consumer of the pass's NN records (the sweep may lay a cloud out again), with the estimate in its final frame
  if (param_.evaluate_consistency_ && localConsistency() != 0) return -1;
  if (param_.evaluate_mom_ && mom() != 0) return -1;
  if (param_.save_immediate_result_) {
    if (param_.enable_debug) std::cout << "INFO: Saving registration results..." << std::endl;
    saveRegistrationResults();
  }
  if (param_.enable_debug) std::cout << "INFO: Results saved successfully." << std::endl;
  return 0;
}

// evaluate_noised_gt: the reference's simulation operators (map_eval.cpp:1745-1829) on a copy of the ground truth, in the
// order deformation -> density -> noise -> outliers (outliers are drawn from the already noisy map, as addSparseOutliers
// copies points of the cloud it gets).  Every draw is a function of simulation_seed, so every GPU builds the same map.
inline int MapEvalB200::simulateEstimate(me_ctx *c, int64_t *n) {
  const Param &p = param_;
  const uint64_t seed = p.simulation_seed_;
  *n = (int64_t)(gt_3d_.size() / 3);
  int rc = me_copy_cloud(c, ME_CLOUD_GT, ME_CLOUD_EST);      // with the ground truth's normals when they were loaded
  if (rc == ME_OK && p.deform_radius_ > 0)
    rc = me_add_local_deformation(c, ME_CLOUD_EST, p.deform_radius_, p.deform_strength_, p.deform_center_);
  if (rc == ME_OK && p.density_set_)
    rc = me_add_non_uniform_density(c, ME_CLOUD_EST, p.density_sparse_ratio_, p.density_dense_ratio_, p.density_region_size_, seed, n);
  if (rc == ME_OK && p.noise_std_dev_ != 0) rc = me_add_gaussian_noise(c, ME_CLOUD_EST, p.noise_std_dev_, seed);
  if (rc == ME_OK && p.outlier_ratio_ > 0) rc = me_add_sparse_outliers(c, ME_CLOUD_EST, p.outlier_ratio_, p.outlier_range_, seed, n);
  return rc;
}

inline std::string MapEvalB200::simulationSummary() const {
  const Param &p = param_;
  std::ostringstream os;
  os << std::setprecision(6) << "evaluate_noised_gt: the estimated map is not read; it is the ground truth";
  std::vector<std::string> ops;
  if (p.deform_radius_ > 0) {
    std::ostringstream o;
    o << std::setprecision(6) << "local deformation (radius " << p.deform_radius_ << ", strength " << p.deform_strength_ << ", centre " << p.deform_center_[0]
      << " " << p.deform_center_[1] << " " << p.deform_center_[2] << ")";
    ops.push_back(o.str());
  }
  if (p.density_set_) {
    std::ostringstream o;
    o << std::setprecision(6) << "non-uniform density (sparse " << p.density_sparse_ratio_ << ", dense " << p.density_dense_ratio_ << ", region "
      << p.density_region_size_ << ")";
    ops.push_back(o.str());
  }
  if (p.noise_std_dev_ != 0) {
    std::ostringstream o;
    o << std::setprecision(6) << "Gaussian noise (std_dev " << p.noise_std_dev_ << ")";
    ops.push_back(o.str());
  }
  if (p.outlier_ratio_ > 0) {
    std::ostringstream o;
    o << std::setprecision(6) << "sparse outliers (ratio " << p.outlier_ratio_ << ", range " << p.outlier_range_ << ")";
    ops.push_back(o.str());
  }
  if (ops.empty()) os << " unchanged";
  for (size_t i = 0; i < ops.size(); ++i) os << (i ? ", then " : " with ") << ops[i];
  os << " (simulation_seed " << p.simulation_seed_ << ")";
  static const double eye[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  if (!std::equal(p.initial_matrix_, p.initial_matrix_ + 16, eye))
    os << "; initial_matrix is not the identity, but the simulated map lies in the ground truth's frame";
  return os.str();
}

// ColorPointCloudByMME (map_eval.cpp:686-736) on the entropies of the sweep that just ran (each GPU holds its shard)
inline int MapEvalB200::renderEntropy(int which, int64_t n, render::ColoredCloud *out) {
  std::vector<double> ent((size_t)n, 0.0), part((size_t)n), xyz((size_t)n * 3);
  for (int r = 0; r < gpus_.size(); ++r) {
    if (me_get_entropies(gpus_.ctx(r), which, part.data()) != ME_OK) { ctx_ = gpus_.ctx(r); const int rc = fail("me_get_entropies"); ctx_ = gpus_.ctx(0); return rc; }
    for (int64_t i = 0; i < n; ++i) ent[i] += part[i];          // disjoint shards: the other ranks hold zeros
  }
  int64_t got = 0;
  if (me_get_cloud(ctx_, which, xyz.data(), n, &got) != ME_OK || got != n) return fail("me_get_cloud");
  *out = render::color_by_entropy(xyz, ent);
  return 0;
}

// renderDistanceOnPointCloud (map_eval.cpp:586-606) for the raw map (every estimated point against the ground truth) and
// the inlier map (the corresponding points against each other), both clipped at accuracy_level[0] (:485-487).
inline int MapEvalB200::renderDistances(bool cutoff_strict) {
  const int64_t n = n_est_;
  std::vector<int32_t> idx((size_t)n, -1), pidx((size_t)n);
  std::vector<double> d2((size_t)n, std::nan("")), pd2((size_t)n), est((size_t)n * 3), gt((size_t)n_gt_ * 3);
  for (int r = 0; r < gpus_.size(); ++r) {
    if (me_get_nn(gpus_.ctx(r), ME_CLOUD_EST, pidx.data(), pd2.data()) != ME_OK) return fail("me_get_nn");
    for (int64_t i = 0; i < n; ++i)
      if (pidx[i] >= 0) { idx[i] = pidx[i]; d2[i] = pd2[i]; }
  }
  int64_t got = 0;
  if (me_get_cloud(ctx_, ME_CLOUD_EST, est.data(), n, &got) != ME_OK || got != n) return fail("me_get_cloud(est)");
  if (me_get_cloud(ctx_, ME_CLOUD_GT, gt.data(), n_gt_, &got) != ME_OK || got != n_gt_) return fail("me_get_cloud(gt)");
  const double dis = param_.trunc_dist_[0];
  map_3d_render_raw_ = render::color_by_distance(est, d2, dis);
  // corresponding_cloud_est / corresponding_cloud_gt: the kept est->gt pairs (:1083-1089); the reference's second call of
  // getDiffRegResultWithCorrespondence on path A overwrites them with index-swapped points (:1241) — not reproduced
  std::vector<double> ce, cg;
  const double R = param_.icp_max_distance_;
  for (int64_t i = 0; i < n; ++i) {
    if (idx[i] < 0) continue;
    if (!(cutoff_strict ? d2[i] < R * R : d2[i] <= R)) continue;
    for (int a = 0; a < 3; ++a) { ce.push_back(est[3 * i + a]); cg.push_back(gt[3 * (size_t)idx[i] + a]); }
  }
  map_3d_render_inlier_ = render::ColoredCloud();
  if (ce.empty()) return 0;
  me_options opt{};
  opt.abi_version = ME_ABI_VERSION; opt.device = param_.gpu_device_; opt.rank = 0; opt.world = 1;
  me_ctx *tmp = nullptr;
  if (me_create(&opt, &tmp) != ME_OK) return fail("me_create (inlier map)");
  const int64_t nc = (int64_t)(ce.size() / 3);
  me_nn_params p{};
  p.icp_max_distance = R; p.cutoff_mode = ME_CUTOFF_DIST_LT_R; p.pairing = ME_PAIRING_GEOMETRIC; p.want_full_cd = 1; p.directions = 1;
  me_nn_accum acc;
  std::vector<int32_t> ci((size_t)nc);
  std::vector<double> cd2((size_t)nc);
  int rc = me_set_cloud(tmp, ME_CLOUD_EST, ce.data(), nc);
  if (rc == ME_OK) rc = me_set_cloud(tmp, ME_CLOUD_GT, cg.data(), nc);
  if (rc == ME_OK) rc = me_eval_nn_accum(tmp, &p, &acc, nullptr);
  if (rc == ME_OK) rc = me_get_nn(tmp, ME_CLOUD_EST, ci.data(), cd2.data());
  if (rc != ME_OK) std::cerr << "ERROR: inlier distance map: " << me_last_error(tmp) << std::endl;
  me_destroy(tmp);
  if (rc != ME_OK) return -1;
  map_3d_render_inlier_ = render::color_by_distance(ce, cd2, dis);
  return 0;
}

inline int MapEvalB200::computeMME() {
  if (!param_.evaluate_mme_) return 0;
  // use_tbb_mme only selects between two CPU threadings of the same arithmetic in the reference (:153-157)
  auto eval_mme = [&](int which, int min_neighbors, int64_t n_total, me_mme_result *out) -> int {
    me_mme_accum acc;
    if (!gpus_.reduce_accum([&](me_ctx *c) { return me_eval_mme_accum_device(c, which, param_.nn_radius_, min_neighbors); }, nullptr,
                            nullptr, which == ME_CLOUD_EST ? &acc : nullptr, which == ME_CLOUD_GT ? &acc : nullptr))
      return -1;
    return me_mme_finalize(&acc, n_total, out) == ME_OK ? 0 : -1;
  };
  if (eval_mme(ME_CLOUD_EST, 10, n_est_, &mme_est_res_) != 0) return fail("me_eval_mme(est)");
  if (param_.save_immediate_result_ && renderEntropy(ME_CLOUD_EST, n_est_, &map_3d_entropy_) != 0) return -1;   // :179
  mme_est = mme_est_res_.mme;
  if (mme_est_res_.n_valid * 100.0 / (double)mme_est_res_.n_total < 0.6)
    std::cerr << "valid points is too small, please check the input point cloud" << std::endl;   // :1732
  min_abs_entropy = mme_est_res_.min_abs_entropy; max_abs_entropy = mme_est_res_.max_abs_entropy;   // :179 -> :700-701
  if (gt_mme()) {
    if (eval_mme(ME_CLOUD_GT, 5, n_gt_, &mme_gt_res_) != 0) return fail("me_eval_mme(gt)");
    if (param_.save_immediate_result_ && renderEntropy(ME_CLOUD_GT, n_gt_, &gt_3d_entropy_) != 0) return -1;      // :181
    mme_gt = mme_gt_res_.mme;
    std::cout << "GT MME Valid_points " << mme_gt_res_.n_valid * 100.0 / (double)mme_gt_res_.n_total << "% " << mme_gt_res_.n_valid
              << " " << mme_gt_res_.n_total << std::endl;
    std::cout << "MME EST-GT: " << mme_est << " " << mme_gt << std::endl;
    min_abs_entropy = mme_gt_res_.min_abs_entropy; max_abs_entropy = mme_gt_res_.max_abs_entropy;   // :181, last call wins
  } else {
    std::cout << "MME EST: " << mme_est << std::endl;
  }
  return 0;
}

inline int MapEvalB200::calculateMetricsWithInitialMatrix() {
  TicToc tic;
  if (!param_.trunc_dist_set_)
    std::cerr << "WARNING: accuracy_level missing: the reference would read an uninitialised trunc_dist_ (map_eval.h:85); using zeros."
              << std::endl;
  me_nn_params p{};
  for (int i = 0; i < 5; ++i) p.tau[i] = param_.trunc_dist_[i];
  p.icp_max_distance = param_.icp_max_distance_;
  p.cutoff_mode = ME_CUTOFF_SQDIST_LE_R;
  p.pairing = param_.geometric_gt_pairing_ ? ME_PAIRING_GEOMETRIC : ME_PAIRING_AS_WRITTEN;
  // path A never calls computeChamferDistance (full_chamfer_dist stays 0, map_eval.h:334); the sums are still cheap,
  // so they are produced and reported on stdout, while the results file keeps the reference's value
  p.want_full_cd = 1;
  p.directions = 3;
  me_nn_accum e2g, g2e;
  if (!gpus_.reduce_accum(
          [&](me_ctx *c) {
            int rc = me_transform(c, ME_CLOUD_EST, param_.initial_matrix_);      // map_3d_->Transform(initial_matrix), :1206
            return rc != ME_OK ? rc : me_eval_nn_accum_device(c, &p);
          },
          &e2g, &g2e, nullptr, nullptr))
    return fail("me_transform / me_eval_nn_accum_device / all-reduce of the NN accumulators");
  if (me_nn_finalize(&p, &e2g, &g2e, n_est_, n_gt_, &nn_) != ME_OK) return fail("me_nn_finalize");
  t_acc = tic.toc() / 1000.0;
  if (param_.accuracy_curve_steps_ > 0 && accuracyCurve(p, e2g, g2e) != 0) return -1;
  if (!param_.distance_quantiles_.empty() && distanceQuantiles() != 0) return -1;
  if (param_.region_size_ > 0.0 && regionErrors() != 0) return -1;
  if (param_.surface_metrics_ && surfaceMetrics() != 0) return -1;
  if (nn_.gt_to_est.n_ub > 0)
    std::cerr << "WARNING: " << nn_.gt_to_est.n_ub << " gt->est pairs index past the end of a cloud (the reference reads out of "
                 "bounds there, map_eval.cpp:1233 vs :1093-1094: undefined behaviour); they are left out of the gt->est statistics, "
                 "so the CD vector / gt->est lines are not comparable with a reference run.  geometric_gt_pairing: true pairs "
                 "the points geometrically instead." << std::endl;
  if (param_.save_immediate_result_ && renderDistances(false) != 0) return -1;
  if (param_.drift_region_size_ > 0.0 && regionDrift() != 0) return -1;
  std::cout << "INFO: Chamfer Distance: " << eigenRow(nn_.cd, 5, 6) << std::endl;
  std::cout << "INFO: F1 Score: " << eigenRow(nn_.f1, 5, 6) << std::endl;
  std::cout << "INFO: est-gt MME: " << mme_est << " " << mme_gt << std::endl;
  std::cout << "INFO: IoU: " << eigenRow(nn_.iou, 5, 6) << std::endl;
  std::cout << "INFO: Full Chamfer distance (not computed by the reference on this path): " << nn_.full_cd << std::endl;
  return 0;
}

// accuracy curve: the pass's NN records at accuracy_curve_steps levels (me_nn_curve_accum_device on every GPU, one NCCL
// all-reduce of the blocks, me_nn_curve_finalize with the reduced accumulators) -> accuracy_curve.txt next to map_results.txt
inline int MapEvalB200::accuracyCurve(const me_nn_params &p, const me_nn_accum &e2g, const me_nn_accum &g2e) {
  const int K = param_.accuracy_curve_steps_;
  std::vector<double> tau(K);
  for (int k = 1; k <= K; ++k) tau[k - 1] = (param_.accuracy_curve_max_ * (double)k) / (double)K;
  std::vector<double> blk;
  if (!gpus_.reduce_curve(tau.data(), K, blk)) return fail("me_nn_curve_accum_device / all-reduce of the accuracy curve");
  std::vector<me_curve_row> rows(K);
  if (me_nn_curve_finalize(&p, &e2g, &g2e, blk.data(), tau.data(), K, n_est_, n_gt_, rows.data()) != ME_OK)
    return fail("me_nn_curve_finalize");
  const std::string path = results_subfolder + "accuracy_curve.txt";
  std::ofstream f(path);
  if (!f.is_open()) {
    std::cerr << "ERROR: cannot write " << path << std::endl;
    return -1;
  }
  f << "tau e2g_n_inlier e2g_mean e2g_rmse e2g_fitness e2g_sigma g2e_n_inlier g2e_mean g2e_rmse g2e_fitness g2e_sigma cd f1 iou\n";
  f << std::fixed << std::setprecision(15);
  for (const me_curve_row &r : rows) {
    f << r.tau;
    for (const me_curve_dir *d : {&r.est_to_gt, &r.gt_to_est})
      f << " " << d->n_inlier << " " << d->mean << " " << d->rmse << " " << d->fitness << " " << d->sigma;
    f << " " << r.cd << " " << r.f1 << " " << r.iou << "\n";
  }
  std::cout << "INFO: accuracy curve (" << K << " levels up to " << param_.accuracy_curve_max_ << ") saved to " << path << std::endl;
  return 0;
}

// distance quantiles: both populations of the pass's NN records at the distance_quantiles probabilities (the me_nn_quantile_*
// loop on every GPU, one NCCL all-reduce of the pass's counts per pass) -> distance_quantiles.txt next to map_results.txt
inline int MapEvalB200::distanceQuantiles() {
  const std::vector<double> &pr = param_.distance_quantiles_;
  const int K = (int)pr.size();
  me_quantile_result res[2];
  for (int pop : {ME_DIST_KEPT, ME_DIST_NN}) {
    if (gpus_.for_each([&](int, me_ctx *c) { return me_nn_quantile_begin(c, pop, pr.data(), K); }) != ME_OK)
      return fail("me_nn_quantile_begin");
    for (int32_t done = 0; !done;) {
      if (!gpus_.reduce_block([](int, me_ctx *c, double **ptr, int32_t *n, int32_t *) { return me_nn_quantile_block(c, ptr, n); }))
        return fail("me_nn_quantile_block / all-reduce of the distance quantile counts");
      if (gpus_.each(me_nn_quantile_step, &done) != ME_OK) return fail("me_nn_quantile_step");
    }
    if (gpus_.each(me_nn_quantile_end, &res[pop]) != ME_OK) return fail("me_nn_quantile_end");
  }
  const std::string path = results_subfolder + "distance_quantiles.txt";
  std::ofstream f(path);
  if (!f.is_open()) {
    std::cerr << "ERROR: cannot write " << path << std::endl;
    return -1;
  }
  f << "# kept: the kept pairs' distances; nn: every query's nearest-neighbour distance.  value: numpy quantile(method=linear)\n";
  f << "population direction n p value lo hi\n";
  f << std::fixed << std::setprecision(15);
  for (int pop : {ME_DIST_KEPT, ME_DIST_NN})
    for (int q = 0; q < 2; ++q) {
      const me_quantile_dir &d = q == 0 ? res[pop].est_to_gt : res[pop].gt_to_est;
      for (int k = 0; k < K; ++k)
        f << (pop == ME_DIST_KEPT ? "kept" : "nn") << " " << (q == 0 ? "est_to_gt" : "gt_to_est") << " " << d.n << " " << pr[k] << " "
          << d.value[k] << " " << d.lo[k] << " " << d.hi[k] << "\n";
    }
  const me_quantile_result &nn = res[ME_DIST_NN];
  f << "hausdorff_est_to_gt " << nn.est_to_gt.max << "\nhausdorff_gt_to_est " << nn.gt_to_est.max << "\nhausdorff " << nn.hausdorff << "\n";
  std::cout << "INFO: Hausdorff distance: " << nn.hausdorff << " (est->gt " << nn.est_to_gt.max << ", gt->est " << nn.gt_to_est.max
            << "); distance quantiles saved to " << path << std::endl;
  return 0;
}

// per-region table: the pass's NN records split by region floor(x / region_size) (me_nn_region_begin on every GPU, one grouped
// NCCL SUM all-reduce of the block's sums and one MAX all-reduce of its maxima) -> region_errors.txt next to map_results.txt
inline int MapEvalB200::regionErrors() {
  const double s = param_.region_size_;
  std::vector<int64_t> n(gpus_.size(), 0);
  if (!gpus_.reduce_block([&](int r, me_ctx *c, double **ptr, int32_t *n_sum, int32_t *n_max) {
        const int rc = me_nn_region_begin(c, s, &n[r]);
        return rc != ME_OK ? rc : me_nn_region_block(c, ptr, n_sum, n_max);
      }))
    return fail("me_nn_region_begin / all-reduce of the region block");
  std::vector<me_region_row> rows((size_t)n[0]);
  if (me_nn_region_end(ctx_, rows.data(), n[0]) != ME_OK) return fail("me_nn_region_end");
  const std::string path = results_subfolder + "region_errors.txt";
  std::ofstream f(path);
  if (!f.is_open()) {
    std::cerr << "ERROR: cannot write " << path << std::endl;
    return -1;
  }
  f << "min_x min_y min_z max_x max_y max_z n_est n_gt";
  for (const char *d : {"e2g", "g2e"}) {
    f << " " << d << "_n_corr";
    for (const char *field : {"n_inlier", "mean", "rmse", "fitness"})
      for (int k = 1; k <= 5; ++k) f << " " << d << "_" << field << "_" << k;
    f << " " << d << "_max_d " << d << "_mean_nn";
  }
  for (const char *field : {"cd", "f1", "iou"})
    for (int k = 1; k <= 5; ++k) f << " " << field << "_" << k;
  f << "\n" << std::fixed << std::setprecision(15);
  for (const me_region_row &r : rows) {
    f << r.min[0] << " " << r.min[1] << " " << r.min[2] << " " << r.max[0] << " " << r.max[1] << " " << r.max[2] << " " << r.n_est
      << " " << r.n_gt;
    for (const me_region_dir *d : {&r.est_to_gt, &r.gt_to_est}) {
      f << " " << d->n_corr;
      for (int k = 0; k < 5; ++k) f << " " << d->n_inlier[k];
      for (const double *v : {d->mean, d->rmse, d->fitness})
        for (int k = 0; k < 5; ++k) f << " " << v[k];
      f << " " << d->max_d << " " << d->mean_nn;
    }
    for (const double *v : {r.cd, r.f1, r.iou})
      for (int k = 0; k < 5; ++k) f << " " << v[k];
    f << "\n";
  }
  std::cout << "INFO: errors of " << n[0] << " regions of edge " << s << " saved to " << path << std::endl;
  return 0;
}

// local consistency without a ground truth: the me_consistency_* loop on every GPU for the est cloud (and the gt cloud with
// evaluate_gt_mme), one grouped NCCL SUM all-reduce of the block's sums and one MAX all-reduce of its maxima per cloud ->
// map_consistency.txt next to map_results.txt
inline int MapEvalB200::localConsistency() {
  const double s = param_.consistency_region_size_, r = param_.nn_radius_;
  struct Run {
    int which, m;
    const char *name;
    me_consistency_result whole;
    std::vector<me_consistency_row> rows;
  };
  std::vector<Run> runs;
  runs.push_back(Run{ME_CLOUD_EST, 10, "est", me_consistency_result{}, {}});
  if (gt_mme()) runs.push_back(Run{ME_CLOUD_GT, 5, "gt", me_consistency_result{}, {}});
  for (Run &run : runs) {
    std::vector<int64_t> n(gpus_.size(), 0);
    if (!gpus_.reduce_block([&](int g, me_ctx *c, double **ptr, int32_t *n_sum, int32_t *n_max) {
          const int rc = me_consistency_begin(c, run.which, r, run.m, s, &n[g]);
          return rc != ME_OK ? rc : me_consistency_block(c, ptr, n_sum, n_max);
        }))
      return fail("me_consistency_begin / all-reduce of the consistency block");
    run.rows.resize((size_t)n[0]);
    if (me_consistency_end(ctx_, run.rows.data(), n[0], &run.whole) != ME_OK) return fail("me_consistency_end");
  }
  const std::string path = results_subfolder + "map_consistency.txt";
  std::ofstream f(path);
  if (!f.is_open()) {
    std::cerr << "ERROR: cannot write " << path << std::endl;
    return -1;
  }
  f << std::setprecision(17) << "# local consistency without a ground truth: per point MME's neighbourhood (d2 < r^2), its entropy "
       "and its plane variance (smallest eigenvalue of the covariance, m^2); r = " << r << ", min_neighbors est 10";
  if (runs.size() > 1) f << ", gt 5";
  f << ", region_size " << s << (s > 0.0 ? "" : " (whole map only)")
    << (param_.evaluate_without_gt_ ? "; est as loaded\n" : "; est in the ground truth's frame\n");
  const char *stats = "n_query n_valid n_pv mme mpv mean_plane_std max_pv";
  f << "cloud n_points " << stats << "\n" << std::fixed << std::setprecision(15);
  auto put = [&](int64_t n_points, int64_t nq, int64_t nv, int64_t np, double mme, double mpv, double sd, double mx) {
    f << " " << n_points << " " << nq << " " << nv << " " << np << " " << mme << " " << mpv << " " << sd << " " << mx << "\n";
  };
  for (const Run &run : runs) {
    const me_consistency_result &w = run.whole;
    f << run.name;
    put(w.n_points, w.n_query, w.n_valid, w.n_pv, w.mme, w.mpv, w.mean_plane_std, w.max_pv);
  }
  if (s > 0.0) {
    f << "cloud min_x min_y min_z max_x max_y max_z n_points " << stats << "\n";
    for (const Run &run : runs)
      for (const me_consistency_row &x : run.rows) {
        f << run.name << " " << x.min[0] << " " << x.min[1] << " " << x.min[2] << " " << x.max[0] << " " << x.max[1] << " " << x.max[2];
        put(x.n_points, x.n_query, x.n_valid, x.n_pv, x.mme, x.mpv, x.mean_plane_std, x.max_pv);
      }
  }
  std::cout << "INFO: local consistency:";
  for (size_t i = 0; i < runs.size(); ++i)
    std::cout << (i ? "," : "") << " " << runs[i].name << " MPV " << runs[i].whole.mpv << " m^2, MME " << runs[i].whole.mme;
  std::cout << "; saved to " << path << std::endl;
  return 0;
}

// the mutually orthogonal metric: the me_mom_* loop on every GPU for the est cloud (and the gt cloud with evaluate_gt_mme), one
// grouped NCCL SUM all-reduce of the block per pass -> map_mom.txt next to map_results.txt
inline int MapEvalB200::mom() {
  const double r = param_.nn_radius_;
  const me_mom_params p{param_.mom_angle_deg_, param_.mom_planarity_, param_.mom_min_family_};
  const double s = param_.mom_region_size_;
  struct Run {
    int which, m;
    const char *name;
    me_mom_result res;
    std::vector<me_mom_region_row> rows;
  };
  std::vector<Run> runs;
  runs.push_back(Run{ME_CLOUD_EST, 10, "est", me_mom_result{}, {}});
  if (gt_mme()) runs.push_back(Run{ME_CLOUD_GT, 5, "gt", me_mom_result{}, {}});
  for (Run &run : runs) {
    if (gpus_.for_each([&](int, me_ctx *c) { return me_mom_begin(c, run.which, r, run.m, &p); }) != ME_OK) return fail("me_mom_begin");
    for (int32_t done = 0; !done;) {
      if (!gpus_.reduce_block([](int, me_ctx *c, double **ptr, int32_t *n, int32_t *) { return me_mom_block(c, ptr, n); }))
        return fail("me_mom_block / all-reduce of the MOM block");
      if (gpus_.each(me_mom_step, &done) != ME_OK) return fail("me_mom_step");
    }
    if (gpus_.each(me_mom_end, &run.res) != ME_OK) return fail("me_mom_end");
    if (s <= 0.0) continue;
    // per region: every GPU writes its points into the block, ONE grouped SUM all-reduce
    std::vector<int64_t> n_regions(gpus_.size(), 0);
    if (!gpus_.reduce_block<int64_t>([&](int g, me_ctx *c, double **ptr, int64_t *n, int64_t *) {
          const int rc = me_mom_region_begin(c, s, p.min_family, &n_regions[g]);
          return rc != ME_OK ? rc : me_mom_region_block(c, ptr, n);
        }))
      return fail("me_mom_region_begin / all-reduce of the MOM region block");
    run.rows.resize((size_t)n_regions[0]);
    if (me_mom_region_end(ctx_, run.rows.data(), n_regions[0]) != ME_OK) return fail("me_mom_region_end");
  }
  const std::string path = results_subfolder + "map_mom.txt";
  std::ofstream f(path);
  if (!f.is_open()) {
    std::cerr << "ERROR: cannot write " << path << std::endl;
    return -1;
  }
  static const char *status[] = {"OK", "NO_PLANAR", "NO_SECOND_AXIS", "SMALL_FAMILY"};
  f << std::setprecision(17) << "# mutually orthogonal metric without a ground truth (after Kornilova & Ferrer 2021, this project's "
       "rule): planar points (v <= planarity lambda2) of MME's neighbourhoods, three orthogonal plane families |n . a_j| >= "
       "cos(angle), mom = the sum of the families' median plane variance (m^2); r = " << r << ", min_neighbors est 10";
  if (runs.size() > 1) f << ", gt 5";
  f << ", angle_deg " << p.angle_deg << ", planarity " << p.planarity << ", min_family " << p.min_family
    << (param_.evaluate_without_gt_ ? "; est as loaded\n" : "; est in the ground truth's frame\n");
  f << "cloud n_points n_query n_pv n_planar a1_x a1_y a1_z a2_x a2_y a2_z a3_x a3_y a3_z n_1 mean_1 median_1 n_2 mean_2 median_2 "
       "n_3 mean_3 median_3 mom status\n" << std::fixed << std::setprecision(15);
  for (const Run &run : runs) {
    const me_mom_result &x = run.res;
    f << run.name << " " << x.n_points << " " << x.n_query << " " << x.n_pv << " " << x.n_planar;
    for (int k = 0; k < 9; ++k) f << " " << x.axis[k];
    for (int j = 0; j < 3; ++j) f << " " << x.n[j] << " " << x.mean[j] << " " << x.median[j];
    f << " " << x.mom << " " << (x.status >= 0 && x.status < 4 ? status[x.status] : "?") << "\n";
  }
  std::cout << "INFO: mutually orthogonal metric:";
  for (size_t i = 0; i < runs.size(); ++i)
    std::cout << (i ? "," : "") << " " << runs[i].name << " MOM " << runs[i].res.mom << " m^2 ("
              << status[std::min(3, std::max(0, (int)runs[i].res.status))] << ")";
  std::cout << "; saved to " << path << std::endl;
  if (s <= 0.0) return 0;

  const std::string rpath = results_subfolder + "map_mom_regions.txt";
  std::ofstream rf(rpath);
  if (!rf.is_open()) {
    std::cerr << "ERROR: cannot write " << rpath << std::endl;
    return -1;
  }
  rf << std::setprecision(17) << "# mutually orthogonal metric per region floor(x / s): the MOM call's axes and families, per "
        "region and family the count, mean and exact median plane variance (m^2) of its members, mom = the sum of the medians "
        "(NaN unless every family has min_family members); s = " << s << ", min_family " << p.min_family
     << (param_.evaluate_without_gt_ ? "; est as loaded\n" : "; est in the ground truth's frame\n");
  rf << "cloud min_x min_y min_z max_x max_y max_z n_points n_planar n_1 mean_1 median_1 n_2 mean_2 median_2 n_3 mean_3 median_3 "
        "mom status\n" << std::fixed << std::setprecision(15);
  for (const Run &run : runs)
    for (const me_mom_region_row &x : run.rows) {
      rf << run.name;
      for (int a = 0; a < 3; ++a) rf << " " << (double)x.index[a] * s;
      for (int a = 0; a < 3; ++a) rf << " " << (double)(x.index[a] + 1) * s;
      rf << " " << x.n_points << " " << x.n_planar;
      for (int j = 0; j < 3; ++j) rf << " " << x.n[j] << " " << x.mean[j] << " " << x.median[j];
      rf << " " << x.mom << " " << (x.status >= 0 && x.status < 4 ? status[x.status] : "?") << "\n";
    }
  for (const Run &run : runs) {
    size_t ok = 0, best = 0;
    int best_j = -1;
    for (size_t r = 0; r < run.rows.size(); ++r) {
      const me_mom_region_row &x = run.rows[r];
      ok += x.status == ME_MOM_OK;
      for (int j = 0; j < 3; ++j)
        if (x.n[j] > 0 && (best_j < 0 || x.median[j] > run.rows[best].median[best_j])) { best = r; best_j = j; }
    }
    std::cout << "INFO: MOM per region: " << run.name << " " << run.rows.size() << " regions of " << s << " m, " << ok << " OK";
    if (best_j >= 0) {
      const me_mom_region_row &x = run.rows[best];
      std::cout << "; largest family median " << x.median[best_j] << " m^2 (family " << best_j + 1 << ") in [" << (double)x.index[0] * s
                << ", " << (double)(x.index[0] + 1) * s << "] x [" << (double)x.index[1] * s << ", " << (double)(x.index[1] + 1) * s
                << "] x [" << (double)x.index[2] * s << ", " << (double)(x.index[2] + 1) * s << "]";
    }
    std::cout << "; saved to " << rpath << std::endl;
  }
  return 0;
}

// evaluate_without_gt: the estimate alone, loaded and down-sampled as on the other paths, then MME, local consistency and MOM
inline int MapEvalB200::processWithoutGt() {
  TicToc tic_toc;
  std::cout << "INFO: evaluate_without_gt: only the estimate is evaluated; gt_map_path, registration_methods, accuracy_level, "
               "initial_matrix, evaluate_using_initial, evaluate_gt_mme and vmd_voxel_size are ignored" << std::endl;
  std::string err;
  const std::string est_path = param_.evaluation_map_pcd_path_ + param_.pcd_file_name_;
  if (!cloud_io::read_pcd(est_path, map_3d_, &err, nullptr)) {
    std::cerr << "ERROR: Failed to load point cloud from the specified path." << std::endl;
    return -1;
  }
  if (map_3d_.empty()) {
    std::cerr << "ERROR: the estimated map is empty!" << std::endl;
    return -1;
  }
  if (!gpus_.create(std::max(1, param_.n_gpus_), param_.gpu_device_, 0.0)) return fail("cannot create the GPU context(s)");
  ctx_ = gpus_.ctx(0);
  if (gpus_.size() > 1) std::cout << "INFO: sharding the sweeps over " << gpus_.size() << " GPUs (NCCL all-reduce of the accumulators)" << std::endl;
  std::vector<int64_t> ne(gpus_.size(), (int64_t)(map_3d_.size() / 3));
  if (gpus_.for_each([&](int r, me_ctx *c) {
        int rc = me_set_cloud(c, ME_CLOUD_EST, map_3d_.data(), (int64_t)(map_3d_.size() / 3));
        if (rc == ME_OK && param_.downsample_size > 0) rc = me_voxel_downsample(c, ME_CLOUD_EST, param_.downsample_size, &ne[r]);
        return rc;
      }) != ME_OK)
    return fail("uploading / down-sampling the estimated map");
  if (!(param_.downsample_size > 0)) std::cout << "INFO: downsample_size <= 0: the map is evaluated as loaded." << std::endl;
  n_est_ = ne[0];
  n_gt_ = 0;
  file_result << std::fixed << std::setprecision(15) << "Estimated-Ground Truth point count: " << n_est_ << " / " << 0 << std::endl;
  t1 = tic_toc.toc();
  if (param_.evaluate_mme_) {
    if (computeMME() != 0) return -1;
    t2 = tic_toc.toc();
    if (param_.save_immediate_result_) saveMmeResults();
    else file_result << std::fixed << std::setprecision(5) << "MME: " << mme_est << " " << mme_gt << " " << min_abs_entropy << " "
                     << max_abs_entropy << std::endl;
  }
  if (param_.evaluate_consistency_ && localConsistency() != 0) return -1;
  if (param_.evaluate_mom_ && mom() != 0) return -1;
  return 0;
}

// point-to-plane metrics: the pass's NN records against the tangent plane of each neighbour (the me_nn_surface_* loop on every
// GPU: one grouped NCCL all-gather per cloud that needs working k-NN normals, then one grouped SUM all-reduce of the block's
// sums and one MAX all-reduce of its maxima) -> surface_metrics.txt next to map_results.txt
inline int MapEvalB200::surfaceMetrics() {
  const int G = gpus_.size(), knn = param_.surface_normals_knn_;
  bool own[2];          // the cloud holds normals (from its file, averaged by VoxelDownSample); else working k-NN normals
  {
    std::vector<double> tmp((size_t)std::max(n_est_, n_gt_) * 3);
    for (int w = 0; w < 2; ++w) own[w] = me_get_normals(ctx_, w, tmp.data()) == ME_OK;
  }
  if (gpus_.for_each([&](int, me_ctx *c) { return me_nn_surface_begin(c, knn); }) != ME_OK) return fail("me_nn_surface_begin");
  for (int w : {ME_CLOUD_EST, ME_CLOUD_GT}) {
    std::vector<double *> nrm(G, nullptr);
    std::vector<int64_t> s(G, 0);
    std::vector<int32_t> pend(G, 0);
    if (gpus_.for_each([&](int r, me_ctx *c) {
          const int rc = me_nn_surface_normals_slice(c, w, &nrm[r], &s[r], &pend[r]);
          return rc != ME_OK ? rc : me_synchronize(c);
        }) != ME_OK)
      return fail("me_nn_surface_normals_slice");
    if (pend[0] && !gpus_.allgather_device(nrm, (size_t)s[0] * 3)) return fail("all-gather of the working normals");
  }
  if (!gpus_.reduce_block([](int, me_ctx *c, double **ptr, int32_t *n_sum, int32_t *n_max) {
        return me_nn_surface_block(c, ptr, n_sum, n_max);
      }))
    return fail("me_nn_surface_block / all-reduce of the surface block");
  me_surface_result res;
  if (gpus_.each(me_nn_surface_end, &res) != ME_OK) return fail("me_nn_surface_end");
  const std::string path = results_subfolder + "surface_metrics.txt";
  std::ofstream f(path);
  if (!f.is_open()) {
    std::cerr << "ERROR: cannot write " << path << std::endl;
    return -1;
  }
  auto source = [&](int w) { return own[w] ? std::string("file") : "k-NN (k = " + std::to_string(knn) + ")"; };
  f << "# e = |(p - t) . n| / |n|: the distance of the query point p to the tangent plane of its geometric nearest neighbour t "
       "(normal n); normal consistency = min(1, |m . n| / (|m| |n|)) with the query's normal m; mean_nn = sum of e over every "
       "query / query count; est normals: " << source(ME_CLOUD_EST) << "; gt normals: " << source(ME_CLOUD_GT) << "\n";
  f << "direction n_corr n_no_normal";
  for (const char *field : {"n_inlier", "mean", "rmse", "fitness", "sigma"})
    for (int k = 1; k <= 5; ++k) f << " " << field << "_" << k;
  f << " mean_nn max_e max_e_nn n_nc normal_consistency\n" << std::fixed << std::setprecision(15);
  for (int q = 0; q < 2; ++q) {
    const me_dir_result &d = q == 0 ? res.plane.est_to_gt : res.plane.gt_to_est;
    const me_surface_dir &x = q == 0 ? res.est_to_gt : res.gt_to_est;
    f << (q == 0 ? "est_to_gt" : "gt_to_est") << " " << d.n_corr << " " << x.n_no_normal;
    for (int k = 0; k < 5; ++k) f << " " << d.n_inlier[k];
    for (const double *v : {d.mean, d.rmse, d.fitness, d.sigma})
      for (int k = 0; k < 5; ++k) f << " " << v[k];
    f << " " << d.sum_nn_dist / (double)d.n_source << " " << x.max_e << " " << x.max_e_nn << " " << x.n_nc << " "
      << x.normal_consistency << "\n";
  }
  for (const char *field : {"cd", "f1", "iou"})
    for (int k = 1; k <= 5; ++k) f << field << "_" << k << " ";
  f << "full_cd normal_consistency\n";
  for (const double *v : {res.plane.cd, res.plane.f1, res.plane.iou})
    for (int k = 0; k < 5; ++k) f << v[k] << " ";
  f << res.plane.full_cd << " " << res.normal_consistency << "\n";
  std::cout << "INFO: point-to-plane CD at level 1: " << res.plane.cd[0] << ", normal consistency: " << res.normal_consistency
            << "; surface metrics saved to " << path << std::endl;
  return 0;
}

// drift per region: every region floor(x / drift_region_size) of the estimate aligned to the ground truth on its own (the
// me_drift_* loop on every GPU, one grouped NCCL SUM all-reduce of the 17 values per region per iteration, as the multi-GPU
// loop of performRegistration) -> region_drift.txt next to map_results.txt.  The estimate is restored bit for bit afterwards,
// so it runs after the consumers of the pass's NN records, which it stales.
inline int MapEvalB200::regionDrift() {
  const double s = param_.drift_region_size_;
  const int G = gpus_.size();
  std::vector<int64_t> n(G, 0);
  if (gpus_.for_each([&](int r, me_ctx *c) { return me_drift_begin(c, s, param_.icp_max_distance_, 30, 1e-6, 1e-6, &n[r]); }) != ME_OK)
    return fail("me_drift_begin");
  for (int32_t done = 0; !done;) {
    if (!gpus_.reduce_block([](int, me_ctx *c, double **ptr, int32_t *n_sum, int32_t *) { return me_drift_block(c, ptr, n_sum); }))
      return fail("me_drift_block / all-reduce of the drift block");
    if (gpus_.each(me_drift_step, &done) != ME_OK) return fail("me_drift_step");
  }
  std::vector<std::vector<me_drift_row>> rows(G, std::vector<me_drift_row>((size_t)std::max<int64_t>(n[0], 1)));
  if (gpus_.for_each([&](int r, me_ctx *c) { return me_drift_end(c, rows[r].data(), n[0]); }) != ME_OK) return fail("me_drift_end");
  rows[0].resize((size_t)n[0]);
  const std::string path = results_subfolder + "region_drift.txt";
  std::ofstream f(path);
  if (!f.is_open()) {
    std::cerr << "ERROR: cannot write " << path << std::endl;
    return -1;
  }
  f << "min_x min_y min_z max_x max_y max_z n_est n_corr_before fitness_before rmse_before n_corr fitness rmse shift_x shift_y "
       "shift_z shift_norm angle_rad iterations status";
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j) f << " T" << i << j;
  f << "\n" << std::fixed << std::setprecision(15);
  int64_t converged = 0, worst = -1;
  for (size_t k = 0; k < rows[0].size(); ++k) {
    const me_drift_row &r = rows[0][k];
    f << r.min[0] << " " << r.min[1] << " " << r.min[2] << " " << r.max[0] << " " << r.max[1] << " " << r.max[2] << " " << r.n_est
      << " " << r.n_corr_before << " " << r.fitness_before << " " << r.rmse_before << " " << r.n_corr << " " << r.fitness << " "
      << r.rmse << " " << r.shift[0] << " " << r.shift[1] << " " << r.shift[2] << " " << r.shift_norm << " " << r.angle << " "
      << r.iterations << " " << r.status;
    for (int i = 0; i < 12; ++i) f << " " << r.T[i];
    f << "\n";
    converged += r.status == ME_DRIFT_CONVERGED;
    if (worst < 0 || r.shift_norm > rows[0][(size_t)worst].shift_norm) worst = (int64_t)k;
  }
  std::cout << "INFO: drift of " << n[0] << " regions of edge " << s << " (" << converged << " converged) saved to " << path;
  if (worst >= 0) {
    const me_drift_row &w = rows[0][(size_t)worst];
    std::cout << "; largest shift " << w.shift_norm << " in [" << w.min[0] << ", " << w.max[0] << "] x [" << w.min[1] << ", "
              << w.max[1] << "] x [" << w.min[2] << ", " << w.max[2] << "]";
  }
  std::cout << std::endl;
  return 0;
}

// global_registration: FPFH + RANSAC on context 0 (me_global_registration) on the loaded, down-sampled clouds.  The result
// is a pure function of the clouds, the parameters and the seed, so every context of a multi-GPU run uses context 0's T
// without a collective.  It replaces initial_matrix: path A's transform, path B's T_init.
inline int MapEvalB200::globalRegistration() {
  static const double eye[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  if (!std::equal(param_.initial_matrix_, param_.initial_matrix_ + 16, eye))
    std::cout << "INFO: global_registration is on: its result replaces the initial_matrix of the configuration, which is not "
                 "the identity" << std::endl;
  const double v = param_.global_registration_voxel_size_;
  me_global_reg_params gp{};
  gp.voxel_size = v;
  gp.normal_knn = 30;
  gp.feature_radius = 10.0 * v;
  gp.feature_max_nn = 128;
  gp.mutual_filter = 1;
  gp.max_correspondence_distance = 1.5 * v;
  gp.edge_ratio = 0.9;
  gp.n_hypotheses = param_.global_registration_hypotheses_;
  gp.seed = param_.global_registration_seed_;
  me_global_reg_result gr{};
  TicToc tic;
  if (me_global_registration(ctx_, &gp, &gr) != ME_OK) return fail("me_global_registration");
  std::copy(gr.T, gr.T + 16, param_.initial_matrix_);
  const double fitness = gr.n_correspondences > 0 ? (double)gr.n_inliers / (double)gr.n_correspondences : 0.0;
  std::cout << "INFO: global registration (" << tic.toc() / 1000.0 << " s): " << gr.n_est_features << " / " << gr.n_gt_features
            << " feature points, " << gr.n_correspondences << " correspondences, " << gr.n_inliers << " inliers, rmse "
            << gr.inlier_rmse << "\n" << eigenMatrix4(gr.T, 6) << std::endl;
  file_result << std::fixed << std::setprecision(5) << "Global registration cloud: " << eigenMatrix4(gr.T, 5) << std::endl;
  file_result << std::fixed << std::setprecision(5) << "Global registration: " << fitness << " " << gr.n_inliers << " "
              << gr.n_correspondences << std::endl;
  return 0;
}

inline int MapEvalB200::performRegistration() {
  TicToc tic_toc;
  // performICPRegistration (:1366-1394): ICPConvergenceCriteria() = {1e-6, 1e-6, 30}; the normals loaded with the
  // clouds (down-sampled along with them) are already on the contexts.  On one GPU: me_icp.  On several, every GPU sweeps
  // its query range and estimates its slice of the missing k-NN normals; the slices are all-gathered and the 17 / 29
  // partial sums all-reduced once per iteration, so that every GPU applies the same update and holds the aligned cloud.
  me_icp_result reg{};
  if (gpus_.size() == 1) {
    if (me_icp(ctx_, param_.evaluation_method_, param_.icp_max_distance_, 30, 1e-6, 1e-6, param_.initial_matrix_, &reg) != ME_OK)
      return fail("me_icp");
  } else {
    const int n = gpus_.size();
    std::vector<double *> ptr(n, nullptr);
    std::vector<int64_t> slice(n, 0);
    std::vector<int32_t> pending(n, 0);
    if (gpus_.for_each([&](int, me_ctx *c) {
          return me_icp_begin(c, param_.evaluation_method_, param_.icp_max_distance_, 30, 1e-6, 1e-6, param_.initial_matrix_);
        }) != ME_OK)
      return fail("me_icp_begin");
    for (int which : {ME_CLOUD_EST, ME_CLOUD_GT}) {
      if (gpus_.for_each([&](int r, me_ctx *c) {
            const int rc = me_icp_normals_slice(c, which, &ptr[r], &slice[r], &pending[r]);
            return rc != ME_OK ? rc : me_synchronize(c);
          }) != ME_OK)
        return fail("me_icp_normals_slice");
      if (pending[0] && !gpus_.allgather_device(ptr, (size_t)slice[0] * 3)) return fail("all-gather of the normals");
    }
    for (int32_t done = 0; !done;) {      // the first me_icp_block sweeps
      if (!gpus_.reduce_block([](int, me_ctx *c, double **blk, int32_t *n_sum, int32_t *) { return me_icp_block(c, blk, n_sum); }))
        return fail("me_icp_block / all-reduce of the ICP block");
      if (gpus_.each(me_icp_step, &done) != ME_OK) return fail("me_icp_step");
    }
    if (gpus_.each(me_icp_end, &reg) != ME_OK) return fail("me_icp_end");
  }
  t4 = tic_toc.toc();
  std::cout << "INFO: ICP registration time: " << (t4 - t3) / 1000.0 << " [s]" << std::endl;
  std::cout << "INFO: Aligned transformation: \n" << eigenMatrix4(reg.transformation, 6) << std::endl;
  std::cout << "INFO: ICP overlap ratio: " << reg.fitness << std::endl;
  std::cout << "INFO: ICP correspondences RMSE: " << reg.inlier_rmse << std::endl;
  std::cout << "INFO: ICP correspondences size: " << reg.n_corr << std::endl;
  file_result << std::fixed << std::setprecision(5) << "Aligned cloud: " << eigenMatrix4(reg.transformation, 5) << std::endl;
  file_result << std::fixed << std::setprecision(5) << "Aligned results: " << reg.fitness << " " << reg.n_corr << std::endl;
  // calculateMetrics(reg) (:1147-1202): est->gt on the ICP correspondences (NN within R, strict), gt->est through
  // EvaluateRegistration(gt, est, R) (:1168), cd_vec (:1171), full Chamfer distance (:1194)
  TicToc tic;
  me_nn_params p{};
  for (int i = 0; i < 5; ++i) p.tau[i] = param_.trunc_dist_[i];
  p.icp_max_distance = param_.icp_max_distance_;
  p.cutoff_mode = ME_CUTOFF_DIST_LT_R;
  p.pairing = ME_PAIRING_GEOMETRIC;
  p.want_full_cd = 1;
  p.directions = 3;
  me_nn_accum e2g, g2e;
  if (!gpus_.reduce_accum([&](me_ctx *c) { return me_eval_nn_accum_device(c, &p); }, &e2g, &g2e, nullptr, nullptr))
    return fail("me_eval_nn_accum_device / all-reduce of the NN accumulators");
  if (me_nn_finalize(&p, &e2g, &g2e, n_est_, n_gt_, &nn_) != ME_OK) return fail("me_nn_finalize");
  t_acc = tic.toc() / 1000.0;
  if (param_.accuracy_curve_steps_ > 0 && accuracyCurve(p, e2g, g2e) != 0) return -1;
  if (!param_.distance_quantiles_.empty() && distanceQuantiles() != 0) return -1;
  if (param_.region_size_ > 0.0 && regionErrors() != 0) return -1;
  if (param_.surface_metrics_ && surfaceMetrics() != 0) return -1;
  if (param_.save_immediate_result_ && renderDistances(true) != 0) return -1;
  if (param_.drift_region_size_ > 0.0 && regionDrift() != 0) return -1;
  full_chamfer_dist = nn_.full_cd;
  t_fcd = t_acc;
  t5 = tic_toc.toc();
  std::cout << "INFO: Chamfer Distance: " << eigenRow(nn_.cd, 5, 6) << std::endl;
  std::cout << "INFO: Full Chamfer Distance: " << full_chamfer_dist << std::endl;
  return 0;
}

inline int MapEvalB200::calculateVMD() {
  TicToc ticToc;
  int64_t n_rows = 0;
  double *rows = nullptr;
  if (me_eval_awd(ctx_, param_.vmd_voxel_size_, 100, 5, &awd_, &n_rows, &rows) != ME_OK) return fail("me_eval_awd");
  std::cout << "Build voxel map: " << awd_.n_voxels_gt << std::endl;
  std::cout << "Build voxel map: " << awd_.n_voxels_est << std::endl;
  std::cout << "Update active/old/new voxel num: " << awd_.n_active << " " << awd_.n_old << " " << awd_.n_new << std::endl;
  t_v = ticToc.toc();
  std::ofstream output_file(results_subfolder + "voxel_errors.txt");
  if (!output_file.is_open()) {
    std::cerr << "ERROR: Failed to open voxel error output file." << std::endl;
    me_free(rows);
    return 0;   // the reference returns early here (map_eval.cpp:257-260)
  }
  for (int64_t r = 0; r < n_rows; ++r) {   // map_eval.cpp:292-302: default ostream formatting, one space apart
    const double *v = rows + r * 27;
    for (int c = 0; c < 27; ++c) {
      if (c == 10 || c == 11) output_file << (long long)v[c];
      else output_file << v[c];
      output_file << (c == 26 ? "" : " ");
    }
    output_file << std::endl;
  }
  output_file.close();
  if (param_.enable_debug) std::cout << "INFO: Voxel errors results saved to " << results_subfolder + "voxel_errors.txt" << std::endl;
  vmd = awd_.awd;
  t_vmd = ticToc.toc();
  std::cout << "INFO: Calculated VMD: " << vmd << std::endl;
  std::vector<double> ws(n_rows);
  for (int64_t r = 0; r < n_rows; ++r) ws[r] = rows[r * 27 + 9];
  me_free(rows);
  std::sort(ws.begin(), ws.end());   // map_eval.cpp:330-341
  std::ofstream cdf_file(results_subfolder + "voxel_wasserstein_cdf.txt");
  if (!cdf_file.is_open()) {
    std::cerr << "ERROR: Failed to open CDF output file." << std::endl;
    return 0;
  }
  for (size_t i = 0; i < ws.size(); ++i) cdf_file << ws[i] << " " << static_cast<double>(i + 1) / ws.size() << std::endl;
  cdf_file.close();
  t_cdf = ticToc.toc();
  if (param_.enable_debug) std::cout << "INFO: CDF results saved to " << results_subfolder + "voxel_wasserstein_cdf.txt" << std::endl;
  scs_overall = awd_.scs;
  t_scs = ticToc.toc();
  std::cout << "INFO: Spatial Consistency Score (SCS): " << scs_overall << std::endl;
  return 0;
}

// the Gaussian 2-Wasserstein distance per voxel (me_eval_w2 on GPU 0, as calculateVMD) -> map_w2.txt and voxel_w2.txt next to
// map_results.txt
inline int MapEvalB200::voxelW2() {
  const double v = param_.vmd_voxel_size_;
  me_w2_result res{};
  int64_t n_rows = 0;
  double *rows = nullptr;
  if (me_eval_w2(ctx_, v, param_.w2_min_points_, 5, &res, &n_rows, &rows) != ME_OK) return fail("me_eval_w2");
  std::vector<double> table(rows, rows + (size_t)n_rows * ME_W2_ROW_COLS);
  me_free(rows);
  const std::string path = results_subfolder + "map_w2.txt", rpath = results_subfolder + "voxel_w2.txt";
  std::ofstream f(path);
  if (!f.is_open()) {
    std::cerr << "ERROR: cannot write " << path << std::endl;
    return -1;
  }
  f << std::setprecision(17) << "# Gaussian 2-Wasserstein distance per voxel floor(x / v): W2 = sqrt(offset^2 + shape^2), offset = "
       "|mu_est - mu_gt|, shape = Bures(Sigma_gt, Sigma_est), Sigma = M2 / (n - 1) (m); scs over W2 with radius 5; v = " << v
    << ", min_points " << param_.w2_min_points_ << "; est in the ground truth's frame\n";
  f << "aw2 mean_offset mean_shape scs n_pairs n_scs n_voxels_est n_voxels_gt\n" << std::fixed << std::setprecision(15)
    << res.aw2 << " " << res.mean_offset << " " << res.mean_shape << " " << res.scs << " " << res.n_pairs << " " << res.n_scs << " "
    << res.n_voxels_est << " " << res.n_voxels_gt << "\n";
  std::ofstream rf(rpath);
  if (!rf.is_open()) {
    std::cerr << "ERROR: cannot write " << rpath << std::endl;
    return -1;
  }
  rf << std::setprecision(17) << "# one row per voxel pair of map_w2.txt (sigma as xx xy xz yy yz zz, m^2); v = " << v << "\n";
  rf << "min_x min_y min_z n_gt n_est mu_est_x mu_est_y mu_est_z mu_gt_x mu_gt_y mu_gt_z sig_est_xx sig_est_xy sig_est_xz "
        "sig_est_yy sig_est_yz sig_est_zz sig_gt_xx sig_gt_xy sig_gt_xz sig_gt_yy sig_gt_yz sig_gt_zz offset shape w2\n";
  for (int64_t r = 0; r < n_rows; ++r) {
    const double *x = table.data() + r * ME_W2_ROW_COLS;
    for (int c = 0; c < ME_W2_ROW_COLS; ++c) {
      if (c == 3 || c == 4) rf << (long long)x[c];
      else rf << x[c];
      rf << (c + 1 == ME_W2_ROW_COLS ? "\n" : " ");
    }
  }
  std::cout << "INFO: Gaussian 2-Wasserstein: AW2 " << res.aw2 << " m (offset " << res.mean_offset << ", shape " << res.mean_shape
            << "), SCS " << res.scs << ", " << res.n_pairs << " pairs; saved to " << path << " and " << rpath << std::endl;
  return 0;
}

inline void MapEvalB200::saveMmeResults() {   // map_eval.cpp:392-421
  if (!param_.evaluate_mme_) return;
  file_result << std::fixed << std::setprecision(5) << "MME: " << mme_est << " " << mme_gt << " " << min_abs_entropy << " "
              << max_abs_entropy << std::endl;
  if (param_.enable_debug) std::cout << "INFO: MME results saved to " << results_file_path << std::endl;
  // map_eval.cpp:404-412
  if (!render::write_pcd(results_subfolder + "map_entropy.pcd", map_3d_entropy_)) std::cerr << "ERROR: cannot write map_entropy.pcd" << std::endl;
  else if (param_.enable_debug) std::cout << "INFO: Saved rendered entropy map to " << results_subfolder + "map_entropy.pcd" << std::endl;
  if (gt_mme()) {
    if (!render::write_pcd(results_subfolder + "gt_entropy.pcd", gt_3d_entropy_)) std::cerr << "ERROR: cannot write gt_entropy.pcd" << std::endl;
    else if (param_.enable_debug)
      std::cout << "INFO: Saved rendered entropy ground truth map to " << results_subfolder + "gt_entropy.pcd" << std::endl;
  }
}

inline void MapEvalB200::saveRegistrationResults() {   // map_eval.cpp:424-482
  if (param_.enable_debug) {
    std::cout << "INFO: AC+MME Time: " << t_acc + (t2 - t1) / 1000.0 << std::endl;
    std::cout << "INFO: CD+MME Time: " << t_fcd + (t2 - t1) / 1000.0 << std::endl;
    std::cout << "INFO: AWD+SCS Time: " << t_v / 1000.0 + (t_vmd - t_v) / 1000.0 + (t_scs - t_cdf) / 1000.0 << std::endl;
  }
  file_result << std::fixed << std::setprecision(15) << "RMSE/AC: " << eigenRow(nn_.est_to_gt.rmse, 5, 15) << std::endl;
  file_result << std::fixed << std::setprecision(15) << "Comp: " << eigenRow(nn_.est_to_gt.fitness, 5, 15) << std::endl;
  file_result << std::fixed << std::setprecision(5) << "FULL CD: " << full_chamfer_dist << std::endl;   // 0 on path A, as the reference
  file_result << std::fixed << std::setprecision(5) << "VMD: " << vmd << std::endl;
  file_result << std::fixed << std::setprecision(5) << "SCS: " << scs_overall << std::endl;
  file_result << "Time load-MME-mesh-ICP-Metric-AC-FCD: " << t1 / 1000.0 << " " << (t2 - t1) / 1000.0 << " " << (t3) / 1000.0 << " "
              << (t4 - t3) / 1000.0 << " " << (t5 - t4) / 1000.0 << " " << t_acc << " " << t_fcd << std::endl;
  file_result << "VMD Time voxelization-WD-CDF-SCS: " << t_v / 1000.0 << " " << (t_vmd - t_v) / 1000.0 << " "
              << (t_cdf - t_vmd) / 1000.0 << " " << (t_scs - t_cdf) / 1000.0 << std::endl;
  file_result << "AC+MME Time: " << t_acc + (t2 - t1) / 1000.0 << std::endl;
  file_result << "CD+MME Time: " << t_fcd + (t2 - t1) / 1000.0 << std::endl;
  file_result << "AWD+SCS Time: " << t_v / 1000.0 + (t_vmd - t_v) / 1000.0 + (t_scs - t_cdf) / 1000.0 << std::endl;
  file_result.close();
  if (param_.enable_debug) std::cout << "INFO: Results saved to " << results_subfolder + "map_results.txt" << std::endl;
  // map_eval.cpp:485-499
  if (!render::write_pcd(results_subfolder + "raw_rendered_dis_map.pcd", map_3d_render_raw_)) std::cerr << "ERROR: cannot write raw_rendered_dis_map.pcd" << std::endl;
  else if (param_.enable_debug) std::cout << "INFO: Saved raw distance error map to " << results_subfolder + "raw_rendered_dis_map.pcd" << std::endl;
  if (!render::write_pcd(results_subfolder + "inlier_rendered_dis_map.pcd", map_3d_render_inlier_)) std::cerr << "ERROR: cannot write inlier_rendered_dis_map.pcd" << std::endl;
  else if (param_.enable_debug) std::cout << "INFO: Saved inlier distance error map to " << results_subfolder + "inlier_rendered_dis_map.pcd" << std::endl;
  // map_eval.cpp:502-507: the estimated cloud as held here (down-sampled and registered, like map_3d_ there), no normals
  if (param_.evaluate_noised_gt_) {
    int64_t n = 0;
    std::vector<double> xyz;
    bool ok = me_get_cloud(ctx_, ME_CLOUD_EST, nullptr, 0, &n) == ME_OK;
    if (ok) {
      xyz.resize((size_t)n * 3);
      ok = me_get_cloud(ctx_, ME_CLOUD_EST, xyz.data(), n, &n) == ME_OK;
    }
    if (!ok || !render::write_pcd_xyz(results_subfolder + "noise_gt_map.pcd", xyz)) std::cerr << "ERROR: cannot write noise_gt_map.pcd" << std::endl;
    else if (param_.enable_debug) std::cout << "INFO: Saved noisy ground truth map to " << results_subfolder + "noise_gt_map.pcd" << std::endl;
  }
}
