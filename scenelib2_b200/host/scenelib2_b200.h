// scenelib2_b200.h — C++ host shim keeping the reference's hot-path class surface
// (SceneLib2::MonoSLAM / Kalman / Feature / Camera, scenelib2/monoslam.h:73-218, kalman.h:44-53,
// feature.h:56-143, camera.h:42-78) on top of the C ABI of libsl2b200.so (include/sl2b200.h).
//
// Same names, same argument meaning, same `bool`/`int` returns as the reference; the arithmetic
// runs in the sm_90a kernels.  Host mirrors (xv_, Pxx_, per-feature y_/Pxy_/Pyy_/
// matrix_block_list_, h_/z_/S_/flags/counters) are refreshed before GoOneStep / the Kalman calls
// return, because the reference's GUI reads them on every redraw (graphic/graphictool.cpp:130-168).
// Also here: the file-based FrameGrabber / FileGrabber (framegrabber/*.h).
// Out of scope (SURVEY.md §2): GUI, USB camera grabber, creation / conversion of partially-initialised features
// (their per-frame cycle is one C-ABI call, sl2_measure_partial_features; the shim keeps the pending templates).
#pragma once
#include <atomic>
#include <mutex>
#include <queue>
#include <string>
#include <thread>
#include <vector>

#include "sl2_compat.h"

struct sl2_ctx;

namespace SceneLib2 {

class MonoSLAM;

class Camera {  // camera.h:42-78 (members used by the example and the hot path)
 public:
  void SetCameraParameters(int camera_width, int camera_height, double fku, double fkv, double u0,
                           double v0, double kd1, int sd);
  int width_ = 0, height_ = 0;
  double kd1_ = 0, fku_ = 0, fkv_ = 0;
  Eigen::Vector2d centre_;
  double measurement_sd_ = 0;
};

class MotionModel {  // motion_model.h: constants + func_xp
 public:
  void func_xp(const Eigen::VectorXd &xv);
  Eigen::VectorXd xpRES_;
  Eigen::Vector3d rRES_;
  const int kPositionStateSize_ = 7, kStateSize_ = 13, kControlSize_ = 3;
};

class Feature {  // feature.h:56-143
 public:
  Eigen::VectorXd y_, xp_org_;
  Eigen::MatrixXd Pyy_, Pxy_;
  cv::Mat patch_;
  std::vector<Eigen::MatrixXd> matrix_block_list_;
  Eigen::VectorXd h_, z_, nu_;
  Eigen::MatrixXd dh_by_dxv_, dh_by_dy_, R_, S_;
  int label_ = 0, position_in_list_ = 0, position_in_total_state_vector_ = 0;
  int attempted_measurements_of_feature_ = 0, successful_measurements_of_feature_ = 0;
  bool selected_flag_ = false, scheduled_for_termination_flag_ = false;
  bool successful_measurement_flag_ = false, fully_initialised_flag_ = true;
};

class Kalman {  // kalman.h:44-53
 public:
  void KalmanFilterPredict(MonoSLAM *monoslam, Eigen::Vector3d &u);
  void KalmanFilterUpdate(MonoSLAM *monoslam);
};

// ---- frame ingestion (framegrabber/framegrabber.h:47-77, filegrabber.h:50-72) ------------------
// The producer side of the main loop (examples/MonoSlamSceneLib1.cpp:132-142): a reader thread fills a
// bounded queue (50 frames, framegrabber.cpp:94-103) from the sorted files of a directory tree.
// cv::imread(path, 0) is replaced by a PGM decoder (P5 binary and P2 ASCII, 8-bit); a file that is not
// a PGM yields an empty Mat like a failed imread.  The USB camera grabber is not built.
struct Frame {
  int frame_id;
  cv::Mat data;
};

class FrameGrabber;

class FileGrabber {
 public:
  FileGrabber();
  ~FileGrabber();
  void Init(const std::string &path, FrameGrabber *frame_grabber);  // throws std::runtime_error
  void operator()();                                                // reader loop (own thread)
  cv::Mat GetImageFile(const std::string &file_full_path);
  size_t NumberOfFiles() const { return files_vec_.size(); }

 private:
  void ProcessFiles(const std::string &directory);
  std::vector<std::string> files_vec_;
  FrameGrabber *frame_grabber_ = nullptr;
  std::atomic<bool> initialised_{false};
  int frame_id_ = 0;
  std::thread fg_thread_;
};

class FrameGrabber {
 public:
  FrameGrabber();
  ~FrameGrabber();
  void Init(const std::string &dev, const bool mode);  // mode == false: directory of image files
  bool GetFrame(int frame_id, Frame *frame);            // false while the queue is empty
  void SetFrame(const Frame &frame);
  bool IsFrameBufferFull();
  // not in the reference: true once every file has been handed out (lets a batch driver stop)
  bool Exhausted();

 private:
  std::queue<Frame> frame_buffer_;
  std::mutex fg_mutex_;
  FileGrabber *file_grabber_ = nullptr;
  int handed_out_ = 0;
};

// graphic/graphictool.h: the two entry points the main loop calls (examples/MonoSlamSceneLib1.cpp:124-126,
// 144-151).  The GUI bodies are out of scope (SURVEY.md 2): headless no-ops that count their calls.
class GraphicTool {
 public:
  explicit GraphicTool(MonoSLAM *monoslam) : monoslam_(monoslam) {}
  void Draw3dScene(const bool &chk_display_trajectory, const bool &chk_display_3d_features,
                   const bool &chk_display_3d_uncertainties);
  void DrawAR(cv::Mat frame, const bool &chk_rectify_image_display, const bool &chk_display_trajectory,
              const bool &chk_display_3d_features, const bool &chk_display_3d_uncertainties,
              const bool &chk_display_2d_descriptors, const bool &chk_display_2d_search_regions,
              const bool &chk_display_initialisation);
  MonoSLAM *monoslam_;
  long draw_calls_ = 0;
};

// a feature the user (InitialiseFeature) or the detector (InitialiseAutoFeature) has asked for: template and
// pixel are kept; turning it into a map feature needs the depth particles of the partially-initialised
// machinery (monoslam.cpp:1262, feature_init_info.cpp), whose per-frame cycle is sl2_measure_partial_features
struct PendingFeature {
  cv::Mat patch;
  int u, v;
};

class MonoSLAM {  // monoslam.h:73-218 (hot-path subset + the calls of examples/MonoSlamSceneLib1.cpp)
 public:
  MonoSLAM();
  ~MonoSLAM();

  void Init(const std::string &config_path);
  bool GoOneStep(cv::Mat frame, bool save_trajectory, bool enable_mapping);
  void print_robot_state();
  // monoslam.h:79-81,142: caller-side surface of the example's buttons
  void InitialiseFeature(cv::Mat frame);      // template at the selected image location (uu_, vv_)
  void InitialiseAutoFeature(cv::Mat frame);  // Shi-Tomasi best patch of the central region, then the above
  bool SavePatch();                           // template of the marked feature -> patch.png

  int auto_select_n_features(int n);
  int make_measurements(cv::Mat image);
  bool measure_feature(cv::Mat image, cv::Mat patch, Eigen::VectorXd &z, const Eigen::VectorXd &h,
                       const Eigen::MatrixXd &S);
  bool elliptical_search(const cv::Mat &image, const cv::Mat &patch, const Eigen::Vector2d centre,
                         const Eigen::Matrix2d &PuInv, int *u, int *v, const int uBOXSIZE);
  // Shi-Tomasi detector (monoslam.cpp:1043-1205)
  double set_image_selection_automatically(cv::Mat frame, int ustart, int vstart, int ufinish,
                                           int vfinish);
  void find_best_patch_inside_region(const cv::Mat &image, int *ubest, int *vbest, double *evbest,
                                     const int BOXSIZE, int ustart, int vstart, int ufinish,
                                     int vfinish);
  void construct_total_state(Eigen::VectorXd &V);
  void construct_total_covariance(Eigen::MatrixXd &M);
  void normalise_state();
  void delete_bad_features();
  void mark_feature_by_lab(int lab);
  bool delete_feature();
  void AddNewKnownFeature(const Eigen::VectorXd &y, const Eigen::VectorXd &xp,
                          const std::string &identifier);
  // same, with the template given in memory (the reference reads it with cv::imread)
  void AddNewKnownFeature(const Eigen::VectorXd &y, const Eigen::VectorXd &xp, const cv::Mat &patch);

  Camera *camera_ = nullptr;
  MotionModel *motion_model_ = nullptr;
  Kalman *kalman_ = nullptr;
  FrameGrabber *frame_grabber_ = nullptr;  // monoslam.h:163; created by Init() when the cfg names an input
  GraphicTool *graphic_tool_ = nullptr;    // monoslam.h:164
  std::vector<PendingFeature> pending_features_;

  Eigen::VectorXd xv_;
  Eigen::MatrixXd Pxx_;
  std::vector<Feature *> feature_list_;
  std::vector<Feature *> selected_feature_list_;
  std::vector<Eigen::Vector3d> trajectory_store_;

  int number_of_visible_features_ = 0, next_free_label_ = 0, marked_feature_label_ = -1;
  int total_state_size_ = 13, successful_measurement_vector_size_ = 0;
  double kDeltaT_ = 0.033333333;
  int kNumberOfFeaturesToSelect_ = 10, kNumberOfFeaturesToKeepVisible_ = 12;
  int minimum_attempted_measurements_of_feature_ = 10;
  double successful_match_fraction_ = 0.5;
  int uu_ = 0, vv_ = 0;
  bool location_selected_flag_ = false;
  const int kBoxSize_;
  const double kNoSigma_, kCorrThresh2_, kCorrelationSigmaThreshold_;

  // ---- device side (not in the reference) ----------------------------------------------------
  // Creates the GPU context; called by Init(), or directly when the map is built in code.
  // max_features bounds the map size; device = CUDA ordinal.  Throws std::runtime_error on failure.
  void CreateDevice(int max_features = 100, int device = 0);
  void UploadMap();    // host y_/xp_org_/patch_/xv_/P blocks -> device (whole map; first upload)
  void SyncFromDevice();  // device state + per-feature results -> host mirrors
  sl2_ctx *ctx_ = nullptr;

 private:
  bool map_dirty_ = true;
};

}  // namespace SceneLib2
