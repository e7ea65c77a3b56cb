// sl2_headless.cpp — headless analogue of the reference's only executable
// (examples/MonoSlamSceneLib1.cpp:132-142: GetFrame -> GoOneStep) without Pangolin/GLUT:
//   sl2_headless <config.cfg> <frames.raw> <width> <height> <nframes> [out_state.txt]
//   sl2_headless <config.cfg> <directory of PGM frames> [out_state.txt]
// frames.raw = nframes * height * width bytes (8-bit gray); a directory is read through the
// FrameGrabber / FileGrabber pair like the reference's file mode (sorted file names, reader thread,
// bounded queue).  Prints the camera state per frame and optionally writes the final total state and
// covariance for comparison.
// SL2_HEADLESS_LOAD_STATE=file resumes from a MonoSLAM::SaveState file (loaded after Init, before the first frame);
// SL2_HEADLESS_SAVE_STATE=file writes one after the last frame.  A run split at frame k into two runs chained by the
// file tracks exactly like the unsplit run.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <filesystem>
#include <fstream>
#include <iostream>
#include <thread>
#include <vector>

#include "scenelib2_b200.h"

static void report(SceneLib2::MonoSLAM *m, int t) {
  std::printf("frame %d visible %d measured %d features %zu\n", t, m->number_of_visible_features_,
              m->successful_measurement_vector_size_ / 2, m->feature_list_.size());
}

int main(int argc, char **argv) {
  const bool dir_mode = argc >= 3 && std::filesystem::is_directory(argv[2]);
  if ((!dir_mode && argc < 6) || argc < 3) {
    std::fprintf(stderr, "usage: %s config.cfg frames.raw width height nframes [out.txt]\n"
                         "       %s config.cfg frames_dir [out.txt]\n", argv[0], argv[0]);
    return 2;
  }
  const char *out_path = dir_mode ? (argc > 3 ? argv[3] : nullptr) : (argc > 6 ? argv[6] : nullptr);
  try {
    SceneLib2::MonoSLAM *g_monoslam = new SceneLib2::MonoSLAM();
    g_monoslam->Init(argv[1]);
    if (const char *load = std::getenv("SL2_HEADLESS_LOAD_STATE")) g_monoslam->LoadState(load);
    if (dir_mode) {
      // examples/MonoSlamSceneLib1.cpp:132-142: poll GetFrame, step on every frame that arrives
      SceneLib2::FrameGrabber grabber;
      grabber.Init(argv[2], false);
      int frame_id = 0;
      SceneLib2::Frame frame;
      while (!grabber.Exhausted()) {
        if (!grabber.GetFrame(frame_id, &frame)) {
          std::this_thread::sleep_for(std::chrono::milliseconds(1));
          continue;
        }
        if (frame.data.empty()) continue;  // not an image (imread would have returned an empty Mat)
        g_monoslam->GoOneStep(frame.data, true, false);
        report(g_monoslam, frame_id++);
      }
    } else {
      const int W = std::atoi(argv[3]), H = std::atoi(argv[4]), T = std::atoi(argv[5]);
      std::vector<unsigned char> buf((size_t)W * H * T);
      std::ifstream f(argv[2], std::ios::binary);
      if (!f.read(reinterpret_cast<char *>(buf.data()), (std::streamsize)buf.size())) {
        std::fprintf(stderr, "cannot read %s\n", argv[2]);
        return 2;
      }
      // SL2_HEADLESS_REPEAT=k: benchmark mode -- the frames are replayed k times without per-frame output and the
      // rate a SceneLib2 caller sees is printed: GoOneStep with the frame upload and BOTH host-mirror refreshes
      // (every Feature's y_/Pxy_/Pyy_/matrix_block_list_, monoslam.cpp:574-614) inside the timed region
      const char *rep = std::getenv("SL2_HEADLESS_REPEAT");
      const int repeat = rep ? std::max(1, std::atoi(rep)) : 1;
      if (rep) {
        cv::Mat warm(H, W, CV_8UC1, buf.data());
        g_monoslam->GoOneStep(warm, false, false);
      }
      const auto t0 = std::chrono::steady_clock::now();
      for (int k = 0; k < repeat; ++k)
        for (int t = 0; t < T; ++t) {
          cv::Mat frame(H, W, CV_8UC1, buf.data() + (size_t)t * W * H);
          g_monoslam->GoOneStep(frame, true, false);
          if (!rep) report(g_monoslam, t);
        }
      if (rep) {
        const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        std::printf("shim_frames_per_s %.3f frames %d features %zu measured %d\n", repeat * T / sec, repeat * T,
                    g_monoslam->feature_list_.size(), g_monoslam->successful_measurement_vector_size_ / 2);
      }
    }
    g_monoslam->print_robot_state();
    if (const char *save = std::getenv("SL2_HEADLESS_SAVE_STATE")) g_monoslam->SaveState(save);
    if (out_path) {
      Eigen::VectorXd V;
      Eigen::MatrixXd M;
      g_monoslam->construct_total_state(V);
      g_monoslam->construct_total_covariance(M);
      std::ofstream o(out_path);
      o.precision(17);
      o << V.size() << "\n";
      for (int i = 0; i < V.size(); ++i) o << V(i) << "\n";
      for (int j = 0; j < M.cols(); ++j)
        for (int i = 0; i < M.rows(); ++i) o << M(i, j) << "\n";
    }
    delete g_monoslam;
  } catch (const std::exception &e) {
    std::fprintf(stderr, "error: %s\n", e.what());
    return 1;
  }
  return 0;
}
