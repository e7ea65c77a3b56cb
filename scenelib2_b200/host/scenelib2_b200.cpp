// scenelib2_b200.cpp — implementation of the host shim over the C ABI (see scenelib2_b200.h).
// Control flow mirrors MonoSLAM::GoOneStep (scenelib2/monoslam.cpp:108-180); every arithmetic
// step is a call into libsl2b200.so.  No CPU fallback: a failing device call throws.
#include "scenelib2_b200.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <filesystem>
#include <fstream>
#include <iostream>
#include <map>
#include <sstream>
#include <stdexcept>

#include "../../include/sl2b200.h"
#include "bmp_decode.h"
#include "jpeg_decode.h"
#include "png_decode.h"

namespace SceneLib2 {

namespace {

void check(sl2_ctx *ctx, int rc, const char *what) {
  if (rc < 0) throw std::runtime_error(std::string(what) + ": " + sl2_last_error(ctx));
}

// `key = value;` files as read by pangolin::ParseVarsFile (monoslam.cpp:1578): '#' comments,
// one assignment per line, trailing ';'.
std::map<std::string, std::string> parse_vars_file(const std::string &path) {
  std::ifstream f(path);
  if (!f) throw std::runtime_error("cannot open config " + path);
  std::map<std::string, std::string> kv;
  std::string line;
  while (std::getline(f, line)) {
    const size_t hash = line.find('#');
    if (hash != std::string::npos) line.erase(hash);
    const size_t eq = line.find('=');
    if (eq == std::string::npos) continue;
    auto trim = [](std::string s) {
      const char *ws = " \t\r\n;";
      const size_t a = s.find_first_not_of(ws), b = s.find_last_not_of(ws);
      return a == std::string::npos ? std::string() : s.substr(a, b - a + 1);
    };
    kv[trim(line.substr(0, eq))] = trim(line.substr(eq + 1));
  }
  return kv;
}
double num(const std::map<std::string, std::string> &kv, const std::string &k, double def) {
  auto it = kv.find(k);
  return it == kv.end() ? def : std::atof(it->second.c_str());
}

// PNM decoder standing in for cv::imread(path, 0) (feature.cpp:119, filegrabber.cpp:106-109): PBM / PGM / PPM, ASCII
// (P1 P2 P3) and binary (P4 P5 P6), '#' comments in the header, with the conversions OpenCV's reader applies
// (tests/test_host_shim.py compares every variant with cv2.imread(path, 0) where OpenCV is installed):
//   bitmaps          1 -> 0, 0 -> 255
//   maxval <= 255    binary samples as they are; ASCII samples scaled v * 255 / maxval when maxval < 255
//   maxval  > 255    16-bit samples (binary: big-endian), high byte
//   colour           Y = (R*4899 + G*9617 + B*1868 + 8192) >> 14 on the 8-bit samples
// Returns an empty Mat for anything else (cv::imread returns an empty Mat when it cannot decode).
cv::Mat decode_pgm_bytes(const std::vector<uint8_t> &b) {
  // hand-rolled header parser (no formatted stream extraction: the library is also loaded into foreign processes)
  size_t pos = 0;
  auto skip = [&]() {
    for (;;) {
      while (pos < b.size() && (b[pos] == ' ' || b[pos] == '\t' || b[pos] == '\n' || b[pos] == '\r')) ++pos;
      if (pos < b.size() && b[pos] == '#') {
        while (pos < b.size() && b[pos] != '\n') ++pos;
        continue;
      }
      return;
    }
  };
  auto number = [&](int &v) {
    skip();
    if (pos >= b.size() || b[pos] < '0' || b[pos] > '9') return false;
    long t = 0;
    while (pos < b.size() && b[pos] >= '0' && b[pos] <= '9' && t < 100000000) t = t * 10 + (b[pos++] - '0');
    v = (int)t;
    return true;
  };
  if (b.size() < 7 || b[0] != 'P' || b[1] < '1' || b[1] > '6') return cv::Mat();
  const int kind = b[1] - '0';
  const bool binary = kind >= 4, bitmap = kind == 1 || kind == 4, colour = kind == 3 || kind == 6;
  pos = 2;
  int w = 0, h = 0, maxval = 1;
  if (!number(w) || !number(h) || (!bitmap && !number(maxval))) return cv::Mat();
  if (w <= 0 || h <= 0 || maxval <= 0 || maxval > 65535 || w > 16384 || h > 16384) return cv::Mat();
  cv::Mat m(h, w, CV_8UC1);
  const int ch = colour ? 3 : 1;
  const bool wide = maxval > 255;
  auto to8 = [&](int v, bool ascii) {  // one sample -> 8 bits
    if (wide) return (v >> 8) & 255;
    if (ascii && maxval < 255) return v * 255 / maxval;
    return v & 255;
  };
  auto luma = [](int r, int g, int bl) { return (r * 4899 + g * 9617 + bl * 1868 + 8192) >> 14; };
  if (binary) ++pos;  // the single whitespace byte after the header
  if (bitmap) {
    if (binary) {
      const size_t rowb = ((size_t)w + 7) / 8;
      if (pos + rowb * h > b.size()) return cv::Mat();
      for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x)
          m.data[(size_t)y * w + x] = ((b[pos + rowb * y + x / 8] >> (7 - x % 8)) & 1) ? 0 : 255;
    } else {
      for (size_t i = 0; i < (size_t)w * h; ++i) {  // digits may be packed without white space
        skip();
        if (pos >= b.size() || (b[pos] != '0' && b[pos] != '1')) return cv::Mat();
        m.data[i] = b[pos++] == '1' ? 0 : 255;
      }
    }
    return m;
  }
  const size_t count = (size_t)w * h;
  if (binary) {
    const size_t bps = wide ? 2 : 1;
    if (pos + count * ch * bps > b.size()) return cv::Mat();
    const uint8_t *q = b.data() + pos;
    for (size_t i = 0; i < count; ++i) {
      int v[3];
      for (int c = 0; c < ch; ++c) v[c] = to8(wide ? (q[(i * ch + c) * 2] << 8) | q[(i * ch + c) * 2 + 1] : q[i * ch + c], false);
      m.data[i] = (unsigned char)(colour ? luma(v[0], v[1], v[2]) : v[0]);
    }
  } else {
    for (size_t i = 0; i < count; ++i) {
      int v[3];
      for (int c = 0; c < ch; ++c) {
        if (!number(v[c])) return cv::Mat();
        v[c] = to8(v[c], true);
      }
      m.data[i] = (unsigned char)(colour ? luma(v[0], v[1], v[2]) : v[0]);
    }
  }
  return m;
}

// cv::imread(path, 0) of the reference (filegrabber.cpp:106-109, feature.cpp:119): PNM, PNG, JPEG or BMP -> 8-bit gray; an
// unreadable / unsupported file gives an empty Mat like a failed imread
cv::Mat decode_image(const std::string &path) {
  std::vector<uint8_t> bytes;
  if (FILE *f = std::fopen(path.c_str(), "rb")) {
    std::fseek(f, 0, SEEK_END);
    const long sz = std::ftell(f);
    std::fseek(f, 0, SEEK_SET);
    if (sz > 0) {
      bytes.resize((size_t)sz);
      if (std::fread(bytes.data(), 1, bytes.size(), f) != bytes.size()) bytes.clear();
    }
    std::fclose(f);
  }
  if (bytes.size() >= 8 && bytes[0] == 0x89 && bytes[1] == 'P' && bytes[2] == 'N' && bytes[3] == 'G') {
    std::vector<uint8_t> gray;
    int w = 0, h = 0;
    if (!sl2png::decode_gray(bytes.data(), bytes.size(), gray, w, h)) return cv::Mat();
    cv::Mat m(h, w, CV_8UC1);
    std::memcpy(m.data, gray.data(), gray.size());
    return m;
  }
  if (bytes.size() >= 2 && bytes[0] == 'B' && bytes[1] == 'M') {
    std::vector<uint8_t> gray;
    int w = 0, h = 0;
    if (!sl2bmp::decode_gray(bytes.data(), bytes.size(), gray, w, h)) return cv::Mat();
    cv::Mat m(h, w, CV_8UC1);
    std::memcpy(m.data, gray.data(), gray.size());
    return m;
  }
  if (bytes.size() >= 4 && bytes[0] == 0xFF && bytes[1] == 0xD8) {
    std::vector<uint8_t> gray;
    int w = 0, h = 0;
    if (!sl2jpeg::decode_gray(bytes.data(), bytes.size(), gray, w, h)) return cv::Mat();
    cv::Mat m(h, w, CV_8UC1);
    std::memcpy(m.data, gray.data(), gray.size());
    return m;
  }
  return decode_pgm_bytes(bytes);
}

cv::Mat read_pgm(const std::string &path) {  // known-feature templates: a missing patch is an error
  cv::Mat m = decode_image(path);
  if (m.empty()) throw std::runtime_error("cannot read patch image " + path);
  return m;
}

}  // namespace

void Camera::SetCameraParameters(int w, int h, double fku, double fkv, double u0, double v0,
                                 double kd1, int sd) {
  width_ = w;
  height_ = h;
  fku_ = fku;
  fkv_ = fkv;
  centre_(0) = u0;
  centre_(1) = v0;
  kd1_ = kd1;
  measurement_sd_ = sd;
}

void MotionModel::func_xp(const Eigen::VectorXd &xv) {  // motion_model.cpp:219-222
  xpRES_.resize(7);
  for (int i = 0; i < 7; ++i) xpRES_(i) = xv(i);
  for (int i = 0; i < 3; ++i) rRES_(i) = xv(i);
}

MonoSLAM::MonoSLAM()
    : kBoxSize_(11), kNoSigma_(3.0), kCorrThresh2_(0.40), kCorrelationSigmaThreshold_(10.0) {}

MonoSLAM::~MonoSLAM() {
  if (ctx_) sl2_destroy(ctx_);
  for (Feature *f : feature_list_) delete f;
  delete camera_;
  delete motion_model_;
  delete kalman_;
  delete frame_grabber_;
  delete graphic_tool_;
}

void GraphicTool::Draw3dScene(const bool &, const bool &, const bool &) { ++draw_calls_; }
void GraphicTool::DrawAR(cv::Mat, const bool &, const bool &, const bool &, const bool &, const bool &,
                         const bool &, const bool &) {
  ++draw_calls_;
}

// monoslam.cpp:1574-1969, minus GUI / grabber / particle parameters
void MonoSLAM::Init(const std::string &config_path) {
  const auto kv = parse_vars_file(config_path);
  camera_ = new Camera();
  camera_->SetCameraParameters((int)num(kv, "cam.width", 0), (int)num(kv, "cam.height", 0),
                               (int)num(kv, "cam.fku", 0), (int)num(kv, "cam.fkv", 0),
                               (int)num(kv, "cam.u0", 0), (int)num(kv, "cam.v0", 0),
                               num(kv, "cam.kd1", 0.0), (int)num(kv, "cam.sd", 0));
  motion_model_ = new MotionModel();
  kalman_ = new Kalman();
  kDeltaT_ = num(kv, "params.delta_t", 0.0);
  kNumberOfFeaturesToSelect_ = (int)num(kv, "params.number_of_features_to_select", 0);
  kNumberOfFeaturesToKeepVisible_ = (int)num(kv, "params.number_of_features_to_keep_visible", 0);
  xv_.resize(13);
  const char *names[13] = {"state.rw_x", "state.rw_y", "state.rw_z", "state.qwr_w", "state.qwr_x",
                           "state.qwr_y", "state.qwr_z", "state.vw_x", "state.vw_y", "state.vw_z",
                           "state.ww_x", "state.ww_y", "state.ww_z"};
  for (int i = 0; i < 13; ++i) xv_(i) = num(kv, names[i], 0.0);
  Pxx_.resize(13, 13);
  for (int i = 0; i < 13; ++i)
    for (int j = 0; j < 13; ++j) {
      std::ostringstream k;
      k << "state.pxx" << i << "_" << j;
      Pxx_(i, j) = num(kv, k.str(), 0.0);
    }
  const size_t slash = config_path.find_last_of('/');
  const std::string dir = slash == std::string::npos ? "" : config_path.substr(0, slash + 1);
  for (int fidx = 1; fidx <= SL2_MAX_FEATURES; ++fidx) {
    std::ostringstream p;
    p << "f" << fidx << ".";
    auto it = kv.find(p.str() + "identifier");
    if (it == kv.end()) break;
    Eigen::VectorXd y(3), xp(7);
    y(0) = num(kv, p.str() + "yi_x", 0);
    y(1) = num(kv, p.str() + "yi_y", 0);
    y(2) = num(kv, p.str() + "yi_z", 0);
    for (int i = 0; i < 7; ++i) {
      std::ostringstream k;
      k << p.str() << "xp_org_" << i;
      xp(i) = num(kv, k.str(), 0);
    }
    const std::string id = it->second;
    AddNewKnownFeature(y, xp, (id.size() && id[0] == '/') ? id : dir + id);
  }
  CreateDevice((int)num(kv, "device.max_features", 100), (int)num(kv, "device.ordinal", 0));
  UploadMap();
  // monoslam.cpp:1959-1963: GUI tool and frame source (file mode only; input.mode = true is the USB camera)
  graphic_tool_ = new GraphicTool(this);
  frame_grabber_ = new FrameGrabber();
  const auto in = kv.find("input.name");
  if (in != kv.end() && in->second != "empty" && num(kv, "input.mode", 0) == 0) {
    const std::string name = in->second;
    frame_grabber_->Init((name.size() && name[0] == '/') ? name : dir + name, false);
  }
}

void MonoSLAM::CreateDevice(int max_features, int device) {
  if (!camera_) throw std::runtime_error("CreateDevice: camera parameters not set");
  if (!motion_model_) motion_model_ = new MotionModel();
  if (!kalman_) kalman_ = new Kalman();
  sl2_config cfg;
  sl2_default_config(&cfg);
  cfg.device = device;
  cfg.width = camera_->width_;
  cfg.height = camera_->height_;
  cfg.boxsize = kBoxSize_;
  cfg.max_features = max_features;
  cfg.number_of_features_to_select = kNumberOfFeaturesToSelect_;
  cfg.fku = camera_->fku_;
  cfg.fkv = camera_->fkv_;
  cfg.u0 = camera_->centre_(0);
  cfg.v0 = camera_->centre_(1);
  cfg.kd1 = camera_->kd1_;
  cfg.sd = camera_->measurement_sd_;
  cfg.delta_t = kDeltaT_;
  cfg.minimum_attempted_measurements_of_feature = minimum_attempted_measurements_of_feature_;
  cfg.successful_match_fraction = successful_match_fraction_;
  const int rc = sl2_create(&cfg, &ctx_);
  if (rc != 0) throw std::runtime_error(std::string("sl2_create: ") + sl2_last_error(nullptr));
}

// monoslam.cpp:1278-1289 + feature.cpp:108-149
void MonoSLAM::AddNewKnownFeature(const Eigen::VectorXd &y, const Eigen::VectorXd &xp,
                                  const cv::Mat &patch) {
  Feature *nf = new Feature();
  nf->y_ = y;
  nf->xp_org_ = xp;
  nf->patch_ = patch;
  nf->label_ = next_free_label_;
  nf->position_in_list_ = (int)feature_list_.size();
  nf->position_in_total_state_vector_ = total_state_size_;
  nf->Pxy_.resize(13, 3);
  nf->Pyy_.resize(3, 3);
  for (int i = 0; i < nf->position_in_list_; ++i) nf->matrix_block_list_.push_back(Eigen::MatrixXd(3, 3));
  nf->h_.resize(2);
  nf->z_.resize(2);
  nf->nu_.resize(2);
  nf->dh_by_dxv_.resize(2, 13);
  nf->dh_by_dy_.resize(2, 3);
  nf->R_.resize(2, 2);
  nf->S_.resize(2, 2);
  feature_list_.push_back(nf);
  total_state_size_ += 3;
  ++next_free_label_;
  if (ctx_ && !map_dirty_) {
    // the device already holds the map: grow it in place (rows / columns of P appended on the device, nothing
    // re-uploaded) -- the mirror of delete_feature
    if (patch.rows != kBoxSize_ || patch.cols != kBoxSize_) throw std::runtime_error("feature patch must be BOXSIZE x BOXSIZE");
    std::vector<uint8_t> pt((size_t)kBoxSize_ * kBoxSize_);
    for (int r = 0; r < kBoxSize_; ++r) std::memcpy(&pt[(size_t)r * kBoxSize_], patch.data + r * patch.step, kBoxSize_);
    check(ctx_, sl2_append_feature(ctx_, 0, y.data(), xp.data(), pt.data(), nullptr), "sl2_append_feature");
  } else {
    map_dirty_ = true;
  }
}
void MonoSLAM::AddNewKnownFeature(const Eigen::VectorXd &y, const Eigen::VectorXd &xp,
                                  const std::string &identifier) {
  AddNewKnownFeature(y, xp, read_pgm(identifier));
}

void MonoSLAM::construct_total_state(Eigen::VectorXd &V) {  // monoslam.cpp:501-512
  V.resize(total_state_size_);
  for (int i = 0; i < 13; ++i) V(i) = xv_(i);
  int pos = 13;
  for (Feature *f : feature_list_) {
    for (int i = 0; i < 3; ++i) V(pos + i) = f->y_(i);
    pos += 3;
  }
}

void MonoSLAM::construct_total_covariance(Eigen::MatrixXd &M) {  // monoslam.cpp:518-546
  M.resize(total_state_size_, total_state_size_);
  for (int i = 0; i < 13; ++i)
    for (int j = 0; j < 13; ++j) M(i, j) = Pxx_(i, j);
  int xpos = 13;
  for (Feature *f : feature_list_) {
    for (int i = 0; i < 13; ++i)
      for (int j = 0; j < 3; ++j) M(i, xpos + j) = M(xpos + j, i) = f->Pxy_(i, j);
    int ypos = 13;
    for (const Eigen::MatrixXd &b : f->matrix_block_list_) {
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) M(ypos + i, xpos + j) = M(xpos + j, ypos + i) = b(i, j);
      ypos += 3;
    }
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) M(ypos + i, xpos + j) = f->Pyy_(i, j);
    xpos += 3;
  }
}

void MonoSLAM::UploadMap() {
  const int n = (int)feature_list_.size();
  std::vector<double> y((size_t)n * 3), xp((size_t)n * 7);
  std::vector<uint8_t> patches((size_t)n * kBoxSize_ * kBoxSize_);
  for (int i = 0; i < n; ++i) {
    Feature *f = feature_list_[i];
    for (int k = 0; k < 3; ++k) y[i * 3 + k] = f->y_(k);
    for (int k = 0; k < 7; ++k) xp[i * 7 + k] = f->xp_org_(k);
    if (f->patch_.rows != kBoxSize_ || f->patch_.cols != kBoxSize_)
      throw std::runtime_error("feature patch must be BOXSIZE x BOXSIZE");
    for (int r = 0; r < kBoxSize_; ++r)
      std::memcpy(&patches[((size_t)i * kBoxSize_ + r) * kBoxSize_], f->patch_.data + r * f->patch_.step,
                  kBoxSize_);
  }
  check(ctx_, sl2_set_features(ctx_, 0, n, y.data(), xp.data(), patches.data()), "sl2_set_features");
  Eigen::VectorXd V;
  Eigen::MatrixXd M;
  construct_total_state(V);
  construct_total_covariance(M);
  check(ctx_, sl2_set_state(ctx_, 0, V.data(), M.data()), "sl2_set_state");
  map_dirty_ = false;
}

void MonoSLAM::SyncFromDevice() {  // fill_states / fill_covariances, monoslam.cpp:574-614
  const int nfeat = sl2_num_features(ctx_, 0);
  check(ctx_, nfeat, "sl2_num_features");
  const int n = 13 + 3 * nfeat;
  total_state_size_ = n;
  std::vector<double> x(n), P((size_t)n * n);
  check(ctx_, sl2_get_state(ctx_, 0, x.data(), P.data()), "sl2_get_state");
  auto Pat = [&](int i, int j) { return P[(size_t)i + (size_t)j * n]; };
  for (int i = 0; i < 13; ++i) xv_(i) = x[i];
  for (int i = 0; i < 13; ++i)
    for (int j = 0; j < 13; ++j) Pxx_(i, j) = Pat(i, j);
  std::vector<double> h(2 * nfeat), z(2 * nfeat), S(4 * nfeat), J(26 * nfeat), Jy(6 * nfeat),
      R(4 * nfeat), nu(2 * nfeat);
  std::vector<uint8_t> flags(nfeat);
  std::vector<int32_t> att(nfeat), suc(nfeat), rank(nfeat);
  check(ctx_, sl2_get_features(ctx_, 0, h.data(), z.data(), S.data(), flags.data(), att.data(),
                               suc.data(), rank.data()), "sl2_get_features");
  check(ctx_, sl2_get_feature_jacobians(ctx_, 0, J.data(), Jy.data(), R.data(), nu.data()),
        "sl2_get_feature_jacobians");
  selected_feature_list_.assign(nfeat, nullptr);
  int nsel = 0;
  for (int i = 0; i < nfeat; ++i) {
    Feature *f = feature_list_[i];
    const int pos = 13 + 3 * i;
    f->position_in_list_ = i;
    f->position_in_total_state_vector_ = pos;
    for (int k = 0; k < 3; ++k) f->y_(k) = x[pos + k];
    for (int r = 0; r < 13; ++r)
      for (int c = 0; c < 3; ++c) f->Pxy_(r, c) = Pat(r, pos + c);
    f->matrix_block_list_.resize(i, Eigen::MatrixXd(3, 3));
    for (int j = 0; j < i; ++j)
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) f->matrix_block_list_[j](r, c) = Pat(13 + 3 * j + r, pos + c);
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) f->Pyy_(r, c) = Pat(pos + r, pos + c);
    for (int k = 0; k < 2; ++k) {
      f->h_(k) = h[2 * i + k];
      f->z_(k) = z[2 * i + k];
      f->nu_(k) = nu[2 * i + k];
    }
    for (int k = 0; k < 4; ++k) {
      f->S_.data()[k] = S[4 * i + k];
      f->R_.data()[k] = R[4 * i + k];
    }
    for (int k = 0; k < 26; ++k) f->dh_by_dxv_.data()[k] = J[26 * i + k];
    for (int k = 0; k < 6; ++k) f->dh_by_dy_.data()[k] = Jy[6 * i + k];
    f->selected_flag_ = (flags[i] & 1) != 0;
    f->successful_measurement_flag_ = (flags[i] & 2) != 0;
    f->attempted_measurements_of_feature_ = att[i];
    f->successful_measurements_of_feature_ = suc[i];
    if (rank[i] >= 0) {
      selected_feature_list_[rank[i]] = f;
      ++nsel;
    }
  }
  selected_feature_list_.resize(nsel);
}

void MonoSLAM::SaveState(const std::string &path) {
  if (!ctx_) throw std::runtime_error("SaveState: Init()/CreateDevice() has not been called");
  if (map_dirty_) UploadMap();
  std::vector<uint8_t> blob(sl2_snapshot_bytes(ctx_));
  size_t size = 0;
  check(ctx_, sl2_save_streams(ctx_, 0, 1, blob.data(), blob.size(), &size), "sl2_save_streams");
  std::ofstream o(path, std::ios::binary);
  if (!o.write(reinterpret_cast<const char *>(blob.data()), (std::streamsize)size))
    throw std::runtime_error("SaveState: cannot write " + path);
}

void MonoSLAM::LoadState(const std::string &path) {
  if (!ctx_) throw std::runtime_error("LoadState: Init()/CreateDevice() has not been called");
  std::ifstream f(path, std::ios::binary);
  const std::vector<uint8_t> blob((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  if (!f.eof() && f.fail()) throw std::runtime_error("LoadState: cannot read " + path);
  if (blob.size() < sizeof(sl2_snapshot_header)) throw std::runtime_error("LoadState: " + path + " is not a snapshot");
  check(ctx_, sl2_load_streams(ctx_, 0, 1, blob.data(), blob.size()), "sl2_load_streams");
  sl2_snapshot_header h;
  std::memcpy(&h, blob.data(), sizeof h);
  const size_t nf = (size_t)h.nfeat, box = (size_t)h.boxsize;
  sl2_snapshot_sections L;
  check(ctx_, sl2_snapshot_layout(h.nfeat, h.boxsize, &L), "sl2_snapshot_layout");
  const size_t o_xp = L.field[0], o_tp = L.templates;  // xp_org, the templates
  for (Feature *g : feature_list_) delete g;
  feature_list_.clear();
  selected_feature_list_.clear();
  total_state_size_ = 13;
  next_free_label_ = 0;
  marked_feature_label_ = -1;
  for (size_t i = 0; i < nf; ++i) {
    Feature *g = new Feature();
    g->y_.resize(3);
    g->xp_org_.resize(7);
    std::memcpy(g->xp_org_.data(), blob.data() + o_xp + 56 * i, 56);
    g->patch_ = cv::Mat((int)box, (int)box, CV_8UC1);
    for (size_t r = 0; r < box; ++r) std::memcpy(g->patch_.data + r * g->patch_.step, blob.data() + o_tp + (i * box + r) * box, box);
    g->label_ = next_free_label_++;
    g->Pxy_.resize(13, 3);
    g->Pyy_.resize(3, 3);
    g->h_.resize(2);
    g->z_.resize(2);
    g->nu_.resize(2);
    g->dh_by_dxv_.resize(2, 13);
    g->dh_by_dy_.resize(2, 3);
    g->R_.resize(2, 2);
    g->S_.resize(2, 2);
    feature_list_.push_back(g);
    total_state_size_ += 3;
  }
  // the stream's camera travels with the blob
  camera_->width_ = h.cam.width;
  camera_->height_ = h.cam.height;
  camera_->fku_ = h.cam.fku;
  camera_->fkv_ = h.cam.fkv;
  camera_->centre_(0) = h.cam.u0;
  camera_->centre_(1) = h.cam.v0;
  camera_->kd1_ = h.cam.kd1;
  camera_->measurement_sd_ = h.cam.sd;
  kDeltaT_ = h.cam.delta_t;
  kNumberOfFeaturesToSelect_ = h.cam.number_of_features_to_select;
  map_dirty_ = false;
  SyncFromDevice();  // y_, P blocks, counters, flags and the last step's results
  number_of_visible_features_ = h.nvisible;
  successful_measurement_vector_size_ = 2 * h.nmeas;
}

void Kalman::KalmanFilterPredict(MonoSLAM *m, Eigen::Vector3d &u) {  // kalman.cpp:50-69
  if (!m->ctx_) throw std::runtime_error("KalmanFilterPredict: no device context");
  check(m->ctx_, sl2_ekf_predict(m->ctx_, 0, u.data()), "sl2_ekf_predict");
}

void Kalman::KalmanFilterUpdate(MonoSLAM *m) {  // kalman.cpp:72-119 (+ normalise, symmetrise)
  check(m->ctx_, sl2_ekf_update_measured(m->ctx_, 0), "sl2_ekf_update_measured");
}

int MonoSLAM::auto_select_n_features(int n) {  // monoslam.cpp:187-254
  (void)n;  // the device uses sl2_config::number_of_features_to_select (set from the same cfg key)
  const int nv = sl2_predict_measurements(ctx_, 0);
  check(ctx_, nv, "sl2_predict_measurements");
  return nv;
}

int MonoSLAM::make_measurements(cv::Mat image) {  // monoslam.cpp:336-359
  check(ctx_, sl2_set_frame(ctx_, 0, 0, image.data, image.step), "sl2_set_frame");
  const int cnt = sl2_make_measurements(ctx_, 0, 0);
  check(ctx_, cnt, "sl2_make_measurements");
  successful_measurement_vector_size_ = 2 * cnt;
  return cnt;
}

// monoslam.cpp:401-477.  `patch` must be the template of one of the map's features (the only way
// the reference calls it, monoslam.cpp:349,378): it is identified by its pixel pointer.
bool MonoSLAM::elliptical_search(const cv::Mat &image, const cv::Mat &patch,
                                 const Eigen::Vector2d centre, const Eigen::Matrix2d &PuInv, int *u,
                                 int *v, const int uBOXSIZE) {
  if (uBOXSIZE != kBoxSize_) throw std::runtime_error("elliptical_search: BOXSIZE mismatch");
  if (map_dirty_) UploadMap();
  int32_t idx = -1;
  for (size_t i = 0; i < feature_list_.size(); ++i)
    if (feature_list_[i]->patch_.data == patch.data) idx = (int32_t)i;
  if (idx < 0) throw std::runtime_error("elliptical_search: patch is not a map feature's template");
  check(ctx_, sl2_set_frame(ctx_, 0, 0, image.data, image.step), "sl2_set_frame");
  const double c[2] = {centre(0), centre(1)};
  const double p[3] = {PuInv(0, 0), PuInv(0, 1), PuInv(1, 1)};
  int32_t uu = -1, vv = -1;
  uint8_t found = 0;
  check(ctx_, sl2_patch_search(ctx_, 0, 0, 1, &idx, c, p, &uu, &vv, &found, nullptr), "sl2_patch_search");
  if (uu >= 0) {  // quirk Q6: *u,*v are only written when a candidate was accepted
    *u = uu;
    *v = vv;
  }
  return found != 0;
}

// monoslam.cpp:368-386 (LLT of S, Sinv = Linv^T Linv, then elliptical_search)
bool MonoSLAM::measure_feature(cv::Mat image, cv::Mat patch, Eigen::VectorXd &z,
                               const Eigen::VectorXd &h, const Eigen::MatrixXd &S) {
  const double l00 = std::sqrt(S(0, 0)), l10 = S(1, 0) / l00;
  const double l11 = std::sqrt(S(1, 1) - l10 * l10);
  const double x00 = 1.0 / l00, x10 = (0.0 - l10 * x00) / l11, x11 = 1.0 / l11;
  Eigen::Matrix2d Sinv;
  Sinv(0, 0) = x00 * x00 + x10 * x10;
  Sinv(0, 1) = Sinv(1, 0) = x10 * x11;
  Sinv(1, 1) = x11 * x11;
  Eigen::Vector2d c;
  c(0) = h(0);
  c(1) = h(1);
  int u = 0, v = 0;
  if (!elliptical_search(image, patch, c, Sinv, &u, &v, kBoxSize_)) return false;
  z(0) = (double)u;
  z(1) = (double)v;
  return true;
}

// monoslam.cpp:1070-1194 (Shi-Tomasi criterion); *ubest/*vbest keep their values when nothing
// beats evbest = 0, like the reference
void MonoSLAM::find_best_patch_inside_region(const cv::Mat &image, int *ubest, int *vbest,
                                             double *evbest, const int BOXSIZE, int ustart,
                                             int vstart, int ufinish, int vfinish) {
  if (BOXSIZE != kBoxSize_) throw std::runtime_error("find_best_patch_inside_region: BOXSIZE mismatch");
  check(ctx_, sl2_set_frame(ctx_, 0, 0, image.data, image.step), "sl2_set_frame");
  const int32_t region[4] = {ustart, vstart, ufinish, vfinish};
  int32_t u = *ubest, v = *vbest;
  check(ctx_, sl2_find_best_patch(ctx_, 0, 0, 1, region, &u, &v, evbest), "sl2_find_best_patch");
  *ubest = u;
  *vbest = v;
}

double MonoSLAM::set_image_selection_automatically(cv::Mat frame, int ustart, int vstart,
                                                   int ufinish, int vfinish) {  // monoslam.cpp:1043-1054
  double evbest = 0;
  find_best_patch_inside_region(frame, &uu_, &vv_, &evbest, kBoxSize_, ustart, vstart, ufinish, vfinish);
  location_selected_flag_ = true;
  return evbest;
}

void MonoSLAM::normalise_state() {  // monoslam.cpp:616-637
  check(ctx_, sl2_normalise_state(ctx_, 0), "sl2_normalise_state");
}

void MonoSLAM::mark_feature_by_lab(int lab) { marked_feature_label_ = lab; }  // monoslam.cpp:743-766

bool MonoSLAM::delete_feature() {  // monoslam.cpp:770-812
  if (marked_feature_label_ == -1) return false;
  for (size_t i = 0; i < feature_list_.size(); ++i) {
    if (feature_list_[i]->label_ != marked_feature_label_) continue;
    check(ctx_, sl2_delete_feature(ctx_, 0, (int)i), "sl2_delete_feature");
    delete feature_list_[i];
    feature_list_.erase(feature_list_.begin() + i);
    total_state_size_ -= 3;
    marked_feature_label_ = -1;
    return true;
  }
  return false;
}

void MonoSLAM::delete_bad_features() {  // monoslam.cpp:644-703
  for (size_t i = 0; i < feature_list_.size();) {
    Feature *f = feature_list_[i];
    if (f->attempted_measurements_of_feature_ >= minimum_attempted_measurements_of_feature_ &&
        double(f->successful_measurements_of_feature_) / double(f->attempted_measurements_of_feature_) <
            successful_match_fraction_) {
      mark_feature_by_lab(f->label_);
      delete_feature();
    } else {
      ++i;
    }
  }
}

// monoslam.cpp:108-180, tracking only (enable_mapping is accepted and ignored: map growth is out of
// scope, SURVEY.md §2 #10-#12)
bool MonoSLAM::GoOneStep(cv::Mat frame, bool save_trajectory, bool enable_mapping) {
  (void)enable_mapping;
  if (!ctx_) throw std::runtime_error("GoOneStep: Init()/CreateDevice() has not been called");
  if (map_dirty_) UploadMap();
  Eigen::Vector3d u;
  kalman_->KalmanFilterPredict(this, u);
  number_of_visible_features_ = auto_select_n_features(kNumberOfFeaturesToSelect_);
  successful_measurement_vector_size_ = 0;
  if (number_of_visible_features_ > 0) make_measurements(frame);
  // Kalman update + normalise_state + symmetrise are one device call.  It runs on EVERY frame: with nothing
  // selected or matched it leaves the state alone but still applies P = 0.5 P + 0.5 P^T, which the reference
  // does unconditionally at the end of GoOneStep (monoslam.cpp:143-150), and books the attempt counters.
  kalman_->KalmanFilterUpdate(this);
  SyncFromDevice();
  const size_t features_before = feature_list_.size();
  delete_bad_features();
  if (feature_list_.size() != features_before) {  // the map shrank: mirror the compacted device state again
    total_state_size_ = 13 + 3 * (int)feature_list_.size();
    SyncFromDevice();
  }
  motion_model_->func_xp(xv_);
  if (save_trajectory) {
    trajectory_store_.push_back(motion_model_->rRES_);
    if (trajectory_store_.size() > 1000) trajectory_store_.erase(trajectory_store_.begin());
  }
  return true;
}

// monoslam.cpp:1495-1541 (caller side): the template under the selected location becomes a pending feature
void MonoSLAM::InitialiseFeature(cv::Mat frame) {
  if (!location_selected_flag_ || frame.empty()) return;
  const int half = (kBoxSize_ - 1) / 2;
  if (uu_ - half < 0 || vv_ - half < 0 || uu_ + half >= frame.cols || vv_ + half >= frame.rows) return;
  PendingFeature p;
  p.patch = cv::Mat(kBoxSize_, kBoxSize_, CV_8UC1);
  for (int r = 0; r < kBoxSize_; ++r)
    std::memcpy(p.patch.data + r * p.patch.step, frame.data + (size_t)(vv_ - half + r) * frame.step + (uu_ - half),
                kBoxSize_);
  p.u = uu_;
  p.v = vv_;
  pending_features_.push_back(p);
  location_selected_flag_ = false;
}

void MonoSLAM::InitialiseAutoFeature(cv::Mat frame) {  // monoslam.cpp:1535-1541 -> AutoInitialiseFeature
  if (frame.empty() || !ctx_) return;
  // the reference searches an 80 x 60 box placed by the predicted motion (monoslam.cpp:823-1032); without a
  // motion prior the shim takes the central box
  const int bw = 80, bh = 60;
  const int us = (frame.cols - bw) / 2, vs = (frame.rows - bh) / 2;
  if (set_image_selection_automatically(frame, us, vs, us + bw, vs + bh) > 0.0) InitialiseFeature(frame);
}

bool MonoSLAM::SavePatch() {  // monoslam.cpp:1551-1572: cv::imwrite("patch.png", patch) -- an 8-bit gray PNG here too
  if (marked_feature_label_ == -1) return false;
  for (Feature *f : feature_list_) {
    if (f->label_ != marked_feature_label_) continue;
    std::vector<uint8_t> png;
    sl2png::encode_gray(f->patch_.data, f->patch_.cols, f->patch_.rows, f->patch_.step, png);
    std::ofstream o("patch.png", std::ios::binary);
    if (!o) return false;
    o.write((const char *)png.data(), (std::streamsize)png.size());
    return (bool)o;
  }
  return false;
}

void MonoSLAM::print_robot_state() {  // monoslam.cpp:1543-1549
  std::cout << "Robot state:" << std::endl;
  for (int i = 0; i < 13; ++i) std::cout << xv_(i) << (i == 12 ? "\n" : " ");
}

// ---- frame ingestion (framegrabber/framegrabber.cpp:40-105, filegrabber.cpp:40-110) -----------------
FileGrabber::FileGrabber() {}

FileGrabber::~FileGrabber() {
  initialised_ = false;  // the reference never stops its thread; here the loop ends and is joined
  if (fg_thread_.joinable()) fg_thread_.join();
  files_vec_.clear();
}

void FileGrabber::Init(const std::string &path, FrameGrabber *frame_grabber) {
  ProcessFiles(path);
  std::sort(files_vec_.begin(), files_vec_.end());
  frame_grabber_ = frame_grabber;
  initialised_ = true;
  fg_thread_ = std::thread(std::ref(*this));
}

void FileGrabber::ProcessFiles(const std::string &directory) {  // filegrabber.cpp:63-83, recursive
  namespace fs = std::filesystem;
  if (!fs::exists(directory)) throw std::runtime_error("provided directory doesn't exist!");
  for (const auto &entry : fs::directory_iterator(directory)) {
    if (entry.is_directory()) ProcessFiles(entry.path().string());
    else files_vec_.push_back(entry.path().string());
  }
}

void FileGrabber::operator()() {  // filegrabber.cpp:85-104
  while (initialised_) {
    if (!frame_grabber_->IsFrameBufferFull() && files_vec_.size() > (size_t)frame_id_) {
      Frame frame;
      frame.frame_id = frame_id_;
      frame.data = GetImageFile(files_vec_.at(frame_id_));
      ++frame_id_;
      frame_grabber_->SetFrame(frame);
    } else {
      std::this_thread::sleep_for(std::chrono::milliseconds(1));
    }
  }
}

cv::Mat FileGrabber::GetImageFile(const std::string &file_full_path) { return decode_image(file_full_path); }

FrameGrabber::FrameGrabber() {}

FrameGrabber::~FrameGrabber() {
  delete file_grabber_;
  while (!frame_buffer_.empty()) frame_buffer_.pop();
}

void FrameGrabber::Init(const std::string &dev, const bool mode) {  // framegrabber.cpp:59-69
  if (mode) throw std::runtime_error("FrameGrabber: the USB camera grabber is not built (file mode only)");
  file_grabber_ = new FileGrabber;
  file_grabber_->Init(dev, this);
}

bool FrameGrabber::GetFrame(int /*frame_id*/, Frame *frame) {  // framegrabber.cpp:71-84
  std::lock_guard<std::mutex> lock(fg_mutex_);
  if (frame_buffer_.size() < 1) return false;
  *frame = frame_buffer_.front();
  frame_buffer_.pop();
  ++handed_out_;
  return true;
}

void FrameGrabber::SetFrame(const Frame &frame) {
  std::lock_guard<std::mutex> lock(fg_mutex_);
  frame_buffer_.push(frame);
}

bool FrameGrabber::IsFrameBufferFull() {  // framegrabber.cpp:94-103
  std::lock_guard<std::mutex> lock(fg_mutex_);
  return !(frame_buffer_.size() < 50);
}

bool FrameGrabber::Exhausted() {
  std::lock_guard<std::mutex> lock(fg_mutex_);
  return file_grabber_ && (size_t)handed_out_ >= file_grabber_->NumberOfFiles();
}

}  // namespace SceneLib2


// test hook: the PNG writer behind MonoSLAM::SavePatch on a caller's 8-bit gray image; 0 on success
extern "C" int sl2_host_write_png(const char *path, const unsigned char *gray, int w, int h) {
  if (!path || !gray || w <= 0 || h <= 0) return -1;
  std::vector<uint8_t> png;
  sl2png::encode_gray(gray, w, h, (size_t)w, png);
  std::ofstream o(path, std::ios::binary);
  if (!o) return -1;
  o.write((const char *)png.data(), (std::streamsize)png.size());
  return o ? 0 : -1;
}

// test hook (tests/test_host_shim.py): decode one image file the way FileGrabber does; returns 0 and fills w / h /
// out (cap bytes) on success, -1 when the file is not an image the shim reads, -2 when out is too small
extern "C" int sl2_host_decode_image(const char *path, unsigned char *out, int cap, int *w, int *h) {
  const cv::Mat m = SceneLib2::decode_image(path);
  if (m.empty()) return -1;
  *w = m.cols;
  *h = m.rows;
  if (cap < m.cols * m.rows) return -2;
  for (int r = 0; r < m.rows; ++r) std::memcpy(out + (size_t)r * m.cols, m.data + (size_t)r * m.step, m.cols);
  return 0;
}
