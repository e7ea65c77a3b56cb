// ORACLE — TEST INFRASTRUCTURE ONLY.
// Storage-only stand-in for the part of cv::Mat that the reference's improc/*.cpp touches
// (improc.cpp:66-67,81-82; search_multiple_overlapping_ellipses.cpp:114,160-177): a pixel
// pointer, a size, a (size,type,fill) constructor and at<T>(row,col).  It contains NO
// arithmetic: every FP/integer operation executed by oracle/_ref/libsl2ref.so is the
// reference's own source, compiled unmodified from the original SceneLib2 checkout.
#pragma once
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <vector>

#define CV_8UC1 0
#define CV_64FC1 6

namespace cv {
struct Size {
  int width, height;
  Size() : width(0), height(0) {}
  Size(int w, int h) : width(w), height(h) {}
};
class Mat {
 public:
  unsigned char *data;
  int rows, cols;
  Mat() : data(nullptr), rows(0), cols(0), esz_(1) {}
  // wrap external u8 pixels (not owned)
  Mat(int r, int c, int type, void *ext) : data((unsigned char *)ext), rows(r), cols(c), esz_(type == CV_64FC1 ? 8 : 1) {}
  // owned, filled with a constant
  Mat(Size s, int type, double fill) : rows(s.height), cols(s.width), esz_(type == CV_64FC1 ? 8 : 1) {
    own_.reset(new std::vector<unsigned char>((size_t)rows * cols * esz_));
    data = own_->data();
    if (type == CV_64FC1) {
      double *d = (double *)data;
      for (size_t i = 0; i < (size_t)rows * cols; ++i) d[i] = fill;
    } else {
      std::memset(data, (int)fill, (size_t)rows * cols);
    }
  }
  Size size() const { return Size(cols, rows); }
  template <typename T>
  T &at(int r, int c) { return ((T *)data)[(size_t)r * cols + c]; }
  template <typename T>
  const T &at(int r, int c) const { return ((const T *)data)[(size_t)r * cols + c]; }

 private:
  int esz_;
  std::shared_ptr<std::vector<unsigned char>> own_;
};
}  // namespace cv
