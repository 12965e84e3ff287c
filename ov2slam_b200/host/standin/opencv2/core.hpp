// Minimal STAND-IN for the OpenCV core types the hot-path class declarations use.
// Only for compile-checking ov2slam_b200/host/*.cpp in a container without OpenCV C++ headers
// (SURVEY.md section 7, step 2).  On a box with real OpenCV, drop `-I host/standin` and the
// real <opencv2/core.hpp> is used instead: the shim code only touches this subset.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <memory>
#include <vector>

#define OV2_STANDIN_OPENCV 1
#define CV_8U 0
#define CV_8UC1 0
#define CV_16UC1 2
#define CV_32FC1 5
#define CV_16SC2 11

namespace cv {

template <typename T> struct Point_ {
    T x, y;
    Point_() : x(0), y(0) {}
    Point_(T x_, T y_) : x(x_), y(y_) {}
    bool operator==(const Point_& o) const { return x == o.x && y == o.y; }
};
typedef Point_<float> Point2f;
typedef Point_<int> Point;

struct Size { int width, height; Size(int w = 0, int h = 0) : width(w), height(h) {} };
struct Rect { int x, y, width, height; Rect(int x_ = 0, int y_ = 0, int w = 0, int h = 0) : x(x_), y(y_), width(w), height(h) {} };

struct TermCriteria {
    enum { COUNT = 1, MAX_ITER = 1, EPS = 2 };
    int type, maxCount;
    double epsilon;
    TermCriteria(int t = 0, int c = 0, double e = 0) : type(t), maxCount(c), epsilon(e) {}
};

template <typename T> using Ptr = std::shared_ptr<T>;

// matrix with shared, ref-counted storage (what the shims need of cv::Mat): 8-bit images, and the CV_16SC2 / CV_16UC1 /
// CV_32FC1 rectification maps
class Mat {
public:
    int rows = 0, cols = 0;
    size_t step = 0;
    unsigned char* data = nullptr;
    Mat() {}
    Mat(int r, int c, int type) { create(r, c, type); }
    Mat(int r, int c, int type, void* ext, size_t st = 0) : rows(r), cols(c), step(st ? st : (size_t)c * esz(type)), data((unsigned char*)ext), type_(type) {}
    void create(int r, int c, int type) {
        if (data && r == rows && c == cols && type == type_) return;
        rows = r; cols = c; type_ = type; step = (size_t)c * esz(type);
        buf_.reset(new unsigned char[(size_t)r * step], std::default_delete<unsigned char[]>());
        data = buf_.get();
    }
    bool empty() const { return data == nullptr || rows == 0 || cols == 0; }
    int type() const { return type_; }
    Size size() const { return Size(cols, rows); }
    unsigned char* ptr(int r = 0) { return data + (size_t)r * step; }
    const unsigned char* ptr(int r = 0) const { return data + (size_t)r * step; }
    Mat row(int r) const { Mat m; m.rows = 1; m.cols = cols; m.step = step; m.data = data + (size_t)r * step; m.buf_ = buf_; m.type_ = type_; return m; }
private:
    static size_t esz(int type) { return type == CV_16UC1 ? 2 : (type == CV_32FC1 || type == CV_16SC2) ? 4 : 1; }
    std::shared_ptr<unsigned char> buf_;
    int type_ = CV_8UC1;
};

class CLAHE { public: virtual ~CLAHE() {} virtual void apply(const Mat&, Mat&) = 0; };

}  // namespace cv
