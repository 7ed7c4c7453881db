// Boost stand-in: the few pieces of Boost.uBLAS and Boost.Geometry the reference's KITTI evaluator
// (kitti_native_evaluation/src/evaluate_object_3d_offline.cpp) uses, so that it compiles without Boost.
// Test infrastructure only (oracle/kitti_eval_build.py); written for this project, not taken from Boost.
//
// Only convex rings are supported, which is all the evaluator builds (box footprints):
//   * intersection: Sutherland-Hodgman clipping of one ring by the other;
//   * union_: a polygon that carries area(a) + area(b) - area(a & b); the evaluator only asks for its area.
// Rectangle intersections therefore agree with Boost.Geometry up to rounding, not bit for bit.
#pragma once
#include <cmath>
#include <cstddef>
#include <vector>

#define BOOST_GEOMETRY_REGISTER_C_ARRAY_CS(cs)

namespace boost {
namespace numeric {
namespace ublas {

template <typename T>
class matrix {
 public:
  matrix(std::size_t rows, std::size_t cols) : rows_(rows), cols_(cols), data_(rows * cols, T()) {}
  T& operator()(std::size_t i, std::size_t j) { return data_[i * cols_ + j]; }
  const T& operator()(std::size_t i, std::size_t j) const { return data_[i * cols_ + j]; }
  std::vector<T>& data() { return data_; }   // row-major storage, as uBLAS's default layout
  std::size_t size1() const { return rows_; }
  std::size_t size2() const { return cols_; }

 private:
  std::size_t rows_, cols_;
  std::vector<T> data_;
};

template <typename T>
matrix<T> prod(const matrix<T>& a, const matrix<T>& b) {
  matrix<T> r(a.size1(), b.size2());
  for (std::size_t i = 0; i < a.size1(); ++i)
    for (std::size_t j = 0; j < b.size2(); ++j) {
      T s = T();
      for (std::size_t k = 0; k < a.size2(); ++k) s += a(i, k) * b(k, j);
      r(i, j) = s;
    }
  return r;
}

}  // namespace ublas
}  // namespace numeric

namespace geometry {
namespace cs {
struct cartesian {};
}  // namespace cs

namespace model {
namespace d2 {
template <typename T>
struct point_xy {
  T x, y;
};
}  // namespace d2

template <typename Point>
struct polygon {
  std::vector<Point> ring;              // open ring (the closing point is dropped)
  double area_override = std::nan("");  // set by union_
};
}  // namespace model

namespace detail {
template <typename Point>
double signed_area(const std::vector<Point>& r) {
  double a = 0.0;
  for (std::size_t i = 0; i < r.size(); ++i) {
    const Point& p = r[i];
    const Point& q = r[(i + 1) % r.size()];
    a += p.x * q.y - p.y * q.x;
  }
  return 0.5 * a;
}
}  // namespace detail

// area of a clockwise ring is positive (Boost.Geometry's default polygon orientation)
template <typename Point>
double area(const model::polygon<Point>& p) {
  if (!std::isnan(p.area_override)) return p.area_override;
  return p.ring.size() < 3 ? 0.0 : -detail::signed_area(p.ring);
}

template <typename Point, std::size_t N>
void append(model::polygon<Point>& p, const double (&pts)[N][2]) {
  for (std::size_t i = 0; i < N; ++i) p.ring.push_back(Point{pts[i][0], pts[i][1]});
  if (p.ring.size() > 1 && p.ring.front().x == p.ring.back().x && p.ring.front().y == p.ring.back().y)
    p.ring.pop_back();
}

template <typename Point>
void intersection(const model::polygon<Point>& a, const model::polygon<Point>& b, std::vector<model::polygon<Point>>& out) {
  std::vector<Point> poly = a.ring, next;
  // walk the clip ring counter-clockwise: inside = left of each edge
  std::vector<Point> clip = b.ring;
  if (detail::signed_area(clip) < 0.0) clip.assign(b.ring.rbegin(), b.ring.rend());
  for (std::size_t e = 0; e < clip.size() && !poly.empty(); ++e) {
    const Point& c0 = clip[e];
    const Point& c1 = clip[(e + 1) % clip.size()];
    const double ex = c1.x - c0.x, ey = c1.y - c0.y;
    next.clear();
    for (std::size_t j = 0; j < poly.size(); ++j) {
      const Point& p = poly[j];
      const Point& q = poly[(j + 1) % poly.size()];
      const double sp = ex * (p.y - c0.y) - ey * (p.x - c0.x);
      const double sq = ex * (q.y - c0.y) - ey * (q.x - c0.x);
      if (sp >= 0.0) next.push_back(p);
      if ((sp >= 0.0) != (sq >= 0.0)) {
        const double t = sp / (sp - sq);
        next.push_back(Point{p.x + t * (q.x - p.x), p.y + t * (q.y - p.y)});
      }
    }
    poly.swap(next);
  }
  if (poly.size() < 3) return;
  model::polygon<Point> r;
  r.ring = poly;
  if (detail::signed_area(r.ring) > 0.0) r.ring.assign(poly.rbegin(), poly.rend());   // clockwise, as Boost returns
  if (area(r) > 0.0) out.push_back(r);
}

template <typename Point>
void union_(const model::polygon<Point>& a, const model::polygon<Point>& b, std::vector<model::polygon<Point>>& out) {
  std::vector<model::polygon<Point>> in;
  intersection(a, b, in);
  model::polygon<Point> u;
  u.area_override = area(a) + area(b) - (in.empty() ? 0.0 : area(in.front()));
  out.push_back(u);
}

}  // namespace geometry
}  // namespace boost
