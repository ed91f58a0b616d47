// isam_facade.hpp -- header-only re-creation of the slice of iSAM's C++ API that pop_planar_slam uses,
// on top of the C-ABI of include/popup_gpu.h (libpopup_gpu.so, CUDA, sm_90a).
//
// pop_planar_slam/src/Mapping.cpp and main_3d.cpp build and solve their factor graph exclusively through
// the calls listed in SURVEY.md 8(b); with this header in place of <isam/isam.h> + "isam_plane3d.h" the
// same call sites compile against the GPU back end:
//     isam::Slam, Properties, Noise / Covariance / Information / SqrtInformation,
//     Pose3d, Pose3d_Node, Pose3d_Factor, Pose3d_Pose3d_Factor,
//     Plane3d, Plane3d_Node, Plane3d_Factor, Pose3d_Plane3d_Factor
// g2o-flavoured names from BASELINE.json's wording are provided as aliases (VertexSE3Expmap, VertexPlane,
// EdgeSE3Plane, EdgeSE3Expmap) -- the reference contains no g2o code (SURVEY.md section 0).
//
// Semantics reproduced (paths relative to the reference checkout; ISAM = pop_planar_slam/Thirdparty/isam):
//   * the caller news nodes / factors and passes raw pointers; Slam never frees them (ISAM/include/isam/Slam.h:123,130)
//   * values are returned by value (NodeT::value, Node.h:130); host mirrors are refreshed after every solve
//   * ids follow insertion order (Slam.cpp:47-48); factors initialise un-initialised nodes
//     (slam3d.h:75-80,123-137; isam_plane3d.h:252-264,443-448) -- done inside the C-ABI
//   * errors: the reference exits on require() failures (util.h:174-184); here a failed C-ABI call throws
//     std::runtime_error carrying pus_last_error() -- there is no CPU fallback.
// Small fixed-size linear algebra is provided by the minimal Mat / Vec types below when Eigen is not
// available (define ISAM_FACADE_USE_EIGEN before including this header to use Eigen types instead).
#pragma once
#include <cmath>
#include <cstring>
#include <list>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

#include "popup_noise.hpp"

#include "popup_gpu.h"

#ifdef ISAM_FACADE_USE_EIGEN
#include <Eigen/Dense>
#endif

namespace isam {

// ---------------------------------------------------------------------------------------------
// minimal dense types (row-major) -- just enough for the call sites of Mapping.cpp / main_3d.cpp
// ---------------------------------------------------------------------------------------------
#ifdef ISAM_FACADE_USE_EIGEN
typedef Eigen::MatrixXd MatrixXd;
typedef Eigen::Matrix4d Matrix4d;
typedef Eigen::Vector3d Vector3d;
typedef Eigen::Vector4d Vector4d;
typedef Eigen::Matrix<double, 6, 1> Vector6d;
typedef Eigen::VectorXd VectorXd;
inline VectorXd to_vectorxd(const std::vector<double>& v) { VectorXd x((int)v.size()); for (size_t i = 0; i < v.size(); i++) x((int)i) = v[i]; return x; }
inline double mget(const MatrixXd& m, int r, int c) { return m(r, c); }
inline int mrows(const MatrixXd& m) { return (int)m.rows(); }
#else
typedef std::vector<double> VectorXd;   // Slam::weighted_errors / Factor::error in the Eigen-free flavour
inline VectorXd to_vectorxd(const std::vector<double>& v) { return v; }
struct MatrixXd {
  int r = 0, c = 0;
  std::vector<double> a;
  MatrixXd() {}
  MatrixXd(int rows, int cols) : r(rows), c(cols), a((size_t)rows * cols, 0.0) {}
  double& operator()(int i, int j) { return a[(size_t)i * c + j]; }
  double operator()(int i, int j) const { return a[(size_t)i * c + j]; }
  int rows() const { return r; }
  int cols() const { return c; }
  static MatrixXd Identity(int n) { MatrixXd m(n, n); for (int i = 0; i < n; i++) m(i, i) = 1; return m; }
  static MatrixXd Diagonal(const std::vector<double>& d) { MatrixXd m((int)d.size(), (int)d.size()); for (size_t i = 0; i < d.size(); i++) m((int)i, (int)i) = d[i]; return m; }
};
struct Matrix4d {
  double a[16];
  Matrix4d() { for (int i = 0; i < 16; i++) a[i] = (i % 5 == 0) ? 1.0 : 0.0; }
  double& operator()(int i, int j) { return a[i * 4 + j]; }
  double operator()(int i, int j) const { return a[i * 4 + j]; }
  Matrix4d operator*(const Matrix4d& o) const {
    Matrix4d m;
    for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) { double s = 0; for (int k = 0; k < 4; k++) s += a[i * 4 + k] * o.a[k * 4 + j]; m.a[i * 4 + j] = s; }
    return m;
  }
  Matrix4d transpose() const { Matrix4d m; for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) m.a[i * 4 + j] = a[j * 4 + i]; return m; }
};
struct Vector3d {
  double v[3];
  Vector3d() : v{0, 0, 0} {}
  Vector3d(double x, double y, double z) : v{x, y, z} {}
  double& operator()(int i) { return v[i]; }
  double operator()(int i) const { return v[i]; }
  double dot(const Vector3d& o) const { return v[0] * o.v[0] + v[1] * o.v[1] + v[2] * o.v[2]; }
  double norm() const { return std::sqrt(dot(*this)); }
  Vector3d operator*(double s) const { return Vector3d(v[0] * s, v[1] * s, v[2] * s); }
  Vector3d operator-(const Vector3d& o) const { return Vector3d(v[0] - o.v[0], v[1] - o.v[1], v[2] - o.v[2]); }
  Vector3d normalized() const { double n = norm(); return Vector3d(v[0] / n, v[1] / n, v[2] / n); }
};
struct Vector4d {
  double v[4];
  Vector4d() : v{0, 0, 0, 0} {}
  Vector4d(double a, double b, double c, double d) : v{a, b, c, d} {}
  double& operator()(int i) { return v[i]; }
  double operator()(int i) const { return v[i]; }
};
struct Vector6d {
  double v[6];
  Vector6d() : v{0, 0, 0, 0, 0, 0} {}
  double& operator()(int i) { return v[i]; }
  double operator()(int i) const { return v[i]; }
};
inline double mget(const MatrixXd& m, int r, int c) { return m(r, c); }
inline int mrows(const MatrixXd& m) { return m.rows(); }
#endif

namespace detail {
inline void check(int rc) { if (rc < 0) throw std::runtime_error(std::string("libpopup_gpu: ") + pus_last_error()); }
using pus_noise::chol_upper;    // include/popup_noise.hpp: shared with the plane map
using pus_noise::inverse_spd;
}  // namespace detail

// ---------------------------------------------------------------------------------------------
// Noise models  (ISAM/include/isam/Noise.h:36-62): all reduce to an upper-triangular sqrt-information
// ---------------------------------------------------------------------------------------------
class Noise {
 public:
  int n = 0;
  std::vector<double> _sqrtinf;  // n x n row-major, upper triangular
  std::vector<double> packed() const { return pus_noise::pack_upper(_sqrtinf, n); }
 protected:
  static std::vector<double> flat(const MatrixXd& m) { int k = mrows(m); std::vector<double> a((size_t)k * k); for (int i = 0; i < k; i++) for (int j = 0; j < k; j++) a[(size_t)i * k + j] = mget(m, i, j); return a; }
};
class SqrtInformation : public Noise { public: SqrtInformation(const MatrixXd& s) { n = mrows(s); _sqrtinf = flat(s); } };
class Information : public Noise { public: Information(const MatrixXd& inf) { n = mrows(inf); _sqrtinf = detail::chol_upper(flat(inf), n); } };
class Covariance : public Noise { public: Covariance(const MatrixXd& cov) { n = mrows(cov); _sqrtinf = detail::chol_upper(detail::inverse_spd(flat(cov), n), n); } };

// ---------------------------------------------------------------------------------------------
// Properties  (ISAM/include/isam/Properties.h:37-110)
// ---------------------------------------------------------------------------------------------
enum Method { GAUSS_NEWTON = 0, LEVENBERG_MARQUARDT = 1 };
struct Properties {
  bool verbose = false, quiet = false, force_numerical_jacobian = false;
  Method method = GAUSS_NEWTON;
  double epsilon1 = 1e-2, epsilon2 = 1e-2, epsilon3 = 1e-2, epsilon_abs = 1e-3, epsilon_rel = 1e-5;
  int max_iterations = 500;
  double lm_lambda0 = 1e-6, lm_lambda_factor = 10.;
  int mod_update = 1, mod_batch = 100, mod_solve = 1;
};
struct UpdateStats { int step = 0; bool batch = false, solve = false; };

// ---------------------------------------------------------------------------------------------
// Pose3d  (ISAM/include/isam/Pose3d.h:70-274 + Rot3d.h): translation + unit quaternion
// ---------------------------------------------------------------------------------------------
class Pose3d {
  double _t[3];
  double _q[4];  // w x y z
 public:
  static const int dim = 6;
  Pose3d() : _t{0, 0, 0}, _q{1, 0, 0, 0} {}
  Pose3d(double x, double y, double z, double yaw, double pitch, double roll) : _t{x, y, z} {   // Rot3d::euler_to_quat Rot3d.h:100-112
    double sy = std::sin(yaw * 0.5), cy = std::cos(yaw * 0.5), sp = std::sin(pitch * 0.5), cp = std::cos(pitch * 0.5);
    double sr = std::sin(roll * 0.5), cr = std::cos(roll * 0.5);
    _q[0] = cr * cp * cy + sr * sp * sy; _q[1] = sr * cp * cy - cr * sp * sy; _q[2] = cr * sp * cy + sr * cp * sy; _q[3] = cr * cp * sy - sr * sp * cy;
  }
  explicit Pose3d(const Matrix4d& m) {  // Pose3d(Matrix4d) Pose3d.h:92-98 (trace / largest-diagonal quaternion, renormalised)
    double T[16]; for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) T[i * 4 + j] = m(i, j) / m(3, 3);
    _t[0] = T[3]; _t[1] = T[7]; _t[2] = T[11];
    double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
    double t = R[0] + R[4] + R[8];
    if (t > 0) { t = std::sqrt(t + 1.0); _q[0] = 0.5 * t; t = 0.5 / t; _q[1] = (R[7] - R[5]) * t; _q[2] = (R[2] - R[6]) * t; _q[3] = (R[3] - R[1]) * t; }
    else {
      int i = 0; if (R[4] > R[0]) i = 1; if (R[8] > R[i * 3 + i]) i = 2; int j = (i + 1) % 3, k = (j + 1) % 3;
      t = std::sqrt(R[i * 3 + i] - R[j * 3 + j] - R[k * 3 + k] + 1.0); double v[3]; v[i] = 0.5 * t; t = 0.5 / t;
      _q[0] = (R[k * 3 + j] - R[j * 3 + k]) * t; v[j] = (R[j * 3 + i] + R[i * 3 + j]) * t; v[k] = (R[k * 3 + i] + R[i * 3 + k]) * t;
      _q[1] = v[0]; _q[2] = v[1]; _q[3] = v[2];
    }
    double nq = std::sqrt(_q[0] * _q[0] + _q[1] * _q[1] + _q[2] * _q[2] + _q[3] * _q[3]);
    for (int i = 0; i < 4; i++) _q[i] /= nq;
  }
  static Pose3d from7(const double* v) { Pose3d p; std::memcpy(p._t, v, 3 * sizeof(double)); std::memcpy(p._q, v + 3, 4 * sizeof(double)); return p; }
  void to7(double* v) const { std::memcpy(v, _t, 3 * sizeof(double)); std::memcpy(v + 3, _q, 4 * sizeof(double)); }
  double x() const { return _t[0]; }
  double y() const { return _t[1]; }
  double z() const { return _t[2]; }
  void ypr(double& yaw, double& pitch, double& roll) const {  // Rot3d::quat_to_euler Rot3d.h:114-124
    const double q0 = _q[0], q1 = _q[1], q2 = _q[2], q3 = _q[3];
    roll = std::atan2(2.0 * (q0 * q1 + q2 * q3), q0 * q0 - q1 * q1 - q2 * q2 + q3 * q3);
    pitch = std::asin(2.0 * (q0 * q2 - q3 * q1));
    yaw = std::atan2(2.0 * (q0 * q3 + q1 * q2), q0 * q0 + q1 * q1 - q2 * q2 - q3 * q3);
  }
  double yaw() const { double a, b, c; ypr(a, b, c); return a; }
  double pitch() const { double a, b, c; ypr(a, b, c); return b; }
  double roll() const { double a, b, c; ypr(a, b, c); return c; }
  Vector6d vector() const { Vector6d v; v(0) = _t[0]; v(1) = _t[1]; v(2) = _t[2]; double a, b, c; ypr(a, b, c); v(3) = a; v(4) = b; v(5) = c; return v; }
  Matrix4d wTo() const {  // Pose3d.h:188-194
    Matrix4d T; const double* q = _q;
    const double tx = 2 * q[1], ty = 2 * q[2], tz = 2 * q[3], twx = tx * q[0], twy = ty * q[0], twz = tz * q[0];
    const double txx = tx * q[1], txy = ty * q[1], txz = tz * q[1], tyy = ty * q[2], tyz = tz * q[2], tzz = tz * q[3];
    T(0, 0) = 1 - (tyy + tzz); T(0, 1) = txy - twz; T(0, 2) = txz + twy; T(0, 3) = _t[0];
    T(1, 0) = txy + twz; T(1, 1) = 1 - (txx + tzz); T(1, 2) = tyz - twx; T(1, 3) = _t[1];
    T(2, 0) = txz - twy; T(2, 1) = tyz + twx; T(2, 2) = 1 - (txx + tyy); T(2, 3) = _t[2];
    T(3, 0) = 0; T(3, 1) = 0; T(3, 2) = 0; T(3, 3) = 1;
    return T;
  }
  Matrix4d oTw() const {  // Pose3d.h:204-213
    Matrix4d W = wTo(), T;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) T(i, j) = W(j, i);
    for (int i = 0; i < 3; i++) T(i, 3) = -(T(i, 0) * _t[0] + T(i, 1) * _t[1] + T(i, 2) * _t[2]);
    T(3, 0) = 0; T(3, 1) = 0; T(3, 2) = 0; T(3, 3) = 1;
    return T;
  }
  Pose3d oplus(const Pose3d& d) const { return Pose3d(wTo() * d.wTo()); }    // Pose3d.h:222-224
  Pose3d ominus(const Pose3d& b) const { return Pose3d(b.oTw() * wTo()); }   // Pose3d.h:233-235
};

// ---------------------------------------------------------------------------------------------
// Plane3d  (pop_planar_slam/src/isam_plane3d.h:27-193)
// ---------------------------------------------------------------------------------------------
class Plane3d {
  double _abcd[4];
  void _normalize() { double n = std::sqrt(_abcd[0] * _abcd[0] + _abcd[1] * _abcd[1] + _abcd[2] * _abcd[2] + _abcd[3] * _abcd[3]); if (n > 0) for (int i = 0; i < 4; i++) _abcd[i] /= n; }
 public:
  int plane_type = -1;
  static const int dim = 3;
  Plane3d() : _abcd{1, 0, 0, 0} {}
  Plane3d(const Vector4d& v) { for (int i = 0; i < 4; i++) _abcd[i] = v(i); _normalize(); }              // :59-66
  Plane3d(const Vector3d& normal, double dist) {                                                           // :52-58
    Vector3d nn = normal.normalized(); _abcd[0] = nn(0); _abcd[1] = nn(1); _abcd[2] = nn(2); _abcd[3] = -dist; _normalize();
  }
  static Plane3d from4(const double* v) { return Plane3d(Vector4d(v[0], v[1], v[2], v[3])); }
  Vector4d vector() const { return Vector4d(_abcd[0], _abcd[1], _abcd[2], _abcd[3]); }
  Vector3d normal() const { return Vector3d(_abcd[0], _abcd[1], _abcd[2]).normalized(); }                  // :149-151
  double d() const { return -_abcd[3] / Vector3d(_abcd[0], _abcd[1], _abcd[2]).norm(); }                   // :154-156
  double distance() const { return std::fabs(d()); }
  Vector3d point0() const { return normal() * d(); }
  double distance(const Vector3d& p) const { return std::fabs(normal().dot(p - point0())); }
  Vector3d project_to_plane(const Vector3d& p) const { Vector3d n = normal(); return p - n * (n.dot(p) - d()); }  // :172-177
  Plane3d transform_to(const Matrix4d& wTo) const { return mul_T(wTo); }                                  // :180-182
  Plane3d transform_from(const Matrix4d& oTw) const { return mul_T(oTw); }                                // :186-188
 private:
  Plane3d mul_T(const Matrix4d& T) const {
    double r[4];
    for (int i = 0; i < 4; i++) { double s = 0; for (int j = 0; j < 4; j++) s += T(j, i) * _abcd[j]; r[i] = s; }
    return Plane3d(Vector4d(r[0], r[1], r[2], r[3]));
  }
};

// ---------------------------------------------------------------------------------------------
// graph elements
// ---------------------------------------------------------------------------------------------
class Slam;
class Factor;
class Node {
 protected:
  friend class Slam;
  friend class Factor;
  pus_handle _h = nullptr;  // set by Slam::add_node
  int _id = -1;
  std::list<Factor*> _factors;
 public:
  virtual ~Node() {}
  int unique_id() const { return _id; }
  const std::list<Factor*>& factors() { return _factors; }   // Node.h:88
  virtual int dim() const = 0;
  virtual bool initialized() const = 0;
};

template <class T> class NodeT;

template <> class NodeT<Pose3d> : public Node {
  bool _init = false;
  Pose3d _pending;
 public:
  int dim() const { return 6; }
  bool initialized() const { return _init; }
  void init(const Pose3d& p) {   // NodeT::init Node.h:123-126
    _init = true; _pending = p;
    if (_h) { double v[7]; p.to7(v); detail::check(pus_init_pose(_h, _id, v)); }
  }
  Pose3d value() const {         // NodeT::value Node.h:130 (by value)
    if (!_h) return _pending;
    double v[7]; detail::check(pus_get_pose(_h, _id, v)); return Pose3d::from7(v);
  }
  void _attach(pus_handle h) { _h = h; double v[7]; if (_init) _pending.to7(v); _id = pus_add_pose(h, _init ? v : nullptr); detail::check(_id); }
  void _mark_initialized() { _init = true; }
};
template <> class NodeT<Plane3d> : public Node {
  bool _init = false;
  Plane3d _pending;
 public:
  int dim() const { return 3; }
  bool initialized() const { return _init; }
  void init(const Plane3d& p) {
    _init = true; _pending = p;
    if (_h) { Vector4d v = p.vector(); double a[4] = {v(0), v(1), v(2), v(3)}; detail::check(pus_init_plane(_h, _id, a)); }
  }
  Plane3d value() const {
    if (!_h) return _pending;
    double v[4]; detail::check(pus_get_plane(_h, _id, v)); return Plane3d::from4(v);
  }
  void _attach(pus_handle h) { _h = h; Vector4d v = _pending.vector(); double a[4] = {v(0), v(1), v(2), v(3)}; _id = pus_add_plane(h, _init ? a : nullptr); detail::check(_id); }
  void _mark_initialized() { _init = true; }
};
typedef NodeT<Pose3d> Pose3d_Node;                       // ISAM/include/isam/slam3d.h:39
class Plane3d_Node : public NodeT<Plane3d> {             // isam_plane3d.h:197-210
  Pose3d_Node* _base = nullptr;
 public:
  void set_base(Pose3d_Node* b) { _base = b; }
  Pose3d_Node* base() { return _base; }
};

class Factor {
 protected:
  friend class Slam;
  pus_handle _h = nullptr;
  int _id = -1;
  std::vector<Node*> _nodes;
  Noise _noise;
 public:
  Factor(const Noise& n) : _noise(n) {}
  virtual ~Factor() {}
  int unique_id() const { return _id; }
  std::vector<Node*>& nodes() { return _nodes; }          // Factor.h:79
  const Noise& noise() const { return _noise; }           // Factor.h:204
  virtual int _attach(pus_handle h) = 0;                  // issues the pus_add_* call
  VectorXd error() const {                                // Factor.h:67-77 at the estimate, evaluated on the device
    std::vector<double> e(6);
    const int n = pus_factor_errors(_h, 1, &_id, e.data());
    if (n < 0) throw std::runtime_error(std::string("Factor::error: ") + pus_last_error());
    e.resize(n);
    return to_vectorxd(e);
  }
};

template <class T> class FactorT : public Factor {
 protected:
  T _measure;
 public:
  FactorT(const Noise& n, const T& m) : Factor(n), _measure(m) {}
  const T& measurement() const { return _measure; }       // Factor.h:203
};

class Pose3d_Factor : public FactorT<Pose3d> {            // slam3d.h:58-89
 public:
  Pose3d_Factor(Pose3d_Node* pose, const Pose3d& prior, const Noise& noise) : FactorT<Pose3d>(noise, prior) { _nodes.push_back(pose); }
  int _attach(pus_handle h) {
    Vector6d m = _measure.vector(); double mv[6]; for (int i = 0; i < 6; i++) mv[i] = m(i);
    std::vector<double> si = _noise.packed();
    int f = pus_add_pose_prior(h, _nodes[0]->unique_id(), mv, si.data()); detail::check(f);
    static_cast<Pose3d_Node*>(_nodes[0])->_mark_initialized();
    return f;
  }
};
class Pose3d_Pose3d_Factor : public FactorT<Pose3d> {     // slam3d.h:91-193 (anchor variant unused by PPS)
 public:
  Pose3d_Pose3d_Factor(Pose3d_Node* p1, Pose3d_Node* p2, const Pose3d& measure, const Noise& noise) : FactorT<Pose3d>(noise, measure) { _nodes.push_back(p1); _nodes.push_back(p2); }
  int _attach(pus_handle h) {
    Vector6d m = _measure.vector(); double mv[6]; for (int i = 0; i < 6; i++) mv[i] = m(i);
    std::vector<double> si = _noise.packed();
    int f = pus_add_odometry(h, _nodes[0]->unique_id(), _nodes[1]->unique_id(), mv, si.data()); detail::check(f);
    static_cast<Pose3d_Node*>(_nodes[0])->_mark_initialized(); static_cast<Pose3d_Node*>(_nodes[1])->_mark_initialized();
    return f;
  }
};
class Plane3d_Factor : public FactorT<Plane3d> {          // isam_plane3d.h:428-474
 public:
  Plane3d_Factor(Plane3d_Node* plane, const Plane3d& prior, const Noise& noise) : FactorT<Plane3d>(noise, prior) { _nodes.push_back(plane); }
  int _attach(pus_handle h) {
    Vector4d v = _measure.vector(); double a[4] = {v(0), v(1), v(2), v(3)};
    std::vector<double> si = _noise.packed();
    int f = pus_add_plane_prior(h, _nodes[0]->unique_id(), a, si.data()); detail::check(f);
    static_cast<Plane3d_Node*>(_nodes[0])->_mark_initialized();
    return f;
  }
};
class Pose3d_Plane3d_Factor : public FactorT<Plane3d> {   // isam_plane3d.h:221-308
 public:
  Pose3d_Plane3d_Factor(Pose3d_Node* pose, Plane3d_Node* plane, const Plane3d& measure, const Noise& noise, bool relative = false)
      : FactorT<Plane3d>(noise, measure) {
    if (relative) throw std::runtime_error("Pose3d_Plane3d_Factor: relative parameterisation is not supported (pop_planar_slam builds with useRelative = false, Mapping.cpp:21)");
    _nodes.push_back(pose); _nodes.push_back(plane);
  }
  void _mirror_measurement(const Plane3d& m) { _measure = m; }   // value already stored on the device (Slam::refresh_plane_measurements)
  void set_measurement(const Plane3d& m) {                // Factor.h:206 (Mapping.cpp:603)
    _measure = m;
    if (_h) { Vector4d v = m.vector(); double a[4] = {v(0), v(1), v(2), v(3)}; detail::check(pus_set_measurement(_h, _id, a)); }
  }
  int _attach(pus_handle h) {
    Vector4d v = _measure.vector(); double a[4] = {v(0), v(1), v(2), v(3)};
    std::vector<double> si = _noise.packed();
    int f = pus_add_pose_plane(h, _nodes[0]->unique_id(), _nodes[1]->unique_id(), a, si.data()); detail::check(f);
    static_cast<Plane3d_Node*>(_nodes[1])->_mark_initialized();
    return f;
  }
};

// Pose3d_Plane3d_Factor2 (isam_plane3d.h:314-424): the measurement is re-popped from the ground edge inside the residual
class Pose3d_Plane3d_Factor2 : public Pose3d_Plane3d_Factor {
  double _rays[6] = {0, 0, 0, 0, 0, 0};
  bool _have_rays = false;
 public:
  Pose3d_Plane3d_Factor2(Pose3d_Node* pose, Plane3d_Node* plane, const Plane3d& measure, const Noise& noise, bool relative = false)
      : Pose3d_Plane3d_Factor(pose, plane, measure, noise, relative) {}
  // precompute_edge_ray (:358-370): invK (row-major 3x3, float) times the homogeneous end points of ONE ground segment
  // (x1 y1 x2 y2, pixels), computed in float and widened to double as upstream; call before Slam::add_factor
  void precompute_edge_ray(const float invK[9], const float seg[4]) {
    for (int k = 0; k < 2; k++)
      for (int i = 0; i < 3; i++) _rays[3 * k + i] = (double)(invK[i * 3] * seg[2 * k] + invK[i * 3 + 1] * seg[2 * k + 1] + invK[i * 3 + 2] * 1.0f);
    _have_rays = true;
  }
  int _attach(pus_handle h) {
    if (!_have_rays) throw std::runtime_error("Pose3d_Plane3d_Factor2: call precompute_edge_ray() before add_factor()");
    Vector4d v = _measure.vector(); double a[4] = {v(0), v(1), v(2), v(3)};
    std::vector<double> si = _noise.packed();
    int f = pus_add_pose_plane2(h, _nodes[0]->unique_id(), _nodes[1]->unique_id(), a, _rays, si.data()); detail::check(f);
    static_cast<Plane3d_Node*>(_nodes[1])->_mark_initialized();
    return f;
  }
};

// Slam::jacobian() of the façade: iSAM returns a SparseSystem (ISAM/include/isam/SparseSystem.h), which the façade does not
// provide; this struct carries the same matrix as CSR (rows in factor order, columns in node order, ascending columns within
// a row, zeros stored) and rhs = Jacobian::rhs() = minus the residual rows.
struct SparseJacobian {
  long long rows = 0, cols = 0;
  std::vector<int> row_ptr, col_idx;   // [rows + 1], [nnz]
  std::vector<double> values, rhs;     // [nnz], [rows]
};

// isam::Covariances (ISAM/include/isam/Covariances.h:58-110), read through Slam::covariances(): Sigma = (J^T J)^-1 at the
// current estimate, undamped, recovered on the device from the band solver's nested-dissection factor (the handle must use
// LINEAR_SOLVER_BAND with ORDERING_NESTED_DISSECTION; see pus_marginal_covariances).  marginal(list) is the joint block over
// the nodes in list order, each node's rows / columns in its tangent order; access(pairs) returns dim(first) x dim(second)
// blocks, as Covariances.cpp:107-150 does.
class Covariances {
  pus_handle _h;
 public:
  typedef std::list<std::list<Node*> > node_lists_t;
  typedef std::list<std::pair<Node*, Node*> > node_pair_list_t;
  explicit Covariances(pus_handle h) : _h(h) {}
  std::list<MatrixXd> access(const node_pair_list_t& pairs) const {                 // Covariances.cpp:107-150
    std::vector<int> ids;
    long long n = 0;
    for (const auto& p : pairs) { ids.push_back(p.first->unique_id()); ids.push_back(p.second->unique_id()); n += p.first->dim() * p.second->dim(); }
    std::vector<double> v((size_t)n + 1);
    detail::check(pus_covariance_blocks(_h, (int)pairs.size(), ids.data(), v.data()) < 0 ? -1 : 0);
    std::list<MatrixXd> out;
    size_t o = 0;
    for (const auto& p : pairs) {
      const int r = p.first->dim(), c = p.second->dim();
      MatrixXd m(r, c);
      for (int i = 0; i < r; i++)
        for (int j = 0; j < c; j++) m(i, j) = v[o + (size_t)i * c + j];
      o += (size_t)r * c;
      out.push_back(m);
    }
    return out;
  }
  std::list<MatrixXd> marginal(const node_lists_t& lists) const {                   // Covariances.cpp:70-99
    // as covariance.cpp:135-144: the upper triangle is computed and mirrored, so the joint matrix is exactly symmetric
    std::list<MatrixXd> out;
    for (const auto& l : lists) {
      const std::vector<Node*> v(l.begin(), l.end());
      std::vector<int> at(v.size() + 1, 0);
      node_pair_list_t pairs;
      for (size_t a = 0; a < v.size(); a++) {
        at[a + 1] = at[a] + v[a]->dim();
        for (size_t b = a; b < v.size(); b++) pairs.push_back(std::make_pair(v[a], v[b]));
      }
      const std::list<MatrixXd> blocks = access(pairs);
      MatrixXd m(at[v.size()], at[v.size()]);
      auto it = blocks.begin();
      for (size_t a = 0; a < v.size(); a++)
        for (size_t b = a; b < v.size(); b++, ++it)
          for (int i = 0; i < v[a]->dim(); i++)
            for (int j = (a == b ? i : 0); j < v[b]->dim(); j++) {
              const double x = mget(*it, i, j);
              m(at[a] + i, at[b] + j) = x;
              m(at[b] + j, at[a] + i) = x;
            }
      out.push_back(m);
    }
    return out;
  }
  MatrixXd marginal(const std::list<Node*>& nodes) const { return marginal(node_lists_t(1, nodes)).front(); }   // :101-105
  std::list<MatrixXd> marginals(const node_lists_t& lists) const { return marginal(lists); }
};

// robust costs (ISAM/include/isam/robust.h:101-118); Slam::set_cost_function takes these tags
struct cost_func_t { int kind; double b; };
inline cost_func_t cost_huber_tag(double b) { return cost_func_t{1, b}; }
inline cost_func_t cost_pseudo_huber_tag(double b) { return cost_func_t{2, b}; }

// ---------------------------------------------------------------------------------------------
// Slam  (ISAM/include/isam/Slam.h, ISAM/isamlib/Slam.cpp)
// ---------------------------------------------------------------------------------------------
class Slam {
  pus_handle _h = nullptr;
  Properties _prop;
  std::list<Node*> _nodes;
  std::list<Factor*> _factors;
  int _step = 0;
  Covariances _covariances{nullptr};
  Slam(const Slam&);
  Slam& operator=(const Slam&);
 public:
  explicit Slam(int device = 0) { detail::check(pus_create(device, &_h)); _covariances = Covariances(_h); }
  const Covariances& covariances() { return _covariances; }                       // Slam.h:210
  ~Slam() { if (_h) pus_destroy(_h); }
  pus_handle handle() { return _h; }
  Properties properties() { return _prop; }                                         // Slam.h:92-94
  void set_properties(const Properties& p) {                                        // Slam.h:99-101
    _prop = p;
    pus_properties q; q.method = p.method; q.epsilon2 = p.epsilon2; q.epsilon_abs = p.epsilon_abs; q.epsilon_rel = p.epsilon_rel;
    q.max_iterations = p.max_iterations; q.lm_lambda0 = p.lm_lambda0; q.lm_lambda_factor = p.lm_lambda_factor;
    q.mod_update = p.mod_update; q.mod_batch = p.mod_batch; q.mod_solve = p.mod_solve;
    detail::check(pus_set_properties(_h, &q));
    // Properties::force_numerical_jacobian (Properties.h:44-45): the reference's own numericalDiff scheme on the device instead
    // of the closed-form blocks -- the mode in which a solve follows the reference's trajectory step for step
    detail::check(pus_set_jacobian_mode(_h, p.force_numerical_jacobian ? 1 : 0));
  }
  void set_cost_function(cost_func_t f) { detail::check(pus_set_robust(_h, f.kind, f.b)); }   // Slam.cpp:212-214
  // Extension, no iSAM counterpart (kept out of Properties, which mirrors iSAM's struct): solve the reduced pose system
  // exactly by a dense Cholesky on the device instead of PCG -- with force_numerical_jacobian, a solve that does what the
  // reference does step for step.  DIRECT: dense, graphs of at most 640 poses; BAND: the same exact solve on the envelope
  // of a bordered system, graphs of any size within its device-memory budget; see pus_set_linear_solver.
  enum LinearSolver { LINEAR_SOLVER_PCG = 0, LINEAR_SOLVER_DIRECT = 1, LINEAR_SOLVER_BAND = 2 };
  void set_linear_solver(LinearSolver kind) { detail::check(pus_set_linear_solver(_h, (int)kind)); }
  // order of the band solve's pose tiles (LINEAR_SOLVER_BAND only): insertion order (the default) or nested dissection, which
  // keeps the fill low where a loop closure re-observes earlier planes; see pus_set_direct_ordering
  enum Ordering { ORDERING_INSERTION = 0, ORDERING_NESTED_DISSECTION = 1 };
  void set_direct_ordering(Ordering order) { detail::check(pus_set_direct_ordering(_h, (int)order)); }
  void add_node(Pose3d_Node* n) { n->_attach(_h); _nodes.push_back(n); }            // Slam.cpp:91-94
  void add_node(Plane3d_Node* n) { n->_attach(_h); _nodes.push_back(n); }
  void add_factor(Factor* f) {                                                      // Slam.cpp:96-105
    f->_h = _h;
    f->_id = f->_attach(_h);
    for (Node* n : f->_nodes) n->_factors.push_back(f);
    _factors.push_back(f);
  }
  void remove_factor(Factor* f) {                                                   // Slam.cpp:117-126
    detail::check(pus_remove_factor(_h, f->_id));
    for (Node* n : f->_nodes) n->_factors.remove(f);
    _factors.remove(f);
  }
  void remove_node(Node* n) {                                                       // Slam.cpp:107-115
    std::list<Factor*> fs = n->_factors;
    for (Factor* f : fs) remove_factor(f);
    detail::check(pus_remove_node(_h, n->_id));
    _nodes.remove(n);
  }
  const std::list<Node*>& get_nodes() const { return _nodes; }                     // Graph.h:61
  const std::list<Factor*>& get_factors() const { return _factors; }               // Graph.h:62
  int num_nodes() const { return (int)_nodes.size(); }
  int num_factors() const { return (int)_factors.size(); }
  int batch_optimization() { int it = 0; detail::check(pus_batch_optimize(_h, &it)); return it; }   // Slam.cpp:198-210
  UpdateStats update() {                                                            // Slam.cpp:157-196
    UpdateStats s; s.batch = (_step % (_prop.mod_batch > 0 ? _prop.mod_batch : 1)) == 0;
    detail::check(pus_update(_h));
    s.step = ++_step; return s;
  }
  double chi2() { double c = 0; detail::check(pus_chi2(_h, &c)); return c; }       // Slam.cpp:266-268
  // the error / Jacobian export at the current estimate (evaluated on the device; see pus_weighted_errors .. pus_local_chi2)
  VectorXd weighted_errors() {                                                      // Slam.cpp:254-264
    const long long rows = pus_weighted_errors(_h, nullptr, 0); detail::check((int)(rows < 0 ? -1 : 0));
    std::vector<double> e((size_t)rows);
    detail::check((int)(pus_weighted_errors(_h, e.data(), rows) < 0 ? -1 : 0));
    return to_vectorxd(e);
  }
  double normalized_chi2() { double c = 0; detail::check(pus_normalized_chi2(_h, &c)); return c; }                 // Slam.cpp:287-289
  double local_chi2(int last_n) { double c = 0; detail::check(pus_local_chi2(_h, last_n, &c)); return c; }       // Slam.cpp:270-285
  SparseJacobian jacobian() {                                                       // Slam.cpp:379-432
    SparseJacobian J;
    detail::check(pus_jacobian_dims(_h, &J.rows, &J.cols));
    const long long nnz = pus_jacobian(_h, nullptr, nullptr, nullptr, nullptr, 0); detail::check((int)(nnz < 0 ? -1 : 0));
    J.row_ptr.resize((size_t)J.rows + 1); J.col_idx.resize((size_t)nnz); J.values.resize((size_t)nnz); J.rhs.resize((size_t)J.rows);
    detail::check((int)(pus_jacobian(_h, J.row_ptr.data(), J.col_idx.data(), J.values.data(), J.rhs.data(), nnz) < 0 ? -1 : 0));
    return J;
  }
  void save(const std::string& fname) const { detail::check(pus_save_graph(_h, fname.c_str(), 0)); }   // Slam.cpp:84-89

  // ---- not in iSAM: the two per-solve loops of Mapper_mono that otherwise round-trip through the host ----
  // Mapper_mono::update_plane_measurement (Mapping.cpp:590-607) in one call: frames[f] = the frame's pose node,
  // seg_ptr / segs = its ground_seg2d_lines (CSR), and for every kept observation its factor, frame index and
  // plane row (good_plane_indices).  The factors' measurement() mirrors are refreshed.
  void refresh_plane_measurements(const std::vector<Pose3d_Node*>& frames, const std::vector<int>& seg_ptr,
                                  const std::vector<float>& segs, const float invK[9],
                                  const std::vector<Pose3d_Plane3d_Factor*>& facs, const std::vector<int>& fac_frame,
                                  const std::vector<int>& fac_row) {
    std::vector<int> ids(frames.size()), fids(facs.size());
    for (size_t i = 0; i < frames.size(); i++) ids[i] = frames[i]->unique_id();
    for (size_t i = 0; i < facs.size(); i++) fids[i] = facs[i]->unique_id();
    std::vector<double> m(4 * facs.size() + 4);
    detail::check(pus_refresh_plane_measurements(_h, (int)frames.size(), ids.data(), seg_ptr.data(), segs.data(), invK, (int)facs.size(),
                                                 fids.data(), fac_frame.data(), fac_row.data(), m.data()));
    for (size_t i = 0; i < facs.size(); i++) {
      Vector4d v; v(0) = m[4 * i]; v(1) = m[4 * i + 1]; v(2) = m[4 * i + 2]; v(3) = m[4 * i + 3];
      facs[i]->_mirror_measurement(Plane3d(v));
    }
  }
  // Plane3d::project_to_plane over all polygon vertices (Mapper_mono::reproj_to_newplane, Mapping.cpp:609-632):
  // xyz[3*i..] is replaced by its projection onto the current estimate of planes[i]
  void project_to_planes(const std::vector<Plane3d_Node*>& planes, std::vector<float>& xyz) {
    std::vector<int> ids(planes.size());
    for (size_t i = 0; i < planes.size(); i++) ids[i] = planes[i]->unique_id();
    std::vector<float> out(xyz.size());
    detail::check(pus_project_to_planes(_h, (int)planes.size(), ids.data(), xyz.data(), out.data()));
    xyz.swap(out);
  }
};

// aliases for BASELINE.json's g2o-flavoured vocabulary (no g2o code exists upstream)
typedef Pose3d_Node VertexSE3Expmap;
typedef Plane3d_Node VertexPlane;
typedef Pose3d_Plane3d_Factor EdgeSE3Plane;
typedef Pose3d_Pose3d_Factor EdgeSE3Expmap;

}  // namespace isam
