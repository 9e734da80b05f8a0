// ORACLE — TEST INFRASTRUCTURE ONLY.  Not linked, imported or executed by the product
// (lio_mapping_b200/); only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
// --impl reference legs may use anything under oracle/.
//
// Dependency-free small linear algebra used by the CPU restatement of hyye/lio-mapping's hot
// path.  The reference gets all of this from Eigen 3.3 (un-vendored, absent in this image:
// "parity unpinned" w.r.t. Eigen's exact floating-point association — see DESIGN.md §oracle).
// Conventions follow Eigen's public semantics: quaternion storage (x,y,z,w), Hamilton product,
// q*v rotates v, row/col-major noted per use.
#pragma once
#include <cmath>
#include <cstddef>
#include <cstring>
#include <vector>
#include <algorithm>
#include <limits>

namespace orc {

template <typename T> struct Vec3 {
  T x, y, z;
  Vec3() : x(0), y(0), z(0) {}
  Vec3(T a, T b, T c) : x(a), y(b), z(c) {}
  T operator[](int i) const { return i == 0 ? x : (i == 1 ? y : z); }
  T &operator[](int i) { return i == 0 ? x : (i == 1 ? y : z); }
  Vec3 operator+(const Vec3 &o) const { return Vec3(x + o.x, y + o.y, z + o.z); }
  Vec3 operator-(const Vec3 &o) const { return Vec3(x - o.x, y - o.y, z - o.z); }
  Vec3 operator-() const { return Vec3(-x, -y, -z); }
  Vec3 operator*(T s) const { return Vec3(x * s, y * s, z * s); }
  Vec3 operator/(T s) const { return Vec3(x / s, y / s, z / s); }
  Vec3 &operator+=(const Vec3 &o) { x += o.x; y += o.y; z += o.z; return *this; }
  Vec3 &operator-=(const Vec3 &o) { x -= o.x; y -= o.y; z -= o.z; return *this; }
  T dot(const Vec3 &o) const { return x * o.x + y * o.y + z * o.z; }
  Vec3 cross(const Vec3 &o) const {
    return Vec3(y * o.z - z * o.y, z * o.x - x * o.z, x * o.y - y * o.x);
  }
  T squaredNorm() const { return x * x + y * y + z * z; }
  T norm() const { return std::sqrt(squaredNorm()); }
  template <typename U> Vec3<U> cast() const { return Vec3<U>((U)x, (U)y, (U)z); }
};
template <typename T> inline Vec3<T> operator*(T s, const Vec3<T> &v) { return v * s; }

template <typename T> struct Mat3 {
  T m[3][3];
  Mat3() { std::memset(m, 0, sizeof(m)); }
  static Mat3 Identity() { Mat3 r; r.m[0][0] = r.m[1][1] = r.m[2][2] = 1; return r; }
  T operator()(int i, int j) const { return m[i][j]; }
  T &operator()(int i, int j) { return m[i][j]; }
  Mat3 operator*(const Mat3 &o) const {
    Mat3 r;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        T s = 0;
        for (int k = 0; k < 3; ++k) s += m[i][k] * o.m[k][j];
        r.m[i][j] = s;
      }
    return r;
  }
  Vec3<T> operator*(const Vec3<T> &v) const {
    return Vec3<T>(m[0][0] * v.x + m[0][1] * v.y + m[0][2] * v.z,
                   m[1][0] * v.x + m[1][1] * v.y + m[1][2] * v.z,
                   m[2][0] * v.x + m[2][1] * v.y + m[2][2] * v.z);
  }
  Mat3 operator*(T s) const { Mat3 r; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r.m[i][j] = m[i][j] * s; return r; }
  Mat3 operator+(const Mat3 &o) const { Mat3 r; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r.m[i][j] = m[i][j] + o.m[i][j]; return r; }
  Mat3 operator-(const Mat3 &o) const { Mat3 r; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r.m[i][j] = m[i][j] - o.m[i][j]; return r; }
  Mat3 operator-() const { Mat3 r; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r.m[i][j] = -m[i][j]; return r; }
  Mat3 transpose() const { Mat3 r; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r.m[i][j] = m[j][i]; return r; }
  Vec3<T> col(int j) const { return Vec3<T>(m[0][j], m[1][j], m[2][j]); }
  template <typename U> Mat3<U> cast() const { Mat3<U> r; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r.m[i][j] = (U)m[i][j]; return r; }
};
template <typename T> inline Mat3<T> operator*(T s, const Mat3<T> &a) { return a * s; }

// mathutils::SkewSymmetric (include/utils/math_utils.h:130-137)
template <typename T> inline Mat3<T> Skew(const Vec3<T> &v) {
  Mat3<T> r;
  r(0, 1) = -v.z; r(0, 2) = v.y;
  r(1, 0) = v.z;  r(1, 2) = -v.x;
  r(2, 0) = -v.y; r(2, 1) = v.x;
  return r;
}

template <typename T> struct Quat {
  T x, y, z, w;
  Quat() : x(0), y(0), z(0), w(1) {}
  Quat(T w_, T x_, T y_, T z_) : x(x_), y(y_), z(z_), w(w_) {}  // Eigen ctor order (w,x,y,z)
  Vec3<T> vec() const { return Vec3<T>(x, y, z); }
  Quat conjugate() const { return Quat(w, -x, -y, -z); }
  T squaredNorm() const { return x * x + y * y + z * z + w * w; }
  T norm() const { return std::sqrt(squaredNorm()); }
  Quat normalized() const { T n = norm(); return Quat(w / n, x / n, y / n, z / n); }
  void normalize() { *this = normalized(); }
  // Eigen: inverse() = conjugate / squaredNorm
  Quat inverse() const {
    T n2 = squaredNorm();
    return Quat(w / n2, -x / n2, -y / n2, -z / n2);
  }
  // Hamilton product (Eigen generic quat_product).
  Quat operator*(const Quat &b) const {
    return Quat(w * b.w - x * b.x - y * b.y - z * b.z,
                w * b.x + x * b.w + y * b.z - z * b.y,
                w * b.y + y * b.w + z * b.x - x * b.z,
                w * b.z + z * b.w + x * b.y - y * b.x);
  }
  // Eigen 3.3 QuaternionBase::_transformVector: v + w*2(q x v) + q x 2(q x v)
  Vec3<T> operator*(const Vec3<T> &v) const {
    Vec3<T> q = vec();
    Vec3<T> uv = q.cross(v);
    uv += uv;
    return v + uv * w + q.cross(uv);
  }
  // Eigen QuaternionBase::toRotationMatrix
  Mat3<T> toRotationMatrix() const {
    Mat3<T> r;
    const T tx = T(2) * x, ty = T(2) * y, tz = T(2) * z;
    const T twx = tx * w, twy = ty * w, twz = tz * w;
    const T txx = tx * x, txy = ty * x, txz = tz * x;
    const T tyy = ty * y, tyz = tz * y, tzz = tz * z;
    r(0, 0) = T(1) - (tyy + tzz); r(0, 1) = txy - twz;          r(0, 2) = txz + twy;
    r(1, 0) = txy + twz;          r(1, 1) = T(1) - (txx + tzz); r(1, 2) = tyz - twx;
    r(2, 0) = txz - twy;          r(2, 1) = tyz + twx;          r(2, 2) = T(1) - (txx + tyy);
    return r;
  }
  // Eigen quaternionbase_assign_impl<Matrix3> (Shepperd)
  static Quat fromRotationMatrix(const Mat3<T> &mat) {
    Quat q;
    T t = mat(0, 0) + mat(1, 1) + mat(2, 2);
    if (t > T(0)) {
      t = std::sqrt(t + T(1.0));
      q.w = T(0.5) * t;
      t = T(0.5) / t;
      q.x = (mat(2, 1) - mat(1, 2)) * t;
      q.y = (mat(0, 2) - mat(2, 0)) * t;
      q.z = (mat(1, 0) - mat(0, 1)) * t;
    } else {
      int i = 0;
      if (mat(1, 1) > mat(0, 0)) i = 1;
      if (mat(2, 2) > mat(i, i)) i = 2;
      int j = (i + 1) % 3;
      int k = (j + 1) % 3;
      t = std::sqrt(mat(i, i) - mat(j, j) - mat(k, k) + T(1.0));
      T c[3];
      c[i] = T(0.5) * t;
      t = T(0.5) / t;
      q.w = (mat(k, j) - mat(j, k)) * t;
      c[j] = (mat(j, i) + mat(i, j)) * t;
      c[k] = (mat(k, i) + mat(i, k)) * t;
      q.x = c[0]; q.y = c[1]; q.z = c[2];
    }
    return q;
  }
  T dot(const Quat &o) const { return x * o.x + y * o.y + z * o.z + w * o.w; }
  // Eigen QuaternionBase::slerp
  Quat slerp(T t, const Quat &other) const {
    const T one = T(1) - std::numeric_limits<T>::epsilon();
    T d = this->dot(other);
    T absD = std::abs(d);
    T scale0, scale1;
    if (absD >= one) {
      scale0 = T(1) - t;
      scale1 = t;
    } else {
      T theta = std::acos(absD);
      T sinTheta = std::sin(theta);
      scale0 = std::sin((T(1) - t) * theta) / sinTheta;
      scale1 = std::sin((t * theta)) / sinTheta;
    }
    if (d < T(0)) scale1 = -scale1;
    return Quat(scale0 * w + scale1 * other.w, scale0 * x + scale1 * other.x,
                scale0 * y + scale1 * other.y, scale0 * z + scale1 * other.z);
  }
  // Eigen QuaternionBase::angularDistance
  T angularDistance(const Quat &other) const {
    Quat d = (*this) * other.conjugate();
    return T(2) * std::atan2(d.vec().norm(), std::abs(d.w));
  }
  template <typename U> Quat<U> cast() const { return Quat<U>((U)w, (U)x, (U)y, (U)z); }
};

// mathutils::DeltaQ (include/utils/math_utils.h:116-129): (1, theta/2) — NOT normalised.
template <typename T> inline Quat<T> DeltaQ(const Vec3<T> &theta) {
  return Quat<T>(T(1), theta.x / T(2), theta.y / T(2), theta.z / T(2));
}

// lio::Twist<T> (include/utils/Twist.h:40-97). All compositions go through a 3x3 rotation
// matrix + translation exactly like the Eigen::Transform round trip in the reference.
template <typename T> struct Twist {
  Quat<T> rot;
  Vec3<T> pos;
  Twist() {}
  Twist(const Quat<T> &r, const Vec3<T> &p) : rot(r), pos(p) {}
  static Twist fromAffine(const Mat3<T> &lin, const Vec3<T> &t) {  // Twist(Eigen::Transform) :55-58
    return Twist(Quat<T>::fromRotationMatrix(lin).normalized(), t);
  }
  Mat3<T> linear() const { return rot.normalized().toRotationMatrix(); }  // transform() :60-65
  Twist inverse() const {  // :67-73 (Affine inverse: R^T, -R^T t); rot NOT re-normalised
    Mat3<T> Rt = linear().transpose();
    Twist r;
    r.rot = Quat<T>::fromRotationMatrix(Rt);
    r.pos = -(Rt * pos);
    return r;
  }
  Twist operator*(const Twist &o) const {  // :75-78
    Mat3<T> R = linear() * o.linear();
    Vec3<T> t = linear() * o.pos + pos;
    return fromAffine(R, t);
  }
  template <typename U> Twist<U> cast() const { return Twist<U>(rot.template cast<U>(), pos.template cast<U>()); }
};

// ---------------------------------------------------------------------------------------------
// Dynamic dense matrix, row-major, double (Eigen::MatrixXd stand-in for the fp64 solver parts).
struct MatX {
  int r = 0, c = 0;
  std::vector<double> d;
  MatX() {}
  MatX(int r_, int c_) : r(r_), c(c_), d((size_t)r_ * c_, 0.0) {}
  double &operator()(int i, int j) { return d[(size_t)i * c + j]; }
  double operator()(int i, int j) const { return d[(size_t)i * c + j]; }
  void setZero() { std::fill(d.begin(), d.end(), 0.0); }
  MatX transpose() const {
    MatX t(c, r);
    for (int i = 0; i < r; ++i) for (int j = 0; j < c; ++j) t(j, i) = (*this)(i, j);
    return t;
  }
};
typedef std::vector<double> VecX;

inline MatX matmul(const MatX &a, const MatX &b) {
  MatX o(a.r, b.c);
  for (int i = 0; i < a.r; ++i)
    for (int k = 0; k < a.c; ++k) {
      double aik = a(i, k);
      if (aik == 0.0) continue;
      for (int j = 0; j < b.c; ++j) o(i, j) += aik * b(k, j);
    }
  return o;
}
inline VecX matvec(const MatX &a, const VecX &x) {
  VecX o(a.r, 0.0);
  for (int i = 0; i < a.r; ++i) {
    double s = 0;
    for (int j = 0; j < a.c; ++j) s += a(i, j) * x[j];
    o[i] = s;
  }
  return o;
}

// In-place lower Cholesky (A = L L^T); returns false if a pivot is <= 0 or not finite.
inline bool cholesky_lower(MatX &a) {
  int n = a.r;
  for (int j = 0; j < n; ++j) {
    double s = a(j, j);
    for (int k = 0; k < j; ++k) s -= a(j, k) * a(j, k);
    if (!(s > 0.0) || !std::isfinite(s)) return false;
    double l = std::sqrt(s);
    a(j, j) = l;
    for (int i = j + 1; i < n; ++i) {
      double t = a(i, j);
      for (int k = 0; k < j; ++k) t -= a(i, k) * a(j, k);
      a(i, j) = t / l;
    }
  }
  for (int i = 0; i < n; ++i) for (int j = i + 1; j < n; ++j) a(i, j) = 0.0;
  return true;
}
inline void chol_solve(const MatX &L, VecX &b) {  // solves L L^T x = b in place
  int n = L.r;
  for (int i = 0; i < n; ++i) {
    double s = b[i];
    for (int k = 0; k < i; ++k) s -= L(i, k) * b[k];
    b[i] = s / L(i, i);
  }
  for (int i = n - 1; i >= 0; --i) {
    double s = b[i];
    for (int k = i + 1; k < n; ++k) s -= L(k, i) * b[k];
    b[i] = s / L(i, i);
  }
}

// Symmetric eigen-decomposition by cyclic Jacobi rotations; eigenvalues ascending (the order
// Eigen::SelfAdjointEigenSolver guarantees), eigenvectors in the columns of V.
template <typename T>
inline void sym_eigen_jacobi(int n, const T *A_in, T *evals, T *V /* n*n row-major */) {
  std::vector<T> A(A_in, A_in + (size_t)n * n);
  for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) V[i * n + j] = (i == j) ? T(1) : T(0);
  for (int sweep = 0; sweep < 100; ++sweep) {
    T off = 0, diag = 0;
    for (int i = 0; i < n; ++i) {
      diag += A[i * n + i] * A[i * n + i];
      for (int j = i + 1; j < n; ++j) off += A[i * n + j] * A[i * n + j];
    }
    if (off <= std::numeric_limits<T>::epsilon() * std::numeric_limits<T>::epsilon() * diag || off == T(0)) break;
    for (int p = 0; p < n - 1; ++p)
      for (int q = p + 1; q < n; ++q) {
        T apq = A[p * n + q];
        if (apq == T(0)) continue;
        T app = A[p * n + p], aqq = A[q * n + q];
        T theta = (aqq - app) / (T(2) * apq);
        T t = (theta >= 0 ? T(1) : T(-1)) / (std::abs(theta) + std::sqrt(theta * theta + T(1)));
        T c = T(1) / std::sqrt(t * t + T(1)), s = t * c;
        for (int k = 0; k < n; ++k) {
          T akp = A[k * n + p], akq = A[k * n + q];
          A[k * n + p] = c * akp - s * akq;
          A[k * n + q] = s * akp + c * akq;
        }
        for (int k = 0; k < n; ++k) {
          T apk = A[p * n + k], aqk = A[q * n + k];
          A[p * n + k] = c * apk - s * aqk;
          A[q * n + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < n; ++k) {
          T vkp = V[k * n + p], vkq = V[k * n + q];
          V[k * n + p] = c * vkp - s * vkq;
          V[k * n + q] = s * vkp + c * vkq;
        }
      }
  }
  std::vector<int> idx(n);
  for (int i = 0; i < n; ++i) idx[i] = i;
  std::sort(idx.begin(), idx.end(), [&](int a, int b) { return A[a * n + a] < A[b * n + b]; });
  std::vector<T> Vc(V, V + (size_t)n * n);
  for (int j = 0; j < n; ++j) {
    evals[j] = A[idx[j] * n + idx[j]];
    for (int k = 0; k < n; ++k) V[k * n + j] = Vc[k * n + idx[j]];
  }
}

// Eigen 3.3 ColPivHouseholderQR<Matrix<T,R,C>>::compute + solve restated for small dense
// systems (used for the 5x3 plane fit, Estimator.cc:1027, and the 6x6 GN step, :1306).
// a: R x C row-major (overwritten), b: R (overwritten), x: C.  Sequential summation order.
template <typename T, int R, int C>
inline void colpiv_householder_qr_solve(T a[R][C], T b[R], T x[C]) {
  const int size = (R < C) ? R : C;
  T hCoeffs[size];
  int colsTranspositions[size];
  T colNormsUpdated[C], colNormsDirect[C];
  for (int k = 0; k < C; ++k) {
    T s = 0;
    for (int i = 0; i < R; ++i) s += a[i][k] * a[i][k];
    colNormsDirect[k] = std::sqrt(s);
    colNormsUpdated[k] = colNormsDirect[k];
  }
  T maxn = colNormsUpdated[0];
  for (int k = 1; k < C; ++k) if (colNormsUpdated[k] > maxn) maxn = colNormsUpdated[k];
  const T eps = std::numeric_limits<T>::epsilon();
  T th = maxn * eps;
  const T threshold_helper = (th * th) / T(R);
  const T norm_downdate_threshold = std::sqrt(eps);
  int nonzero_pivots = size;
  T maxpivot = 0;
  for (int k = 0; k < size; ++k) {
    int biggest = k;
    T bn = colNormsUpdated[k];
    for (int j = k + 1; j < C; ++j) if (colNormsUpdated[j] > bn) { bn = colNormsUpdated[j]; biggest = j; }
    T biggest_sq = bn * bn;
    if (nonzero_pivots == size && biggest_sq < threshold_helper * T(R - k)) nonzero_pivots = k;
    colsTranspositions[k] = biggest;
    if (k != biggest) {
      for (int i = 0; i < R; ++i) std::swap(a[i][k], a[i][biggest]);
      std::swap(colNormsUpdated[k], colNormsUpdated[biggest]);
      std::swap(colNormsDirect[k], colNormsDirect[biggest]);
    }
    // makeHouseholderInPlace on a[k..R-1][k]
    T tailSqNorm = 0;
    for (int i = k + 1; i < R; ++i) tailSqNorm += a[i][k] * a[i][k];
    T c0 = a[k][k];
    T tau, beta;
    const T tol = std::numeric_limits<T>::min();
    if (R - k == 1 || tailSqNorm <= tol) {
      tau = 0; beta = c0;
      for (int i = k + 1; i < R; ++i) a[i][k] = 0;
    } else {
      beta = std::sqrt(c0 * c0 + tailSqNorm);
      if (c0 >= 0) beta = -beta;
      T den = c0 - beta;
      for (int i = k + 1; i < R; ++i) a[i][k] = a[i][k] / den;
      tau = (beta - c0) / beta;
    }
    hCoeffs[k] = tau;
    a[k][k] = beta;
    if (std::abs(beta) > maxpivot) maxpivot = std::abs(beta);
    // applyHouseholderOnTheLeft to a[k..R-1][k+1..C-1]
    if (R - k == 1) {
      for (int j = k + 1; j < C; ++j) a[k][j] *= (T(1) - tau);
    } else if (tau != T(0)) {
      for (int j = k + 1; j < C; ++j) {
        T tmp = 0;
        for (int i = k + 1; i < R; ++i) tmp += a[i][k] * a[i][j];
        tmp += a[k][j];
        a[k][j] -= tau * tmp;
        for (int i = k + 1; i < R; ++i) a[i][j] -= tau * a[i][k] * tmp;
      }
    }
    // LAPACK-style column-norm downdating
    for (int j = k + 1; j < C; ++j) {
      if (colNormsUpdated[j] != T(0)) {
        T temp = std::abs(a[k][j]) / colNormsUpdated[j];
        temp = (T(1) + temp) * (T(1) - temp);
        temp = temp < T(0) ? T(0) : temp;
        T ratio = colNormsUpdated[j] / colNormsDirect[j];
        T temp2 = temp * (ratio * ratio);
        if (temp2 <= norm_downdate_threshold) {
          T s = 0;
          for (int i = k + 1; i < R; ++i) s += a[i][j] * a[i][j];
          colNormsDirect[j] = std::sqrt(s);
          colNormsUpdated[j] = colNormsDirect[j];
        } else {
          colNormsUpdated[j] *= std::sqrt(temp);
        }
      }
    }
  }
  // permutation indices from the transpositions
  int perm[C];
  for (int k = 0; k < C; ++k) perm[k] = k;
  for (int k = 0; k < size; ++k) std::swap(perm[k], perm[colsTranspositions[k]]);
  // solve: c = Q^T b
  for (int k = 0; k < nonzero_pivots; ++k) {
    T tau = hCoeffs[k];
    if (R - k == 1) { b[k] *= (T(1) - tau); continue; }
    if (tau == T(0)) continue;
    T tmp = 0;
    for (int i = k + 1; i < R; ++i) tmp += a[i][k] * b[i];
    tmp += b[k];
    b[k] -= tau * tmp;
    for (int i = k + 1; i < R; ++i) b[i] -= tau * a[i][k] * tmp;
  }
  // back substitution on the leading nonzero_pivots x nonzero_pivots upper triangle
  for (int i = nonzero_pivots - 1; i >= 0; --i) {
    T s = b[i];
    for (int j = i + 1; j < nonzero_pivots; ++j) s -= a[i][j] * b[j];
    b[i] = (s != T(0)) ? s / a[i][i] : s;  // Eigen divides only a nonzero rhs (triangular_solve_vector)
  }
  for (int k = 0; k < C; ++k) x[k] = 0;
  for (int i = 0; i < nonzero_pivots; ++i) x[perm[i]] = b[i];
  (void)maxpivot;
}

}  // namespace orc
