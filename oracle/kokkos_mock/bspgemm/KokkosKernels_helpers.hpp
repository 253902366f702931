// Minimal stand-ins for what the reference's sparse/impl/KokkosSparse_bspgemm_impl_seq.hpp and
// batched/dense/impl/KokkosBatched_Gemm_Serial_Internal.hpp use, so that both compile where they lie
// (oracle/kkref_bspgemm.cpp).  TEST INFRASTRUCTURE ONLY.
//   Kokkos::View     host rank-1 view (owning when constructed with a label, else a window on caller memory); its
//                    host mirror is itself, as for a HostSpace view
//   create_mirror_view / deep_copy (view <- view, view <- scalar) / fence / make_pair / subview(view, [first, last))
#pragma once
#include <cstddef>
#include <cstdint>
#include <memory>
#include <utility>
#include <vector>

#define KOKKOS_INLINE_FUNCTION inline
#define KOKKOS_RESTRICT __restrict__

namespace Kokkos {

template <class T>
class View {
 public:
  using value_type       = T;
  using host_mirror_type = View<T>;
  View() = default;
  View(T* p, size_t n) : p_(p), n_(n) {}
  View(const char*, size_t n) : own_(std::make_shared<std::vector<T>>(n, T(0))), p_(own_->data()), n_(n) {}
  T& operator()(size_t i) const { return p_[i]; }
  T* data() const { return p_; }
  size_t extent(int) const { return n_; }
  size_t size() const { return n_; }

 private:
  std::shared_ptr<std::vector<T>> own_;
  T* p_     = nullptr;
  size_t n_ = 0;
};

template <class T>
inline View<T> create_mirror_view(const View<T>& v) {
  return v;
}
template <class T>
inline void deep_copy(const View<T>& dst, const View<T>& src) {
  if (dst.data() == src.data()) return;
  for (size_t i = 0; i < dst.size(); ++i) dst(i) = src(i);
}
template <class T>
inline void deep_copy(const View<T>& dst, const T& v) {
  for (size_t i = 0; i < dst.size(); ++i) dst(i) = v;
}
inline void fence() {}

template <class A, class B>
inline std::pair<A, B> make_pair(A a, B b) {
  return std::pair<A, B>(a, b);
}
template <class T, class A, class B>
inline View<T> subview(const View<T>& v, std::pair<A, B> r) {
  return View<T>(v.data() + (int64_t)r.first, (size_t)((int64_t)r.second - (int64_t)r.first));
}

}  // namespace Kokkos

namespace KokkosBlas {
namespace Impl {
struct OpID {
  template <class T>
  KOKKOS_INLINE_FUNCTION T operator()(const T& v) const {
    return v;
  }
};
// A(i, j) = alpha / A(i, j) *= alpha over an m x n strided block (not reached with beta = 1, but named by the GEMM)
struct SerialSetInternal {
  template <class S, class V>
  KOKKOS_INLINE_FUNCTION static int invoke(int m, int n, const S alpha, V* A, int as0, int as1) {
    for (int i = 0; i < m; ++i)
      for (int j = 0; j < n; ++j) A[i * as0 + j * as1] = alpha;
    return 0;
  }
};
struct SerialScaleInternal {
  template <class S, class V>
  KOKKOS_INLINE_FUNCTION static int invoke(int m, int n, const S alpha, V* A, int as0, int as1) {
    for (int i = 0; i < m; ++i)
      for (int j = 0; j < n; ++j) A[i * as0 + j * as1] *= alpha;
    return 0;
  }
};
}  // namespace Impl
}  // namespace KokkosBlas
