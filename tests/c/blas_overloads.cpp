// A C++ caller of the four inline libxsmm_gemm overloads of include/libxsmm.h (f64 / f32, m n k by pointer / by value), compiled with
// g++ -Wall -Werror and linked with -lxsmm.
//
//   blas_overloads reject   each overload with lda < m: every call prints "LIBXSMM_GEMM failed" and C keeps its bytes (no GPU needed)
//   blas_overloads run      each overload on HOST buffers, C += A B (beta 1, alpha NULL), against a triple loop in the exact-order
//                           kernel's order: prints "max_abs_diff <x>"
#include <libxsmm.h>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

template <typename T> static double check(bool by_value, bool run) {
  const libxsmm_blasint m = 19, n = 6, k = 11, ld = run ? m : 4;   // ld < m is rejected
  std::vector<T> a(static_cast<size_t>(m) * k), b(static_cast<size_t>(k) * n), c(static_cast<size_t>(m) * n), want;
  for (size_t i = 0; i < a.size(); ++i) a[i] = static_cast<T>(static_cast<int>((i * 7) % 23) - 11) / static_cast<T>(7);
  for (size_t i = 0; i < b.size(); ++i) b[i] = static_cast<T>(static_cast<int>((i * 5) % 19) - 9) / static_cast<T>(3);
  for (size_t i = 0; i < c.size(); ++i) c[i] = static_cast<T>(static_cast<int>(i % 17) - 8) / static_cast<T>(5);
  want = c;
  if (by_value) libxsmm_gemm("N", "N", m, n, k, nullptr, a.data(), &ld, b.data(), nullptr, nullptr, c.data(), nullptr);
  else libxsmm_gemm("N", "N", &m, &n, &k, nullptr, a.data(), &ld, b.data(), nullptr, nullptr, c.data(), nullptr);
  if (run) {
    for (libxsmm_blasint j = 0; j < n; ++j) for (libxsmm_blasint i = 0; i < m; ++i)
      for (libxsmm_blasint s = 0; s < k; ++s) want[j * m + i] += a[s * m + i] * b[j * k + s];
  }
  double diff = 0;
  for (size_t i = 0; i < c.size(); ++i) diff = std::fmax(diff, std::isnan(static_cast<double>(c[i])) ? INFINITY : std::fabs(static_cast<double>(c[i] - want[i])));
  return diff;
}

int main(int argc, char* argv[]) {
  const bool run = argc > 1 && 0 == std::strcmp(argv[1], "run");
  const double diff = std::fmax(std::fmax(check<double>(false, run), check<double>(true, run)), std::fmax(check<float>(false, run), check<float>(true, run)));
  if (run) std::printf("max_abs_diff %.3e\n", diff);
  else std::printf(diff == 0 ? "reject ok\n" : "C was written\n");
  return (diff == 0) ? 0 : 2;
}
