// The reference-side binding of INTEGRATION.md section 5, as code that compiles and runs.
//
// This translation unit defines the C++ reference's entry point
//
//   Eigen::Matrix<double, 4, 4> SimpleICP(X_fix, X_mov, correspondences, neighbors, min_planarity,
//                                         max_overlap_distance, min_change, max_iterations)
//
// exactly as /root/reference/c++/src/simpleicp.h:11-18 declares it, on top of the C ABI of
// libsicp_b200.so (include/sicp_b200.h) and nothing else.  It REPLACES c++/src/simpleicp.cpp,
// pointcloud.cpp and corrpts.cpp in the reference's build: linked with the reference's own,
// unmodified c++/src/simpleicp-cli.cpp it gives the reference CLI running on the H100
// (built by the recipe that also builds the CPU reference for the tests, oracle/Makefile target
// _ref/simpleicp_cpp_b200; tests/test_gpu_linearized.py runs it).
// Same arguments and defaults, same screen output (simpleicp.cpp:17-127), same exception for
// non-overlapping clouds (simpleicp.cpp:26-36).
//
// The only Eigen interface used is MatrixXd::rows() / operator()(i, j) / Matrix4d::operator(),
// so the file builds against real Eigen and against oracle/cpp_standin alike.
#include "simpleicp.h"  // the reference's header: the signature this file implements

#include "sicp_b200.h"

#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

namespace
{

struct Ctx
{
  sicp_ctx *p = nullptr;
  ~Ctx()
  {
    if (p)
      sicp_destroy(p);
  }
};

std::vector<double> row_major(const Eigen::MatrixXd &X)
{
  const long n = static_cast<long>(X.rows());
  std::vector<double> out(static_cast<size_t>(3 * n));
  for (long i = 0; i < n; i++)
    for (int j = 0; j < 3; j++)
      out[static_cast<size_t>(3 * i + j)] = X(i, j);
  return out;
}

} // namespace

Eigen::Matrix<double, 4, 4> SimpleICP(const Eigen::MatrixXd &X_fix,
                                      const Eigen::MatrixXd &X_mov,
                                      const int &correspondences,
                                      const int &neighbors,
                                      const double &min_planarity,
                                      const double &max_overlap_distance,
                                      const double &min_change,
                                      const int &max_iterations)
{
  auto start = std::chrono::system_clock::now();

  printf("Create point cloud objects ...\n");
  const std::vector<double> fix = row_major(X_fix), mov = row_major(X_mov);
  Ctx ctx;
  if (sicp_create(0, nullptr, &ctx.p) != SICP_OK)
    throw std::runtime_error(sicp_last_error(nullptr));
  auto check = [&](int32_t rc) {
    if (rc != SICP_OK)
      throw std::runtime_error(sicp_last_error(ctx.p));
  };
  // the C++ driver's semantics: one linear solve per iteration, 1.4826 * MAD, H_new = H_old * dH
  check(sicp_set_option(ctx.p, "variant", static_cast<double>(SICP_VARIANT_LINEARIZED_CPP)));

  if (max_overlap_distance > 0)
    printf("Consider partial overlap of point clouds ...\n");
  printf("Select points for correspondences in fixed point cloud ...\n");
  printf("Estimate normals of selected points ...\n");
  printf("Start iterations ...\n");

  sicp_register_params rp;
  std::memset(&rp, 0, sizeof(rp));
  rp.correspondences = correspondences;
  rp.neighbors = neighbors;
  rp.max_overlap_distance = max_overlap_distance; // <= 0: fully overlapping, as the CLI's -1
  rp.run.min_planarity = min_planarity;
  rp.run.min_change = min_change;
  rp.run.max_iterations = max_iterations;
  rp.run.lsq.distance_weight = 1.0;
  sicp_run_result res;
  std::vector<sicp_iter_record> log(static_cast<size_t>(max_iterations > 0 ? max_iterations : 1));
  const int32_t rc = sicp_register(ctx.p, fix.data(), static_cast<int64_t>(X_fix.rows()), mov.data(),
                                   static_cast<int64_t>(X_mov.rows()), &rp, &res, log.data(), nullptr, nullptr);
  if (rc == SICP_ERR_NO_OVERLAP)
  {
    char buff[200];
    snprintf(buff, sizeof(buff),
             "Point clouds do not overlap within max_overlap_distance = %.5f. "
             "Consider increasing the value of max_overlap_distance.\n",
             max_overlap_distance);
    throw std::runtime_error(std::string(buff));
  }
  check(rc);

  // the table of simpleicp.cpp:82-101: the iteration that met the stop rule is not printed
  const int rows = res.converged ? res.iterations - 1 : res.iterations;
  for (int i = 0; i < rows; i++)
  {
    if (i == 0)
    {
      printf("%9s | %15s | %15s | %15s\n", "Iteration", "correspondences", "mean(residuals)", "std(residuals)");
      printf("%9s | %15d | %15.4f | %15.4f\n", "orig:0", static_cast<int>(log[0].n_kept), log[0].mean_dist,
             log[0].std_dist);
    }
    printf("%9d | %15d | %15.4f | %15.4f\n", i + 1, static_cast<int>(log[static_cast<size_t>(i)].n_kept),
           log[static_cast<size_t>(i)].mean_res, log[static_cast<size_t>(i)].std_res);
  }
  if (res.converged)
    printf("Convergence criteria fulfilled -> stop iteration!\n");

  Eigen::Matrix<double, 4, 4> H_new;
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++)
      H_new(i, j) = res.H[4 * i + j];

  printf("Estimated transformation matrix H:\n");
  for (int i = 0; i < 4; i++)
    printf("[%12.6f %12.6f %12.6f %12.6f]\n", H_new(i, 0), H_new(i, 1), H_new(i, 2), H_new(i, 3));

  auto end = std::chrono::system_clock::now();
  std::chrono::duration<double> elapsed_seconds = end - start;
  printf("Finished in %.3f seconds!\n", elapsed_seconds.count());

  return H_new;
}
