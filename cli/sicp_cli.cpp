// sicp_cli — command-line front end of libsicp_b200 with the flag set of the reference CLIs
// (c++/src/simpleicp-cli.cpp:15-35, rust/src/main.rs:10-46):
//   -f/--fixed  -m/--movable  -c/--correspondences  -n/--neighbors  -p/--min_planarity
//   -o/--max_overlap_distance (<= 0: fully overlapping)  -i/--min_change  -x/--max_iterations
// plus  --out FILE (write the transformed movable cloud)  --device N  --quiet  --variant V.
// --variant python (default): the Python reference's semantics (raw MAD, converged non-linear
// solve); --variant linearized | cpp: the algorithm of the native reference CLIs themselves (one
// linear solve per iteration, 1.4826 MAD, sample std; "cpp" also reports H * dH as
// c++/src/simpleicp.cpp:66 does), see sicp_variant in include/sicp_b200.h.  Prints the reference's iteration table, H and "Finished in N.NNN seconds!" (the line
// scripts/benchmark.sh:43-51 greps; file I/O excluded from it, as in every reference CLI).
#include <cfenv>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "sicp_b200.h"

static void usage() {
  puts("A simple version of the ICP algorithm (H100 build).\nUsage:\n  sicp_cli [OPTION...]\n\n"
       "  -f, --fixed arg                 Path to fixed point cloud\n"
       "  -m, --movable arg               Path to movable point cloud\n"
       "  -c, --correspondences arg       Number of initially selected correspondences (default: 1000)\n"
       "  -n, --neighbors arg             Number of neighbors used for plane estimation (default: 10)\n"
       "  -p, --min_planarity arg         Minimal planarity value of planes used as correspondence (default: 0.3)\n"
       "  -o, --max_overlap_distance arg  Maximum initial overlap distance. Set to negative value if point\n"
       "                                  clouds are fully overlapping. (default: -1)\n"
       "  -i, --min_change arg            Minimal change of mean and standard deviation of distances (in\n"
       "                                  percent) needed to proceed to next iteration (default: 1)\n"
       "  -x, --max_iterations arg        Maximum number of iterations (default: 100)\n"
       "      --out arg                   Write the transformed movable cloud to this .xyz file\n"
       "      --device arg                CUDA device index (default: 0)\n"
       "      --variant arg               python | linearized | cpp (default: python)\n"
       "      --quiet                     Only print H\n"
       "  -h, --help                      Print usage");
}

#define CHECK(call)                                                          \
  do {                                                                       \
    int rc__ = (call);                                                       \
    if (rc__ != SICP_OK) {                                                   \
      fprintf(stderr, "Caught exception: %s\n", sicp_last_error(ctx));       \
      return 1;                                                              \
    }                                                                        \
  } while (0)

int main(int argc, char** argv) {
  std::string fixed, movable, out;
  long long correspondences = 1000;
  int neighbors = 10, max_iterations = 100, device = 0;
  double min_planarity = 0.3, max_overlap = -1.0, min_change = 1.0;
  bool quiet = false;
  int variant = SICP_VARIANT_PYTHON;
  if (argc == 1) {
    usage();
    return 0;
  }
  for (int i = 1; i < argc; ++i) {
    std::string a = argv[i];
    auto val = [&](const char* name) -> const char* {
      if (i + 1 >= argc) {
        fprintf(stderr, "Caught exception: option %s requires an argument\n", name);
        exit(1);
      }
      return argv[++i];
    };
    if (a == "-h" || a == "--help") { usage(); return 0; }
    else if (a == "-f" || a == "--fixed") fixed = val("--fixed");
    else if (a == "-m" || a == "--movable") movable = val("--movable");
    else if (a == "-c" || a == "--correspondences") correspondences = atoll(val("--correspondences"));
    else if (a == "-n" || a == "--neighbors") neighbors = atoi(val("--neighbors"));
    else if (a == "-p" || a == "--min_planarity") min_planarity = atof(val("--min_planarity"));
    else if (a == "-o" || a == "--max_overlap_distance") max_overlap = atof(val("--max_overlap_distance"));
    else if (a == "-i" || a == "--min_change") min_change = atof(val("--min_change"));
    else if (a == "-x" || a == "--max_iterations") max_iterations = atoi(val("--max_iterations"));
    else if (a == "--out") out = val("--out");
    else if (a == "--device") device = atoi(val("--device"));
    else if (a == "--quiet") quiet = true;
    else if (a == "--variant") {
      const std::string v = val("--variant");
      if (v == "python") variant = SICP_VARIANT_PYTHON;
      else if (v == "linearized") variant = SICP_VARIANT_LINEARIZED;
      else if (v == "cpp") variant = SICP_VARIANT_LINEARIZED_CPP;
      else { fprintf(stderr, "Caught exception: unknown variant '%s'\n", v.c_str()); return 1; }
    }
    else { fprintf(stderr, "Caught exception: Option '%s' does not exist\n", a.c_str()); return 1; }
  }
  if (fixed.empty() || movable.empty()) {
    fprintf(stderr, "Caught exception: --fixed and --movable are required\n");
    return 1;
  }
  double *xf = nullptr, *xm = nullptr;
  int64_t nf = 0, nm = 0;
  if (sicp_xyz_load(fixed.c_str(), &xf, &nf) != SICP_OK || sicp_xyz_load(movable.c_str(), &xm, &nm) != SICP_OK) {
    fprintf(stderr, "Caught exception: %s\n", sicp_io_last_error());
    return 1;
  }
  sicp_ctx* ctx = nullptr;
  if (sicp_create(device, nullptr, &ctx) != SICP_OK) {
    fprintf(stderr, "Caught exception: %s\n", sicp_last_error(nullptr));
    return 1;
  }
  const auto t0 = std::chrono::steady_clock::now();
  CHECK(sicp_set_option(ctx, "variant", (double)variant));
  CHECK(sicp_set_clouds(ctx, xf, nf, xm, nm));
  std::vector<int64_t> idx;
  int64_t m = nf;
  const double I4[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  if (max_overlap > 0) {
    if (!quiet) puts("Consider partial overlap of point clouds ...");
    CHECK(sicp_set_selected(ctx, nullptr, nf));
    std::vector<uint8_t> keep((size_t)nf);
    int64_t nk = 0;
    CHECK(sicp_select_in_range(ctx, I4, max_overlap, keep.data(), &nk));
    idx.reserve((size_t)nk);
    for (int64_t i = 0; i < nf; ++i)
      if (keep[(size_t)i]) idx.push_back(i);
    m = nk;
  }
  if (!quiet) puts("Select points for correspondences in fixed point cloud ...");
  if (m > correspondences) {
    // rint(linspace(0, m - 1, n)) with round-half-even (python/simpleicp/pointcloud.py:142-144);
    // the native CLIs round half away from zero (c++/src/pointcloud.cpp:92-96)
    std::fesetround(FE_TONEAREST);
    std::vector<int64_t> pick((size_t)correspondences);
    const double step = (double)(m - 1) / (double)(correspondences - 1);
    for (long long i = 0; i < correspondences; ++i) {
      const double y = (i == correspondences - 1) ? (double)(m - 1) : (double)i * step;
      const int64_t p = (int64_t)(variant == SICP_VARIANT_PYTHON ? std::nearbyint(y) : std::round(y));
      pick[(size_t)i] = idx.empty() ? p : idx[(size_t)p];
    }
    idx.swap(pick);
  }
  if (idx.empty() && m == nf) CHECK(sicp_set_selected(ctx, nullptr, nf));
  else CHECK(sicp_set_selected(ctx, idx.data(), (int64_t)idx.size()));
  if (!quiet) puts("Estimate normals of selected points ...");
  CHECK(sicp_estimate_normals(ctx, neighbors, nullptr, nullptr, nullptr, nullptr));
  if (!quiet) puts("Start iterations ...");
  sicp_run_params p;
  memset(&p, 0, sizeof(p));
  p.min_planarity = min_planarity;
  p.min_change = min_change;
  p.max_iterations = max_iterations;
  p.lsq.distance_weight = 1.0;
  sicp_run_result res;
  std::vector<sicp_iter_record> log((size_t)max_iterations);
  CHECK(sicp_run(ctx, &p, &res, log.data()));
  std::vector<double> xt((size_t)nm * 3);
  double T[16];
  CHECK(sicp_get_transform(ctx, T));  // == res.H except for --variant cpp
  CHECK(sicp_transform(ctx, T, xt.data()));
  const double secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  if (!quiet) {
    const int rows = res.converged ? res.iterations - 1 : res.iterations;
    for (int it = 0; it < rows; ++it) {
      if (it == 0) {
        printf("%9s | %15s | %15s | %15s\n", "Iteration", "correspondences", "mean(residuals)", "std(residuals)");
        printf("%9s | %15lld | %15.4f | %15.4f\n", "orig:0", (long long)log[0].n_kept, log[0].mean_dist, log[0].std_dist);
      }
      printf("%9d | %15lld | %15.4f | %15.4f\n", it + 1, (long long)log[(size_t)it].n_kept, log[(size_t)it].mean_res,
             log[(size_t)it].std_res);
    }
    if (res.converged) puts("Convergence criteria fulfilled -> stop iteration!");
    puts("Estimated transformation matrix H:");
  }
  for (int i = 0; i < 4; ++i)
    printf("[%12.6f %12.6f %12.6f %12.6f]\n", res.H[4 * i], res.H[4 * i + 1], res.H[4 * i + 2], res.H[4 * i + 3]);
  if (!quiet) printf("Finished in %.3f seconds!\n", secs);
  if (!out.empty() && sicp_xyz_save(out.c_str(), xt.data(), nm, 6, 1) != SICP_OK) {
    fprintf(stderr, "Caught exception: %s\n", sicp_io_last_error());
    return 1;
  }
  sicp_destroy(ctx);
  sicp_xyz_free(xf);
  sicp_xyz_free(xm);
  return 0;
}
