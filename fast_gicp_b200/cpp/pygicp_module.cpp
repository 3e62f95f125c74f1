// pygicp -- the reference's Python module (src/python/main.cpp:21-224) rebuilt on the C++ mirror classes: same function
// and method names, same defaults.  Only the VGICP_CUDA method exists here (the CPU variants and NDT are outside the
// accelerated path; asking for them prints the reference's error message and returns identity, main.cpp:117-139).
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <array>
#include <cstring>
#include <iostream>
#include <limits>
#include <unordered_map>

#include <fast_gicp_b200/fast_vgicp_cuda.hpp>
#include <fast_gicp_b200/ndt_cuda.hpp>

#include "../../include/vgicp_prep_b200.h"

namespace py = pybind11;
using Cloud = pcl::PointCloud<pcl::PointXYZ>;
using LsqReg = fast_gicp::LsqRegistration<pcl::PointXYZ, pcl::PointXYZ>;
using VgicpCuda = fast_gicp::FastVGICPCuda<pcl::PointXYZ, pcl::PointXYZ>;
using NdtCuda = fast_gicp::NDTCuda<pcl::PointXYZ, pcl::PointXYZ>;
using ArrD = py::array_t<double, py::array::c_style | py::array::forcecast>;
using ArrF = py::array_t<float, py::array::c_style | py::array::forcecast>;

static fast_gicp::NeighborSearchMethod search_method(const std::string& m) {  // main.cpp:21-34
  if (m == "DIRECT1") return fast_gicp::NeighborSearchMethod::DIRECT1;
  if (m == "DIRECT7") return fast_gicp::NeighborSearchMethod::DIRECT7;
  if (m == "DIRECT27") return fast_gicp::NeighborSearchMethod::DIRECT27;
  if (m == "DIRECT_RADIUS") return fast_gicp::NeighborSearchMethod::DIRECT_RADIUS;
  std::cerr << "error: unknown neighbor search method " << m << std::endl;
  return fast_gicp::NeighborSearchMethod::DIRECT1;
}

static fast_gicp::RobustKernel robust_kernel(const std::string& k) {  // vgicp_set_robust_kernel kinds
  if (k == "NONE") return fast_gicp::RobustKernel::NONE;
  if (k == "HUBER") return fast_gicp::RobustKernel::HUBER;
  if (k == "CAUCHY") return fast_gicp::RobustKernel::CAUCHY;
  if (k == "GEMAN_MCCLURE") return fast_gicp::RobustKernel::GEMAN_MCCLURE;
  throw std::invalid_argument("unknown robust kernel " + k + " (NONE, HUBER, CAUCHY or GEMAN_MCCLURE)");
}

static Cloud::Ptr eigen2pcl(const ArrD& points) {  // main.cpp:36-44 (double -> float)
  if (points.ndim() != 2 || points.shape(1) < 3) throw std::invalid_argument("points must be (N, 3)");
  auto cloud = pcl::make_shared<Cloud>();
  cloud->resize(points.shape(0));
  auto a = points.unchecked<2>();
  for (py::ssize_t i = 0; i < points.shape(0); i++) {
    cloud->at(i).x = static_cast<float>(a(i, 0));
    cloud->at(i).y = static_cast<float>(a(i, 1));
    cloud->at(i).z = static_cast<float>(a(i, 2));
  }
  return cloud;
}

// pcl::ApproximateVoxelGrid<PointXYZ> (main.cpp:46-62,81-91) on the device: include/vgicp_prep_b200.h reproduces the serial
// filter's output (points and order) bit for bit (tests/test_input_prep.py); no host implementation is kept in the product.
static vgicp_prep_handle prep_handle() {
  static vgicp_prep_handle prep = nullptr;  // one per process, device 0 like the registration objects' default
  if (!prep && vgicp_prep_create(0, &prep) != 0) throw std::runtime_error("pygicp: the input-preparation library found no usable CUDA device (sm_90a required)");
  return prep;
}

static Cloud::Ptr approximate_voxel_grid(const Cloud& in, float leaf) {
  vgicp_prep_handle prep = prep_handle();
  auto out = pcl::make_shared<Cloud>();
  const size_t n = in.points.size();
  if (n == 0) return out;
  out->points.resize(n);
  size_t m = 0;
  static_assert(sizeof(pcl::PointXYZ) % 4 == 0, "point stride");
  std::vector<float> packed(3 * n);
  const int rc = vgicp_prep_approximate_voxel_grid(prep, &in.points[0].x, n, sizeof(pcl::PointXYZ), 0, leaf, 0, packed.data(), n, 0, &m);
  if (rc != 0) throw std::runtime_error(std::string("pygicp.downsample: ") + vgicp_prep_last_error(prep));
  out->points.resize(m);
  for (size_t i = 0; i < m; i++) out->points[i] = pcl::PointXYZ(packed[3 * i], packed[3 * i + 1], packed[3 * i + 2]);
  return out;
}

static ArrD downsample(const ArrD& points, double resolution) {  // main.cpp:46-62
  auto filtered = approximate_voxel_grid(*eigen2pcl(points), static_cast<float>(resolution));
  ArrD out({static_cast<py::ssize_t>(filtered->size()), static_cast<py::ssize_t>(3)});
  auto o = out.mutable_unchecked<2>();
  for (size_t i = 0; i < filtered->size(); i++) { o(i, 0) = filtered->at(i).x; o(i, 1) = filtered->at(i).y; o(i, 2) = filtered->at(i).z; }
  return out;
}

// the same filter on (n, k) float32 records, averaging the given columns (e.g. time, intensity) per voxel next to x y z
// (pcl::ApproximateVoxelGrid<PointT>'s default) -> (m, 3 + F) float32: x y z, then the fields in the order given
static ArrF downsample_fields(const ArrF& points, double resolution, const std::vector<int>& field_columns) {
  if (points.ndim() != 2 || points.shape(1) < 3) throw std::invalid_argument("points must be (N, K >= 3)");
  const size_t n = static_cast<size_t>(points.shape(0)), k = static_cast<size_t>(points.shape(1)), F = field_columns.size();
  std::vector<size_t> offsets;
  for (int c : field_columns) {
    if (c < 3 || static_cast<size_t>(c) >= k) throw std::invalid_argument("field columns must lie in 3 ... K-1");
    offsets.push_back(static_cast<size_t>(c) * sizeof(float));
  }
  std::vector<float> records(n * (3 + F));
  size_t m = 0;
  vgicp_prep_handle prep = prep_handle();
  const int rc = vgicp_prep_approximate_voxel_grid_fields(prep, points.data(), n, k * sizeof(float), 0, static_cast<float>(resolution), 0, offsets.data(),
                                                          static_cast<int>(F), records.data(), n, 0, &m);
  if (rc != 0) throw std::runtime_error(std::string("pygicp.downsample_fields: ") + vgicp_prep_last_error(prep));
  ArrF out({static_cast<py::ssize_t>(m), static_cast<py::ssize_t>(3 + F)});
  if (m > 0) std::memcpy(out.mutable_data(), records.data(), m * (3 + F) * sizeof(float));
  return out;
}

// pcl::VoxelGrid, the exact grid (vgicp_prep_voxel_grid), on (n, k) float32 records: one centroid per occupied voxel in ascending
// voxel index, averaging x y z and the given columns -> (m, 3 + F) float32
static ArrF voxel_grid(const ArrF& points, double resolution, const std::vector<int>& field_columns, unsigned min_points_per_voxel) {
  if (points.ndim() != 2 || points.shape(1) < 3) throw std::invalid_argument("points must be (N, K >= 3)");
  const size_t n = static_cast<size_t>(points.shape(0)), k = static_cast<size_t>(points.shape(1)), F = field_columns.size();
  std::vector<size_t> offsets;
  for (int c : field_columns) {
    if (c < 3 || static_cast<size_t>(c) >= k) throw std::invalid_argument("field columns must lie in 3 ... K-1");
    offsets.push_back(static_cast<size_t>(c) * sizeof(float));
  }
  std::vector<float> records(n * (3 + F));
  size_t m = 0;
  vgicp_prep_handle prep = prep_handle();
  const int rc = vgicp_prep_voxel_grid(prep, points.data(), n, k * sizeof(float), 0, static_cast<float>(resolution), 0, offsets.data(), static_cast<int>(F),
                                       min_points_per_voxel, records.data(), n, 0, &m);
  if (rc != 0) throw std::runtime_error(std::string("pygicp.voxel_grid: ") + vgicp_prep_last_error(prep));
  ArrF out({static_cast<py::ssize_t>(m), static_cast<py::ssize_t>(3 + F)});
  if (m > 0) std::memcpy(out.mutable_data(), records.data(), m * (3 + F) * sizeof(float));
  return out;
}

static Eigen::Matrix4f to_mat4f(const ArrF& m) {
  if (m.ndim() != 2 || m.shape(0) != 4 || m.shape(1) != 4) throw std::invalid_argument("initial_guess must be 4x4");
  Eigen::Matrix4f T;
  auto a = m.unchecked<2>();
  for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) T(r, c) = a(r, c);
  return T;
}
static vgicp_carve_params carve_defaults() {
  vgicp_carve_params P;
  vgicp_carve_default_params(&P);
  return P;
}
template <typename S, int N>
static py::array_t<S> to_numpy(const Eigen::Matrix<S, N, N>& M) {
  py::array_t<S> out({N, N});
  auto o = out.template mutable_unchecked<2>();
  for (int r = 0; r < N; r++) for (int c = 0; c < N; c++) o(r, c) = M(r, c);
  return out;
}
static ArrD filled(py::ssize_t n, double v) {
  ArrD a(n);
  for (py::ssize_t i = 0; i < n; i++) a.mutable_at(i) = v;
  return a;
}
static ArrF identity4f() {
  ArrF m({4, 4});
  auto o = m.mutable_unchecked<2>();
  for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) o(r, c) = r == c ? 1.0f : 0.0f;
  return m;
}

static py::array_t<double> align_points(const ArrD& target, const ArrD& source, const std::string& method, double downsample_resolution, int k_correspondences,
                                        double max_correspondence_distance, double voxel_resolution, int num_threads, const std::string& neighbor_search_method,
                                        double neighbor_search_radius, const ArrF& initial_guess) {  // main.cpp:64-142
  (void)max_correspondence_distance; (void)num_threads;
  Cloud::Ptr target_cloud = eigen2pcl(target), source_cloud = eigen2pcl(source);
  if (downsample_resolution > 0.0) {
    target_cloud = approximate_voxel_grid(*target_cloud, static_cast<float>(downsample_resolution));
    source_cloud = approximate_voxel_grid(*source_cloud, static_cast<float>(downsample_resolution));
  }
  if (method == "NDT_CUDA") {  // main.cpp:125-133
    NdtCuda ndt;
    ndt.setResolution(voxel_resolution);
    ndt.setNeighborSearchMethod(search_method(neighbor_search_method), neighbor_search_radius);
    ndt.setInputTarget(target_cloud);
    ndt.setInputSource(source_cloud);
    Cloud aligned;
    {
      py::gil_scoped_release release;
      ndt.align(aligned, to_mat4f(initial_guess));
    }
    return to_numpy(ndt.getFinalTransformation().cast<double>());
  }
  if (method != "VGICP_CUDA") {
    if (method == "GICP" || method == "VGICP")
      std::cerr << "error: this build provides only VGICP_CUDA and NDT_CUDA (the GPU paths); " << method << " is outside it" << std::endl;
    else
      std::cerr << "error: unknown registration method " << method << std::endl;
    return to_numpy(Eigen::Matrix4d::Identity());
  }
  VgicpCuda vgicp;
  vgicp.setCorrespondenceRandomness(k_correspondences);
  vgicp.setNeighborSearchMethod(search_method(neighbor_search_method), neighbor_search_radius);
  vgicp.setResolution(voxel_resolution);
  vgicp.setInputTarget(target_cloud);
  vgicp.setInputSource(source_cloud);
  Cloud aligned;
  {
    py::gil_scoped_release release;  // (the reference holds the GIL throughout)
    vgicp.align(aligned, to_mat4f(initial_guess));
  }
  return to_numpy(vgicp.getFinalTransformation().cast<double>());
}

PYBIND11_MODULE(pygicp, m) {
  m.def("downsample", &downsample, "downsample points");
  m.def("downsample_fields", &downsample_fields, "downsample (N, K) float32 records, averaging the field columns per voxel", py::arg("points"), py::arg("resolution"),
        py::arg("field_columns"));
  m.def("voxel_grid", &voxel_grid, "pcl::VoxelGrid of (N, K) float32 records: per-voxel centroids of x y z and the field columns, in voxel index order",
        py::arg("points"), py::arg("resolution"), py::arg("field_columns") = std::vector<int>(), py::arg("min_points_per_voxel") = 0u);
  m.def("align_points", &align_points, "align two point sets", py::arg("target"), py::arg("source"), py::arg("method") = "GICP", py::arg("downsample_resolution") = -1.0,
        py::arg("k_correspondences") = 15, py::arg("max_correspondence_distance") = std::numeric_limits<double>::max(), py::arg("voxel_resolution") = 1.0,
        py::arg("num_threads") = 0, py::arg("neighbor_search_method") = "DIRECT1", py::arg("neighbor_search_radius") = 1.5, py::arg("initial_guess") = identity4f());

  py::class_<LsqReg, std::shared_ptr<LsqReg>>(m, "LsqRegistration")
    .def("set_input_target", [](LsqReg& reg, const ArrD& points) { reg.setInputTarget(eigen2pcl(points)); })
    .def("set_input_source", [](LsqReg& reg, const ArrD& points) { reg.setInputSource(eigen2pcl(points)); })
    .def("swap_source_and_target", &LsqReg::swapSourceAndTarget)
    .def("get_final_hessian", [](LsqReg& reg) { return to_numpy(reg.getFinalHessian()); })
    .def("get_final_transformation", [](LsqReg& reg) { return to_numpy(reg.getFinalTransformation()); })
    .def("has_converged", &LsqReg::hasConverged)
    .def("align",
         [](LsqReg& reg, const ArrF& initial_guess) {
           Cloud aligned;
           Eigen::Matrix4f guess = to_mat4f(initial_guess);
           {
             py::gil_scoped_release release;
             reg.align(aligned, guess);
           }
           return to_numpy(reg.getFinalTransformation());
         },
         py::arg("initial_guess") = identity4f())
    // multi-hypothesis alignment (not in the reference binding): (B,4,4) guesses -> (T (B,4,4) float32, converged (B,) bool)
    .def("align_multi",
         [](LsqReg& reg, const ArrF& initial_guesses) {
           if (initial_guesses.ndim() != 3 || initial_guesses.shape(1) != 4 || initial_guesses.shape(2) != 4) throw std::invalid_argument("initial_guesses must be (B, 4, 4)");
           const py::ssize_t B = initial_guesses.shape(0);
           auto a = initial_guesses.unchecked<3>();
           std::vector<Eigen::Matrix4f> guesses(B), T;
           for (py::ssize_t i = 0; i < B; i++)
             for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) guesses[i](r, c) = a(i, r, c);
           std::vector<bool> converged;
           {
             py::gil_scoped_release release;
             reg.alignMulti(guesses, T, converged);
           }
           const py::ssize_t n = static_cast<py::ssize_t>(T.size());
           py::array_t<float> T_out({n, static_cast<py::ssize_t>(4), static_cast<py::ssize_t>(4)});
           py::array_t<bool> conv_out(n);
           auto t = T_out.mutable_unchecked<3>();
           auto cv = conv_out.mutable_unchecked<1>();
           for (py::ssize_t i = 0; i < n; i++) {
             for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) t(i, r, c) = T[i](r, c);
             cv(i) = converged[i];
           }
           return py::make_tuple(T_out, conv_out);
         },
         py::arg("initial_guesses"))
    // (B,4,4) poses scored in one launch -> (err (B,), n_corr (B,) int64)
    .def("evaluate_poses",
         [](LsqReg& reg, const ArrD& poses) {
           if (poses.ndim() != 3 || poses.shape(1) != 4 || poses.shape(2) != 4) throw std::invalid_argument("poses must be (B, 4, 4)");
           const py::ssize_t B = poses.shape(0);
           auto a = poses.unchecked<3>();
           std::vector<Eigen::Matrix4d> P(B);
           for (py::ssize_t i = 0; i < B; i++)
             for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) P[i](r, c) = a(i, r, c);
           std::vector<double> err;
           std::vector<int64_t> n_corr;
           {
             py::gil_scoped_release release;
             reg.evaluatePoses(P, err, n_corr);
           }
           const py::ssize_t n = static_cast<py::ssize_t>(err.size());
           py::array_t<double> err_out(n);
           py::array_t<int64_t> corr_out(n);
           for (py::ssize_t i = 0; i < n; i++) {
             err_out.mutable_at(i) = err[i];
             corr_out.mutable_at(i) = n_corr[i];
           }
           return py::make_tuple(err_out, corr_out);
         },
         py::arg("poses"));

  py::class_<VgicpCuda, LsqReg, std::shared_ptr<VgicpCuda>>(m, "FastVGICPCuda")
    .def(py::init([]() { return std::make_shared<VgicpCuda>(0); }))
    .def(py::init([](int device) { return std::make_shared<VgicpCuda>(device); }), py::arg("device"))
    .def("set_resolution", &VgicpCuda::setResolution)
    .def("set_neighbor_search_method", [](VgicpCuda& v, const std::string& method, double radius) { v.setNeighborSearchMethod(search_method(method), radius); },
         py::arg("method") = "DIRECT1", py::arg("radius") = 1.5)
    .def("set_correspondence_randomness", &VgicpCuda::setCorrespondenceRandomness)
    .def("set_robust_kernel", [](VgicpCuda& v, const std::string& kind, double scale) { v.setRobustKernel(robust_kernel(kind), scale); }, py::arg("kind") = "NONE",
         py::arg("scale") = 1.0)
    // local map for scan-to-map odometry (not in the reference binding)
    .def("append_source_to_target", [](VgicpCuda& v, const ArrF& T) { v.appendSourceToTarget(to_mat4f(T)); }, py::arg("T"))
    .def("crop_target",
         [](VgicpCuda& v, const ArrD& center, double radius, size_t max_points) {
           if (center.size() != 3) throw std::invalid_argument("center must have 3 elements");
           v.cropTarget(center.data(), radius, max_points);
         },
         py::arg("center"), py::arg("radius"), py::arg("max_points") = 0)
    .def("thin_target", &VgicpCuda::thinTarget, py::arg("leaf_size"), py::arg("max_points_per_voxel"))
    .def("carve_target",
         [](VgicpCuda& v, const ArrF& T, int width, int height, double elevation_min, double elevation_max, int window, double margin, double margin_rel) {
           const vgicp_carve_params P{width, height, elevation_min, elevation_max, window, margin, margin_rel};
           return v.carveTarget(to_mat4f(T), &P);
         },
         py::arg("T"), py::arg("width") = carve_defaults().width, py::arg("height") = carve_defaults().height,
         py::arg("elevation_min") = carve_defaults().elevation_min, py::arg("elevation_max") = carve_defaults().elevation_max,
         py::arg("window") = carve_defaults().window, py::arg("margin") = carve_defaults().margin, py::arg("margin_rel") = carve_defaults().margin_rel)
    // motion compensation (not in the reference binding): one relative timestamp per source point, twist = [omega, v]
    .def("deskew_source",
         [](VgicpCuda& v, const ArrF& times, const ArrD& twist, double t_ref) {
           if (twist.size() != 6) throw std::invalid_argument("twist must have 6 elements");
           v.deskewSource(times.data(), static_cast<size_t>(times.size()), sizeof(float), twist.data(), t_ref);
         },
         py::arg("times"), py::arg("twist"), py::arg("t_ref") = 0.0)
    // the same with the timestamps and t_ref stored by set_source_timestamps (no upload)
    .def("deskew_source_stored",
         [](VgicpCuda& v, const ArrD& twist) {
           if (twist.size() != 6) throw std::invalid_argument("twist must have 6 elements");
           v.deskewSourceStored(twist.data());
         },
         py::arg("twist"))
    // continuous-time registration (not in the reference binding): pose at t_ref and the sweep's twist together
    .def("set_source_timestamps",
         [](VgicpCuda& v, const ArrF& times, double t_ref) { v.setSourceTimestamps(times.data(), static_cast<size_t>(times.size()), sizeof(float), t_ref); },
         py::arg("times"), py::arg("t_ref") = 0.0)
    // -> dict: T (4x4, the float transformation as double, like align), twist (6), H (12x12, double), and the counters.
    // twist_prior None: the twist guess; twist_weight: 6 weights > 0 (a scalar applies to all)
    .def("align_ct",
         [](VgicpCuda& v, const ArrF& initial_guess, const ArrD& twist_guess, py::object twist_prior, const ArrD& twist_weight) {
           if (twist_guess.size() != 6) throw std::invalid_argument("twist_guess must have 6 elements");
           std::array<double, 6> tg, tp, tw;
           for (int j = 0; j < 6; j++) tg[j] = twist_guess.data()[j];
           tp = tg;
           if (!twist_prior.is_none()) {
             ArrD p = twist_prior.cast<ArrD>();
             if (p.size() != 6) throw std::invalid_argument("twist_prior must have 6 elements");
             for (int j = 0; j < 6; j++) tp[j] = p.data()[j];
           }
           if (twist_weight.size() != 6 && twist_weight.size() != 1) throw std::invalid_argument("twist_weight must have 6 elements or one");
           for (int j = 0; j < 6; j++) tw[j] = twist_weight.data()[twist_weight.size() == 6 ? j : 0];
           const Eigen::Matrix4f guess = to_mat4f(initial_guess);
           vgicp_align_ct_result r;
           {
             py::gil_scoped_release release;
             v.alignCT(guess, tg.data(), tp.data(), tw.data(), &r);
           }
           py::array_t<double> twist(6), H({12, 12});
           auto h = H.mutable_unchecked<2>();
           for (int j = 0; j < 6; j++) twist.mutable_at(j) = r.twist[j];
           for (int row = 0; row < 12; row++) for (int c = 0; c < 12; c++) h(row, c) = r.H[c * 12 + row];
           py::dict out;
           out["T"] = to_numpy(v.getFinalTransformation().cast<double>());
           out["twist"] = twist;
           out["H"] = H;
           out["nr_iterations"] = r.nr_iterations;
           out["converged"] = r.converged != 0;
           out["n_linearize"] = r.n_linearize;
           out["n_compute_error"] = r.n_compute_error;
           out["lm_failed"] = r.lm_failed != 0;
           return out;
         },
         py::arg("initial_guess") = identity4f(), py::arg("twist_guess") = filled(6, 0.0), py::arg("twist_prior") = py::none(),
         py::arg("twist_weight") = filled(1, 1e-6))
    // multi-source alignment (not in the reference binding): B (N_i, 3) sources against the current target, (B,4,4) guesses or None
    // -> (T (B,4,4) float32, converged (B,) bool)
    .def("align_sources",
         [](VgicpCuda& v, const std::vector<ArrD>& sources, py::object initial_guesses) {
           std::vector<VgicpCuda::PointCloudSourceConstPtr> clouds;
           for (const ArrD& s : sources) clouds.push_back(eigen2pcl(s));
           std::vector<Eigen::Matrix4f> guesses, T;
           if (!initial_guesses.is_none()) {
             ArrF g = initial_guesses.cast<ArrF>();
             if (g.ndim() != 3 || g.shape(1) != 4 || g.shape(2) != 4) throw std::invalid_argument("initial_guesses must be (B, 4, 4)");
             auto a = g.unchecked<3>();
             guesses.resize(g.shape(0));
             for (py::ssize_t i = 0; i < g.shape(0); i++)
               for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) guesses[i](r, c) = a(i, r, c);
           }
           std::vector<bool> converged;
           {
             py::gil_scoped_release release;
             v.alignSources(clouds, guesses, T, converged);
           }
           const py::ssize_t n = static_cast<py::ssize_t>(T.size());
           py::array_t<float> T_out({n, static_cast<py::ssize_t>(4), static_cast<py::ssize_t>(4)});
           py::array_t<bool> conv_out(n);
           auto t = T_out.mutable_unchecked<3>();
           auto cv = conv_out.mutable_unchecked<1>();
           for (py::ssize_t i = 0; i < n; i++) {
             for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) t(i, r, c) = T[i](r, c);
             cv(i) = converged[i];
           }
           return py::make_tuple(T_out, conv_out);
         },
         py::arg("sources"), py::arg("initial_guesses") = py::none())
    .def("get_fitness_score",
         [](VgicpCuda& v, double max_range) {
           double T[16], score = 0.0;
           Eigen::Matrix4f F = v.getFinalTransformation();
           for (int i = 0; i < 16; i++) T[i] = F.v[i];
           if (vgicp_get_fitness_score(v.handle(), T, max_range, &score) != VGICP_OK) throw std::runtime_error(vgicp_last_error(v.handle()));
           return score;
         },
         py::arg("max_range") = std::numeric_limits<double>::max());

  py::class_<NdtCuda, LsqReg, std::shared_ptr<NdtCuda>>(m, "NDTCuda")  // main.cpp:204-212
    .def(py::init([]() { return std::make_shared<NdtCuda>(0); }))
    .def("set_neighbor_search_method", [](NdtCuda& v, const std::string& method, double radius) { v.setNeighborSearchMethod(search_method(method), radius); },
         py::arg("method") = "DIRECT1", py::arg("radius") = 1.5)
    .def("set_resolution", &NdtCuda::setResolution)
    .def("set_distance_mode", [](NdtCuda& v, const std::string& mode) { v.setDistanceMode(mode == "P2D" ? fast_gicp::NDTDistanceMode::P2D : fast_gicp::NDTDistanceMode::D2D); });

  m.attr("__version__") = "b200-dev";
}
