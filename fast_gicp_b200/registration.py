"""Host-side mirror of the reference's registration classes for the VGICP-CUDA path, on top of the C ABI.

  LsqRegistration  <- include/fast_gicp/gicp/lsq_registration.hpp:16-85, impl/lsq_registration_impl.hpp:9-168
                      (+ the pcl::Registration surface it inherits: setInputSource/Target, align, getFinalTransformation,
                       hasConverged, getFitnessScore, setMaximumIterations, setTransformationEpsilon)
  FastVGICPCuda    <- include/fast_gicp/gicp/fast_vgicp_cuda.hpp:27-85, impl/fast_vgicp_cuda_impl.hpp:22-178

Method names follow the C++ API (camelCase) and the pygicp binding (snake_case, src/python/main.cpp:152-217).
All numerical work happens in libvgicp_b200.so on the GPU; this file is state machine + LM bookkeeping only.
"""
import enum

import numpy as np

from . import core as _core
from .core import Core, default_params


class RegularizationMethod(enum.IntEnum):  # gicp_settings.hpp:6
    NONE = 0
    MIN_EIG = 1
    NORMALIZED_MIN_EIG = 2
    PLANE = 3
    FROBENIUS = 4


class NeighborSearchMethod(enum.IntEnum):  # gicp_settings.hpp:8
    DIRECT27 = 0
    DIRECT7 = 1
    DIRECT1 = 2
    DIRECT_RADIUS = 3


class NearestNeighborMethod(enum.IntEnum):  # fast_vgicp_cuda.hpp:21
    CPU_PARALLEL_KDTREE = 0  # reference: FLANN kd-tree on the host. Here: the same exact k-NN, computed on the GPU.
    GPU_BRUTEFORCE = 1
    GPU_RBF_KERNEL = 2


class LSQ_OPTIMIZER_TYPE(enum.IntEnum):  # lsq_registration.hpp:13
    GaussNewton = 0
    LevenbergMarquardt = 1


def _as_cloud(points):
    a = np.asarray(points)
    if a.ndim != 2 or a.shape[1] < 3:
        raise ValueError("point cloud must be (N, >=3)")
    return np.ascontiguousarray(a[:, :3], dtype=np.float32)  # eigen2pcl: double -> float (main.cpp:36-44)


class LsqRegistration:
    """pcl::Registration + fast_gicp::LsqRegistration state."""

    def __init__(self):
        self.reg_name_ = "LsqRegistration"
        self.max_iterations_ = 64
        self.rotation_epsilon_ = 2e-3
        self.transformation_epsilon_ = 5e-4
        self.lsq_optimizer_type_ = LSQ_OPTIMIZER_TYPE.LevenbergMarquardt
        self.lm_debug_print_ = False
        self.lm_max_iterations_ = 10
        self.lm_init_lambda_factor_ = 1e-9
        self.final_hessian_ = np.eye(6)
        self.final_transformation_ = np.eye(4, dtype=np.float32)
        self.converged_ = False
        self.nr_iterations_ = 0
        self.input_ = None
        self.target_ = None

    # -- pcl::Registration setters used by the reference
    def setMaximumIterations(self, n):
        self.max_iterations_ = int(n)

    def setTransformationEpsilon(self, eps):
        self.transformation_epsilon_ = float(eps)

    def setRotationEpsilon(self, eps):  # lsq_registration_impl.hpp:28-30
        self.rotation_epsilon_ = float(eps)

    def setInitialLambdaFactor(self, f):  # :33-35
        self.lm_init_lambda_factor_ = float(f)

    def setDebugPrint(self, flag):  # :38-40
        self.lm_debug_print_ = bool(flag)

    def setMaxCorrespondenceDistance(self, d):  # ignored by the voxel paths (only FastGICP reads corr_dist_threshold_)
        self.corr_dist_threshold_ = float(d)

    def getFinalHessian(self):
        return self.final_hessian_

    def getFinalTransformation(self):
        return self.final_transformation_

    def hasConverged(self):
        return self.converged_

    def _params(self):
        return default_params(
            max_iterations=self.max_iterations_,
            rotation_epsilon=self.rotation_epsilon_,
            transformation_epsilon=self.transformation_epsilon_,
            use_gauss_newton=int(self.lsq_optimizer_type_ == LSQ_OPTIMIZER_TYPE.GaussNewton),
            lm_max_iterations=self.lm_max_iterations_,
            lm_init_lambda_factor=self.lm_init_lambda_factor_,
        )

    # -- multi-hypothesis alignment (not in the reference): the subclasses provide _core() and _prelude()
    def align_multi(self, initial_guesses):
        """Register the source from each of the (B, 4, 4) initial guesses, the evaluations of all hypotheses sharing launches.

        Returns (T (B, 4, 4) float32, converged (B,) bool); T[i] equals what align(initial_guesses[i]) returns.  The state of
        the single registration (getFinalTransformation, hasConverged, the final Hessian) is left alone."""
        if self.input_ is None or self.target_ is None:
            raise RuntimeError("align_multi: input source/target not set")
        G = np.asarray(initial_guesses, dtype=np.float32).astype(np.float64)  # cast like align's guess
        if G.ndim != 3 or G.shape[1:] != (4, 4):
            raise ValueError("initial_guesses must be (B, 4, 4)")
        self._prelude()
        res = self._core().align_multi(G, self._params())
        T = np.stack([_core.pose_from_c(r.T) for r in res]).astype(np.float32)
        return T, np.array([bool(r.converged) for r in res])

    def evaluate_poses(self, poses):
        """Score the (B, 4, 4) poses in one launch -> (err (B,), n_corr (B,) int64): the error of update_correspondences(T) +
        compute_error(T) and the number of (source point, voxel) correspondences at each pose.  A pose without overlap scores
        err 0 with n_corr 0, so rank hypotheses by err normalised with n_corr."""
        if self.input_ is None or self.target_ is None:
            raise RuntimeError("evaluate_poses: input source/target not set")
        self._prelude()
        err, _, _, n_corr = self._core().evaluate_poses(np.asarray(poses, dtype=np.float64))
        return err, n_corr

    # pygicp names (main.cpp:152-168)
    def set_input_target(self, points):
        self.setInputTarget(_as_cloud(points))

    def set_input_source(self, points):
        self.setInputSource(_as_cloud(points))

    def swap_source_and_target(self):
        self.swapSourceAndTarget()

    def get_final_hessian(self):
        return self.getFinalHessian()

    def get_final_transformation(self):
        return self.getFinalTransformation()

    def get_fitness_score(self, max_range=float("inf")):
        return self.getFitnessScore(max_range)


class NDTDistanceMode(enum.IntEnum):  # ndt_settings.hpp:6
    P2D = 0
    D2D = 1


class NDTCuda(LsqRegistration):
    """fast_gicp::NDTCuda (include/fast_gicp/ndt/ndt_cuda.hpp:22-71, impl/ndt_cuda_impl.hpp:11-90) on the same engine:
    voxel Gaussians from the raw points (MIN_EIG-regularised), Cauchy-weighted P2D / D2D residuals, DIRECT7 by default."""

    def __init__(self, device=0):
        super().__init__()
        self.reg_name_ = "NDTCuda"
        self.ndt_cuda_ = Core(device)
        self._mode = NDTDistanceMode.D2D  # ndt_cuda.cu:21
        self.ndt_cuda_.set_problem(2)
        self.ndt_cuda_.set_neighbor_search_method(int(NeighborSearchMethod.DIRECT7), 0.0)  # ndt_cuda.cu:22

    def setDistanceMode(self, mode):
        self._mode = NDTDistanceMode(mode)
        self.ndt_cuda_.set_problem(1 if self._mode == NDTDistanceMode.P2D else 2)

    def setResolution(self, resolution):
        self.ndt_cuda_.set_resolution(resolution)

    def setNeighborSearchMethod(self, method, radius=-1.0):
        if isinstance(method, str):
            method = NeighborSearchMethod[method]
        self.ndt_cuda_.set_neighbor_search_method(int(method), radius)

    # pygicp names (main.cpp:204-212)
    def set_resolution(self, r):
        self.setResolution(r)

    def set_neighbor_search_method(self, method="DIRECT1", radius=1.5):
        self.setNeighborSearchMethod(method, radius)

    def swapSourceAndTarget(self):
        self.ndt_cuda_.swap_source_and_target()
        self.input_, self.target_ = self.target_, self.input_

    def clearSource(self):
        self.input_ = None

    def clearTarget(self):
        self.target_ = None

    def setInputSource(self, cloud):
        if cloud is self.input_:
            return
        self.input_ = cloud
        self.ndt_cuda_.set_source_cloud(cloud)

    def setInputTarget(self, cloud):
        if cloud is self.target_:
            return
        self.target_ = cloud
        self.ndt_cuda_.set_target_cloud(cloud)

    def linearize(self, trans):
        return self.ndt_cuda_.linearize(trans)

    def compute_error(self, trans):
        return self.ndt_cuda_.compute_error(trans, want_H=False)[0]

    def _core(self):
        return self.ndt_cuda_

    def _prelude(self):
        self.ndt_cuda_.ndt_create_voxelmaps()  # computeTransformation, ndt_cuda_impl.hpp:71-73

    def align(self, initial_guess=None, aligned_out=None):
        if self.input_ is None or self.target_ is None:
            raise RuntimeError("align: input source/target not set")
        guess = np.eye(4) if initial_guess is None else np.asarray(initial_guess, dtype=np.float32).astype(np.float64)
        self._prelude()
        self.converged_ = False
        res = self.ndt_cuda_.align(guess, self._params())
        if res.lm_failed:
            print("lm not converged!!")
        self.nr_iterations_ = res.nr_iterations
        self.converged_ = bool(res.converged)
        self.final_hessian_ = np.array(res.H).reshape(6, 6).T.copy()
        self.final_transformation_ = _core.pose_from_c(res.T).astype(np.float32)
        if aligned_out is not None:
            self.ndt_cuda_.transform_source(self.final_transformation_.astype(np.float64), out=aligned_out)
        return self.final_transformation_

    def getFitnessScore(self, max_range=float("inf")):
        return self.ndt_cuda_.fitness_score(self.final_transformation_.astype(np.float64), max_range)


class FastVGICPCuda(LsqRegistration):
    """Fast Voxelized GICP on an H100 behind the reference's FastVGICPCuda interface."""

    def __init__(self, device=0):
        super().__init__()
        self.reg_name_ = "FastVGICPCuda"
        self.k_correspondences_ = 20
        self.voxel_resolution_ = 1.0
        self.regularization_method_ = RegularizationMethod.PLANE
        self.neighbor_search_method_ = NearestNeighborMethod.CPU_PARALLEL_KDTREE
        self.vgicp_cuda_ = Core(device)
        self.vgicp_cuda_.set_resolution(self.voxel_resolution_)
        self.vgicp_cuda_.set_kernel_params(0.5, 3.0)  # fast_vgicp_cuda_impl.hpp:31

    # -- setters (fast_vgicp_cuda_impl.hpp:37-66)
    def setCorrespondenceRandomness(self, k):  # empty in the reference (:38): k stays 20 on the CUDA path
        pass

    def setResolution(self, resolution):  # :41-43 writes the core only (SURVEY Q3)
        self.vgicp_cuda_.set_resolution(resolution)

    def setKernelWidth(self, kernel_width, max_dist=-1.0):  # :46-51
        if max_dist <= 0.0:
            max_dist = kernel_width * 5.0
        self.vgicp_cuda_.set_kernel_params(kernel_width, max_dist)

    def setRegularizationMethod(self, method):
        self.regularization_method_ = RegularizationMethod(method)

    def setNeighborSearchMethod(self, method, radius=-1.0):
        if isinstance(method, str):
            method = NeighborSearchMethod[method]
        self.vgicp_cuda_.set_neighbor_search_method(int(method), radius)

    def setNearestNeighborSearchMethod(self, method):
        self.neighbor_search_method_ = NearestNeighborMethod(method)

    # pygicp names (main.cpp:194-202)
    def set_resolution(self, r):
        self.setResolution(r)

    def set_neighbor_search_method(self, method="DIRECT1", radius=1.5):
        self.setNeighborSearchMethod(method, radius)

    def set_correspondence_randomness(self, k):
        self.setCorrespondenceRandomness(k)

    # -- state machine (:69-141)
    def swapSourceAndTarget(self):
        self.vgicp_cuda_.swap_source_and_target()
        self.input_, self.target_ = self.target_, self.input_

    def clearSource(self):
        self.input_ = None

    def clearTarget(self):
        self.target_ = None

    def _covariances(self, which):
        c = self.vgicp_cuda_
        m = self.neighbor_search_method_
        reg = int(self.regularization_method_)
        if m == NearestNeighborMethod.GPU_RBF_KERNEL:
            (c.calculate_source_covariances_rbf if which == "source" else c.calculate_target_covariances_rbf)(reg)
        else:  # CPU_PARALLEL_KDTREE and GPU_BRUTEFORCE give the same neighbour sets; both run on the GPU here
            (c.find_source_neighbors if which == "source" else c.find_target_neighbors)(self.k_correspondences_)
            (c.calculate_source_covariances if which == "source" else c.calculate_target_covariances)(reg)

    def setInputSource(self, cloud):
        if cloud is self.input_:  # pointer-equality early out (:87-89)
            return
        self.input_ = cloud
        self.vgicp_cuda_.set_source_cloud(cloud)
        self._covariances("source")

    def setInputTarget(self, cloud):
        if cloud is self.target_:  # (:116-118)
            return
        self.target_ = cloud
        self.vgicp_cuda_.set_target_cloud(cloud)
        self._covariances("target")
        self.vgicp_cuda_.create_target_voxelmap()

    # -- LsqRegistration virtuals (:170-178)
    def linearize(self, trans):
        return self.vgicp_cuda_.linearize(trans)

    def compute_error(self, trans):
        return self.vgicp_cuda_.compute_error(trans, want_H=False)[0]

    def evaluateCost(self, relative_pose, want_H=False):  # lsq_registration_impl.hpp:48-50
        err, H, b = self.vgicp_cuda_.linearize(np.asarray(relative_pose, dtype=np.float32).astype(np.float64))
        return (err, H, b) if want_H else err

    def _core(self):
        return self.vgicp_cuda_

    def _prelude(self):
        self.vgicp_cuda_.set_resolution(self.voxel_resolution_)  # :145 (the wrapper's stale resolution, SURVEY Q3)

    def align(self, initial_guess=None, return_aligned=False, aligned_out=None):
        """pcl::Registration::align -> computeTransformation (:144-148 + lsq_registration_impl.hpp:53-79).

        Returns the final 4x4 float transformation (pygicp's align).  The C++ align(output, guess) also fills `output`
        with the transformed source (pcl::transformPointCloud, lsq_registration_impl.hpp:78): pass `aligned_out`
        ((N,3) float32, written in place) or `return_aligned=True` to get it.
        """
        if self.input_ is None or self.target_ is None:
            raise RuntimeError("align: input source/target not set")
        guess = np.eye(4) if initial_guess is None else np.asarray(initial_guess, dtype=np.float32).astype(np.float64)
        self._prelude()
        self.converged_ = False
        res = self.vgicp_cuda_.align(guess, self._params())
        if res.lm_failed:
            print("lm not converged!!")
        self.nr_iterations_ = res.nr_iterations
        self.converged_ = bool(res.converged)
        self.final_hessian_ = np.array(res.H).reshape(6, 6).T.copy()
        self.final_transformation_ = _core.pose_from_c(res.T).astype(np.float32)
        if aligned_out is not None:
            self.vgicp_cuda_.transform_source(self.final_transformation_.astype(np.float64), out=aligned_out)
        if return_aligned:
            return self.final_transformation_, self.vgicp_cuda_.transform_source(self.final_transformation_.astype(np.float64))[:, :3]
        return self.final_transformation_

    def getFitnessScore(self, max_range=float("inf")):
        """pcl::Registration::getFitnessScore: mean squared nearest-neighbour distance of the aligned source to the target."""
        return self.vgicp_cuda_.fitness_score(self.final_transformation_.astype(np.float64), max_range)
