"""The checker of initial_guess_search: the same level data and the same search driver, with every score from the CPU
oracle's CostCalculatorNID::calculate (oracle.nid_calculate) instead of the GPU sweep.  Toy sizes only: it scores one
pose at a time."""
import numpy as np

from direct_visual_lidar_calibration_b200 import initial_guess as ig


class OracleScorer:
    """score(level, search_set) -> (scores, inliers, 0.0): sum over the bags, in bag order, of the oracle's NID of every pose
    and of its histogram's total."""

    def __init__(self, O, camera_model, intrinsics, distortion, dataset, nid_bins=16, seed=0):
        """dataset: [(image, points_xyzw, intensities)] per bag."""
        self.O, self.camera_model, self.intrinsics, self.distortion = O, camera_model, list(intrinsics), list(distortion)
        self.dataset, self.bins, self.seed = dataset, nid_bins, seed
        self._levels = {}

    def level_data(self, level):
        key = (level["scale"], level["points"])
        if key not in self._levels:
            cam = self.O.create_camera(self.camera_model, ig.pyramid_intrinsics(self.camera_model, self.intrinsics, level["scale"]), self.distortion)
            bags = []
            for b, (image, points, intensities) in enumerate(self.dataset):
                sub = np.sort(ig.cloud_subset(points.shape[0], level["points"], self.seed + b))
                bags.append((ig.pyramid_image(image, level["scale"]), np.ascontiguousarray(points[sub]), np.ascontiguousarray(intensities[sub])))
            H, W = bags[0][0].shape
            self._levels[key] = (cam, self.O.estimate_camera_fov(cam, W, H), bags)
        return self._levels[key]

    def __call__(self, level, sset):
        cam, fov, bags = self.level_data(level)
        poses = sset.poses()
        scores, inliers = np.empty(len(poses)), np.zeros(len(poses), dtype=np.int64)
        for p, T in enumerate(poses):
            s = 0.0
            for bag in bags:
                nid, hist = self.O.nid_calculate(cam, *bag, self.bins, fov, T, omp=True)
                s = nid if len(bags) == 1 else s + nid
                inliers[p] += int(hist.sum())
            scores[p] = s
        return scores, inliers, 0.0
