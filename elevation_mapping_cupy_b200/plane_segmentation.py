"""Parameters of ElevationMap.segment_planes, extract_planar_regions and planar_terrain: the plane decomposition node's
`preprocessing`, `sliding_window_plane_extractor`, `contour_extraction` and `postprocessing` sections
(convex_plane_decomposition_ros/config/parameters.yaml), with the two inclination thresholds as cosines, as
ParameterLoading.cpp stores them."""
import math
from dataclasses import dataclass

from . import _lib


@dataclass
class PlaneSegmentationParams:
    # preprocessing
    median_kernel: int = 3
    median_repeats: int = 1
    resolution: float = 0.04           # resampled by plane_decomposition; the window calls take <= 0 or the map's
    # sliding_window_plane_extractor
    kernel_size: int = 3
    planarity_opening_filter: int = 0
    plane_inclination_cos: float = math.cos(math.radians(30.0))
    local_plane_inclination_cos: float = math.cos(math.radians(35.0))
    plane_patch_error_threshold: float = 0.02
    min_number_points_per_label: int = 4
    connectivity: int = 4
    include_ransac_refinement: bool = False
    # contour_extraction and postprocessing (extract_planar_regions only)
    margin_size: int = 1
    extracted_planes_height_offset: float = 0.0
    # postprocessing (planar_terrain only)
    nonplanar_height_offset: float = 0.02
    nonplanar_horizontal_offset: int = 1
    smoothing_dilation_size: float = 0.2
    smoothing_box_kernel_size: float = 0.1
    smoothing_gauss_kernel_size: float = 0.05

    @classmethod
    def from_yaml(cls, path):
        """Reads the `preprocessing`, `sliding_window_plane_extractor`, `contour_extraction` (marginSize) and
        `postprocessing` sections of a node parameter file; keys that are absent keep their defaults, and `*_degrees`
        become cosines (ParameterLoading.cpp:49-59)."""
        import yaml
        with open(path) as f:
            doc = yaml.safe_load(f) or {}
        pre = doc.get("preprocessing") or {}
        sw = doc.get("sliding_window_plane_extractor") or {}
        p = cls()
        for key, name in (("kernelSize", "median_kernel"), ("numberOfRepeats", "median_repeats"),
                          ("resolution", "resolution")):
            if key in pre:
                setattr(p, name, pre[key])
        for key, name in (("kernel_size", "kernel_size"), ("planarity_opening_filter", "planarity_opening_filter"),
                          ("plane_patch_error_threshold", "plane_patch_error_threshold"),
                          ("min_number_points_per_label", "min_number_points_per_label"),
                          ("connectivity", "connectivity"), ("include_ransac_refinement", "include_ransac_refinement")):
            if key in sw:
                setattr(p, name, sw[key])
        if "marginSize" in (doc.get("contour_extraction") or {}):
            p.margin_size = doc["contour_extraction"]["marginSize"]
        post = doc.get("postprocessing") or {}
        for key in ("extracted_planes_height_offset", "nonplanar_height_offset", "nonplanar_horizontal_offset",
                    "smoothing_dilation_size", "smoothing_box_kernel_size", "smoothing_gauss_kernel_size"):
            if key in post:
                setattr(p, key, post[key])
        if "plane_inclination_threshold_degrees" in sw:
            p.plane_inclination_cos = math.cos(sw["plane_inclination_threshold_degrees"] * math.pi / 180.0)
        if "local_plane_inclination_threshold_degrees" in sw:
            p.local_plane_inclination_cos = math.cos(sw["local_plane_inclination_threshold_degrees"] * math.pi / 180.0)
        return p

    def to_c(self):
        return _lib.EmapPlaneParams(int(self.median_kernel), int(self.median_repeats), float(self.resolution),
                                    int(self.kernel_size), int(self.planarity_opening_filter),
                                    int(self.min_number_points_per_label), int(self.connectivity),
                                    float(self.plane_inclination_cos), float(self.local_plane_inclination_cos),
                                    float(self.plane_patch_error_threshold), int(bool(self.include_ransac_refinement)))

    def regions_to_c(self):
        return _lib.EmapRegionParams(int(self.margin_size), float(self.extracted_planes_height_offset))

    def postprocess_to_c(self):
        return _lib.EmapPostprocessParams(float(self.nonplanar_height_offset), int(self.nonplanar_horizontal_offset),
                                          float(self.smoothing_dilation_size), float(self.smoothing_box_kernel_size),
                                          float(self.smoothing_gauss_kernel_size))
