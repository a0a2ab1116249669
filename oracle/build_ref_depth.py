"""oracle/build_ref_depth.py -- TEST INFRASTRUCTURE ONLY.

Runs the semantic sensor node's own depth-image -> cloud step, from where it lies under /root/reference
(sensor_processing/semantic_sensor/script/semantic_sensor/pointcloud_node.py: create_pcl_from_image, get_coordinates,
process_image, perform_segmentation), unmodified, on the host.  Nothing is copied into the repository: the module is
imported from the reference tree with stub modules in place of its imports:

  * `cupy` backed by NumPy: arrays are an `ndarray` subclass with `.get()`, `nonzero` returns such arrays;
  * `rospy`, `ros_numpy`, `cv_bridge`, `sensor_msgs`, `message_filters`, `skimage`, `matplotlib`, `sklearn` and the
    package's `pointcloud_parameters` / `networks` / `utils`: empty modules with the names the node imports.

The node's methods are then called on a stub `self` that carries P, `param.channels` / `param.fusion` /
`param.confidence_threshold`, the structured dtype and, for feature channels, a segmentation "model" that returns the
caller's feature planes (the node reads `prediction[:, v, u]` into its `actual_channels`).

Used by tests/golden/make_depth_golden.py; needs the reference tree.  One link is not checked here: CuPy is not
installed, so the node's `u.astype(float32) - P[0, 2]` is promoted as NumPy 2 promotes it (NEP 50: to float64).
"""
import os
import sys
import types

import numpy as np

NODE_DIR = "/root/reference/sensor_processing/semantic_sensor/script/semantic_sensor"

_node = None


class _DevArray(np.ndarray):
    def get(self):
        return np.asarray(self)


def _wrap(x):
    return np.asarray(x).view(_DevArray)


def node_module():
    """pointcloud_node imported from the reference tree with the stub modules."""
    global _node
    if _node is not None:
        return _node
    if not os.path.isdir(NODE_DIR):
        raise FileNotFoundError(f"{NODE_DIR} is missing: the depth golden needs the reference tree")
    cp = types.ModuleType("cupy")
    for name in ("where", "rint", "maximum", "isfinite", "ones", "zeros", "argmax", "resize", "uint8", "float32"):
        setattr(cp, name, getattr(np, name))
    cp.asarray = _wrap
    cp.asnumpy = np.asarray
    cp.nonzero = lambda x: tuple(_wrap(a) for a in np.nonzero(x))
    stubs = {"cupy": cp}
    for m in ("rospy", "ros_numpy", "matplotlib", "matplotlib.pyplot", "skimage", "skimage.io", "message_filters",
              "sensor_msgs", "sensor_msgs.msg", "cv_bridge", "semantic_sensor", "semantic_sensor.pointcloud_parameters",
              "semantic_sensor.networks", "semantic_sensor.utils", "sklearn", "sklearn.decomposition"):
        stubs[m] = types.ModuleType(m)
    stubs["skimage.io"].imshow = None
    for n in ("Image", "CameraInfo", "PointCloud2"):
        setattr(stubs["sensor_msgs.msg"], n, object)
    stubs["cv_bridge"].CvBridge = object
    stubs["semantic_sensor.pointcloud_parameters"].PointcloudParameter = object
    stubs["semantic_sensor.networks"].resolve_model = None
    stubs["semantic_sensor.utils"].decode_max = None
    stubs["sklearn.decomposition"].PCA = None
    before = {m: sys.modules.get(m) for m in stubs}
    sys.modules.update(stubs)
    sys.path.insert(0, NODE_DIR)
    try:
        import pointcloud_node as PN
    finally:
        sys.path.remove(NODE_DIR)
        for m, old in before.items():          # the stubs do not leak into the importer's process
            if old is None:
                sys.modules.pop(m, None)
            else:
                sys.modules[m] = old
    _node = PN
    return PN


class _Model:
    def __init__(self, planes, names):
        self.planes, self.actual_channels = planes, names

    def __call__(self, image):
        return _wrap(self.planes)


def node_cloud(depth, P, channels=(), fusion=(), rgb=None, features=None, confidence=None, confidence_threshold=10.0):
    """The node's structured cloud (x, y, z, *channels, all float32) of one depth image.  Channel j fuses with fusion[j];
    the `color` channel reads rgb, the others are the node's segmentation channels and read the planes of `features` in
    order."""
    PN = node_module()
    Node = PN.PointcloudNode
    s = types.SimpleNamespace()
    s.P = _wrap(np.asarray(P, np.float64))
    s.param = types.SimpleNamespace(channels=list(channels), fusion=list(fusion), confidence_threshold=confidence_threshold,
                                    publish_segmentation_image=False, semantic_segmentation=False)
    seg = [c for c, f in zip(channels, fusion) if f != "color"]
    s.segmentation_channels = seg or None
    s.semantic_model = {"model": _Model(features, seg)} if seg else None
    s.feature_channels = None
    s.dtype = [(n, np.float32) for n in ["x", "y", "z", *channels]]
    s.get_coordinates = lambda d, c: Node.get_coordinates(s, d, c)
    s.process_image = lambda i, u, v, p: Node.process_image(s, i, u, v, p)
    s.perform_segmentation = lambda i, p, u, v: Node.perform_segmentation(s, i, p, u, v)
    image = _wrap(rgb) if rgb is not None else None
    conf = _wrap(confidence) if confidence is not None else None
    return Node.create_pcl_from_image(s, image, _wrap(depth), conf)
