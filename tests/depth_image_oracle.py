"""The semantic sensor node's depth-image -> cloud step (pointcloud_node.py create_pcl_from_image, get_coordinates,
process_image) restated in NumPy, as include/emap.h defines it for emap_input_depth_images (steps 1-4): the cloud a
depth frame must fuse bit for bit like emap_input_sensors.  tests/test_depth_image_cpu.py pins it against the node's
own code run on the golden images (tests/golden/depth_image_core.npz)."""
import numpy as np


def keep_mask(depth, confidence=None, confidence_threshold=10.0, max_depth=8.0):
    """isfinite(d) && d > 0 && d < max_depth && (no confidence || q >= fp32(threshold)), compared in fp32."""
    d = np.asarray(depth, np.float32)
    with np.errstate(invalid="ignore"):
        m = np.isfinite(d) & (d > 0) & (d < np.float32(max_depth))
        if confidence is not None:
            m &= np.asarray(confidence, np.float32) >= np.float32(confidence_threshold)
    return m


def pack_rgb(rgb):
    """(r << 16) | (g << 8) | b of (..., 3) uint8, as float32 bits."""
    c = np.asarray(rgb, np.uint8).astype(np.uint32)
    return ((c[..., 0] << 16) | (c[..., 1] << 8) | c[..., 2]).view(np.float32)


def depth_cloud(depth, P, sources=(), rgb=None, features=None, confidence=None, confidence_threshold=10.0, max_depth=8.0):
    """(cloud (n_kept, 3 + len(sources)) float32, kept (H*W,) bool) of one camera.  sources[j]: -1 colour, k feature
    plane k.  x = fp32(((double)u - cx) * (double)d / fx), y likewise, z = d; rows in row-major pixel order."""
    P = np.asarray(P, np.float64)
    m = keep_mask(depth, confidence, confidence_threshold, max_depth)
    v, u = np.nonzero(m)
    d = np.asarray(depth, np.float32)[v, u].astype(np.float64)
    x = (((u.astype(np.float64) - P[0, 2]) * d) / P[0, 0]).astype(np.float32)
    y = (((v.astype(np.float64) - P[1, 2]) * d) / P[1, 1]).astype(np.float32)
    cols = [x, y, d.astype(np.float32)]
    for s in sources:
        cols.append(pack_rgb(np.asarray(rgb)[v, u]) if s < 0 else np.asarray(features, np.float32)[s, v, u])
    return np.ascontiguousarray(np.stack(cols, 1).astype(np.float32)), m.reshape(-1)


def special_depth(rng, H, W, max_depth=8.0):
    """Random depths with every special value of the mask: NaN, +-inf, 0, -0, negative, max_depth and the float below."""
    d = rng.uniform(-1.0, max_depth + 2.0, (H, W)).astype(np.float32)
    specials = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, -0.5, max_depth, np.nextafter(np.float32(max_depth), 0),
                         np.float32(1e-30), 0.3], np.float32)
    pick = rng.random((H, W)) < 0.3
    d[pick] = rng.choice(specials, int(pick.sum()))
    return d
