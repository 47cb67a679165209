"""Time image reprojection at 4000x2200: image_transformation_map() for OPENCV8 -> pinhole and splined -> pinhole
(tests/golden/cameramodels, pinhole_model_for_reprojection(fit="corners")), the call and the device time of its two
kernels; then transform_image() per frame on a uint8 RGB image through the OPENCV8 map: the numpy path (upload,
kernel, copy back), the torch device-resident path (map and image on the device, one kernel; CUDA events) and, if
cv2 imports, cv2.remap() on the host. Times are medians in ms. Prints one JSON line with the card's name, power limit
and SM clocks, read in the same run."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import mrcal_b200  # noqa: E402
import measure  # noqa: E402


def event_ms(f, reps):
    """median device time of f() on the current stream, CUDA events around each call. Not measure.median_ms(): a frame
    on the device takes about 0.1 ms, to which a host clock would add the launch and the synchronisation"""
    f()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        f()
        b.record()
        b.synchronize()
        t.append(a.elapsed_time(b))
    return float(np.median(t))


def map_case(name, reps):
    m = mrcal_b200.cameramodel(os.path.join(ROOT, "tests", "golden", "cameramodels", name))
    pinhole = mrcal_b200.pinhole_model_for_reprojection(m, fit="corners")
    f = lambda: mrcal_b200.image_transformation_map(m, pinhole, intrinsics_only=True)
    W, H = (int(x) for x in pinhole.imagersize())
    return f(), {"imager_to": [W, H], "ms_call": measure.median_ms(f, reps),
                 "ms_unprojection_kernel": measure.kernel_ms(f, "reprojection_rays_kernel"),
                 "ms_projection_kernel": measure.kernel_ms(f, "reprojection_map_kernel")}


def main():
    out = {}
    mapxy, out["map_opencv8_to_pinhole"] = map_case("cam0.opencv8.cameramodel", 5)
    _, out["map_splined_to_pinhole"] = map_case("cam0.splined.cameramodel", 5)
    H, W = mapxy.shape[:2]
    image = np.random.default_rng(0).integers(0, 256, (H, W, 3), dtype=np.uint8)
    res = {"ms_numpy_call": measure.median_ms(lambda: mrcal_b200.transform_image(image, mapxy), 10)}
    image_d, map_d = torch.from_numpy(image).cuda(), torch.from_numpy(mapxy).cuda()
    out_d = torch.empty_like(image_d)
    frame = lambda: mrcal_b200.transform_image(image_d, map_d, out=out_d)
    res["ms_torch_device"] = event_ms(frame, 50)
    res["ms_torch_kernel"] = measure.kernel_ms(frame, "remap_kernel")
    try:
        import cv2
        res["ms_cv2_remap_host"] = measure.median_ms(
            lambda: cv2.remap(image, mapxy, None, interpolation=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT), 10)
    except ImportError:
        res["ms_cv2_remap_host"] = "not measured: cv2 does not import"
    out["transform_image_uint8_rgb"] = res
    measure.emit(out)


if __name__ == "__main__":
    main()
