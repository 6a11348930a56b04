""""Next" row N2 (SURVEY.md §8f): the input formats that feed the boundary, as the reference's loaders read them
(aerial_mapper_io/src/aerial-mapper-io.cc).  Host-side only; no compute.

    load_poses_from_file_standard   :103-121   text stream  x y z qw qx qy qz
    load_point_cloud_from_file      :309-347   text stream  x y z intensity, keeps z > -100
    load_images_from_file           :207-227   <prefix><i>.jpg, gray (IMREAD_GRAYSCALE) or colour (BGR)
    load_camera_rig_from_file       :251-261   aslam NCamera YAML (camera 0: pinhole + distortion, T_B_C)

and the output side ("next" row N4):

    write_geotiff                   :349-509   toGeoTiff / writeDataToDEMGeoTiffColor, with the map's geotransform
"""
import struct

import numpy as np

from . import _lib
from .api import NCamera


def _tokens(path):
    with open(path, "r") as f:
        for line in f:
            for tok in line.split():
                yield tok


def load_poses_from_file_standard(filename):
    """`while (infile >> x >> y >> z >> qw >> qx >> qy >> qz)` (aerial-mapper-io.cc:110): a whitespace-separated
    stream, line breaks irrelevant, stops at the first token that is not a number or at an incomplete record.
    Returns float64 [n, 7]; raises if no pose was read (CHECK(T_G_Bs->size() > 0), :119)."""
    if not filename:
        raise ValueError("Empty filename")  # CHECK(!filename.empty()), :106
    vals = []
    for tok in _tokens(filename):
        try:
            vals.append(float(tok))
        except ValueError:
            break
    n = len(vals) // 7
    if n == 0:
        raise ValueError("No poses loaded.")
    return np.asarray(vals[:7 * n], dtype=np.float64).reshape(n, 7)


def load_point_cloud_from_file(filename, with_intensities=False):
    """`while (infile >> x >> y >> z >> intensity)` with `int intensity`; a point is kept iff z > -100
    (aerial-mapper-io.cc:318-323 / :338-344).  Returns xyz float64 [n, 3] (and int32 intensities)."""
    if not filename:
        raise ValueError("Empty filename")
    xyz, inten = [], []
    it = _tokens(filename)
    while True:
        rec = []
        try:
            for _ in range(3):
                rec.append(float(next(it)))
            tok = next(it)
            rec.append(int(tok))  # operator>>(int&): a token like "12.5" fails the extraction -> the loop ends
        except (StopIteration, ValueError):
            break
        if rec[2] > -100:
            xyz.append(rec[:3])
            inten.append(rec[3])
    if not xyz:
        raise ValueError("No points loaded.")  # CHECK(point_cloud_xyz->size() > 0)
    xyz = np.asarray(xyz, dtype=np.float64)
    if with_intensities:
        return xyz, np.asarray(inten, dtype=np.int32)
    return xyz


def load_images_from_file(filename_base, num_poses, load_colored_images=False):
    """filename_base + str(i) + ".jpg" for i in [0, num_poses) (aerial-mapper-io.cc:211-222).  Gray: uint8 [H, W];
    colour: uint8 [H, W, 3] in OpenCV's B, G, R byte order — what OrthoBackwardGrid.process expects."""
    import cv2
    images = []
    for i in range(int(num_poses)):
        name = "%s%d.jpg" % (filename_base, i)
        img = cv2.imread(name, cv2.IMREAD_COLOR if load_colored_images else cv2.IMREAD_GRAYSCALE)
        if img is None:
            raise IOError("cannot read %s" % name)
        images.append(np.ascontiguousarray(img))
    if not images:
        raise ValueError("No images loaded.")
    return images


def _matrix(node):
    rows, cols = int(node["rows"]), int(node["cols"])
    return np.asarray(node["data"], dtype=np.float64).reshape(rows, cols)


def _quat_from_matrix(R):
    """Unit quaternion (w, x, y, z) of a rotation matrix (Shepperd's method)."""
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0) * 2
        q = [0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s]
    else:
        k = int(np.argmax(np.diag(R)))
        a, b = (k + 1) % 3, (k + 2) % 3
        s = np.sqrt(1.0 + R[k, k] - R[a, a] - R[b, b]) * 2
        q = [0.0, 0.0, 0.0, 0.0]
        q[0] = (R[b, a] - R[a, b]) / s
        q[1 + k] = 0.25 * s
        q[1 + a] = (R[a, k] + R[k, a]) / s
        q[1 + b] = (R[b, k] + R[k, b]) / s
    q = np.asarray(q, dtype=np.float64)
    q /= np.linalg.norm(q)
    return q if q[0] >= 0 else -q


_DISTORTION = {"none": _lib.DIST_NONE, "null": _lib.DIST_NONE, "radial-tangential": _lib.DIST_RADTAN,
               "radtan": _lib.DIST_RADTAN, "equidistant": _lib.DIST_EQUIDISTANT,
               "fisheye": _lib.DIST_FOV, "fov": _lib.DIST_FOV}  # aslam FisheyeDistortion (restated from recollection, see
                                                                  # include/aerial_mapper_b200.h AMB_DIST_FOV)


def load_camera_rig_from_file(filename_ncameras_yaml, camera_index=0):
    """aslam::NCamera::deserializeFromFile (aerial-mapper-io.cc:251-261), camera `camera_index` only (the path uses
    camera 0: ortho-backward-grid.cc:131).  The YAML stores T_B_C; the path needs get_T_C_B = T_B_C^-1."""
    import yaml
    if not filename_ncameras_yaml:
        raise ValueError("Empty filename")
    with open(filename_ncameras_yaml, "r") as f:
        doc = yaml.safe_load(f)
    entry = doc["cameras"][camera_index]
    cam = entry["camera"]
    if cam.get("type", "pinhole") != "pinhole":
        raise ValueError("only pinhole cameras are on this path (got %r)" % cam.get("type"))
    fu, fv, cu, cv = _matrix(cam["intrinsics"]).ravel()[:4]
    dist = cam.get("distortion") or {"type": "none"}
    dtype = str(dist.get("type", "none")).lower()
    if dtype not in _DISTORTION:
        raise ValueError("unsupported distortion model %r" % dtype)
    params = [0.0, 0.0, 0.0, 0.0]
    if _DISTORTION[dtype] != _lib.DIST_NONE:
        p = _matrix(dist["parameters"]).ravel()
        params[:len(p[:4])] = [float(v) for v in p[:4]]
    T_B_C = _matrix(entry["T_B_C"])
    R_C_B = T_B_C[:3, :3].T
    t_C_B = -R_C_B @ T_B_C[:3, 3]
    return NCamera(int(cam["image_width"]), int(cam["image_height"]), fu, fv, cu, cv, _DISTORTION[dtype], params,
                   tuple(_quat_from_matrix(R_C_B)), tuple(t_C_B))


# ---- GeoTIFF (baseline TIFF 6.0 + GeoTIFF 1.0 tags), little-endian, uncompressed strips ----
_SHORT, _ASCII, _LONG, _DOUBLE = 3, 2, 4, 12
_TYPE_FMT = {_SHORT: "H", _LONG: "I", _DOUBLE: "d"}
_STRIP_BYTES = 1 << 20


def write_geotiff(path, raster, geotransform, epsg=32632, nodata=None):
    """io::AerialMapperIO::toGeoTiff (aerial-mapper-io.cc:349-509) with the map's own geotransform: a north-up raster
    whose GDAL-order `geotransform` is (west, res_x, 0, north, 0, -res_y) (GridMap.geotransform()), in the projected CRS
    `epsg` (default: the reference's hard-coded UTM zone 32N, :391-393).

    raster: uint8 or float32 [H, W] (one band; float32 is written with SampleFormat 3), or uint8 [H, W, 3] in B, G, R
    order (GridMap.to_raster(.., "bgr8")), stored as RGB one strip at a time.  nodata: GDAL_NODATA, e.g. "nan" for a DEM
    with NaN as no-data.  Uncompressed, no BigTIFF: a file over 4 GiB raises ValueError."""
    a = np.asarray(raster)
    if a.ndim == 2 and a.dtype in (np.uint8, np.float32):
        bands = 1
    elif a.ndim == 3 and a.shape[2] == 3 and a.dtype == np.uint8:
        bands = 3
    else:
        raise ValueError("raster must be uint8 or float32 [H, W], or uint8 [H, W, 3] (B, G, R); got %s %r"
                         % (a.dtype, a.shape))
    height, width = a.shape[:2]
    if height < 1 or width < 1:
        raise ValueError("empty raster")
    gt = [float(v) for v in geotransform]
    if len(gt) != 6 or gt[2] != 0.0 or gt[4] != 0.0 or not gt[1] > 0.0 or not gt[5] < 0.0:
        raise ValueError("a north-up geotransform (x0, res, 0, y0, 0, -res) is required, got %r" % (gt,))
    bits = 32 if a.dtype == np.float32 else 8
    row_bytes = width * bands * bits // 8
    rows_per_strip = max(1, min(height, _STRIP_BYTES // row_bytes))
    n_strips = (height + rows_per_strip - 1) // rows_per_strip
    strip_counts = [min(rows_per_strip, height - s * rows_per_strip) * row_bytes for s in range(n_strips)]

    geokeys = [1, 1, 0, 3,                 # GeoKeyDirectory header: version 1.1.0, 3 keys
               1024, 0, 1, 1,              # GTModelTypeGeoKey = ModelTypeProjected
               1025, 0, 1, 1,              # GTRasterTypeGeoKey = RasterPixelIsArea
               3072, 0, 1, int(epsg)]      # ProjectedCSTypeGeoKey
    tags = [(256, _LONG, [width]), (257, _LONG, [height]), (258, _SHORT, [bits] * bands), (259, _SHORT, [1]),
            (262, _SHORT, [2 if bands == 3 else 1]), (273, _LONG, [0] * n_strips), (277, _SHORT, [bands]),
            (278, _LONG, [rows_per_strip]), (279, _LONG, strip_counts), (284, _SHORT, [1]),
            (339, _SHORT, [3 if bits == 32 else 1] * bands),
            (33550, _DOUBLE, [gt[1], -gt[5], 0.0]),                  # ModelPixelScale
            (33922, _DOUBLE, [0.0, 0.0, 0.0, gt[0], gt[3], 0.0]),    # ModelTiepoint: pixel corner (0, 0) -> (west, north)
            (34735, _SHORT, geokeys)]
    if nodata is not None:
        tags.append((42113, _ASCII, ("%s" % nodata).encode("ascii") + b"\0"))   # GDAL_NODATA

    def payload(typ, vals):
        return bytes(vals) if typ == _ASCII else struct.pack("<%d%s" % (len(vals), _TYPE_FMT[typ]), *vals)

    ifd_at = 8
    extra_at = ifd_at + 2 + 12 * len(tags) + 4
    # sizes of the out-of-line values, then the strip offsets once the image data's position is known
    extra = sum((len(payload(t, v)) + 1) & ~1 for _, t, v in tags if len(payload(t, v)) > 4)
    data_at = (extra_at + extra + 15) & ~15
    total = data_at + sum(strip_counts)
    if total > 0xFFFFFFFF:
        raise ValueError("%d bytes: larger than a classic TIFF can address (4 GiB); BigTIFF is not supported" % total)
    offsets = [data_at + sum(strip_counts[:s]) for s in range(n_strips)]
    tags[5] = (273, _LONG, offsets)

    ifd = struct.pack("<H", len(tags))
    blobs = b""
    for tag, typ, vals in tags:
        p = payload(typ, vals)
        count = len(vals)
        if len(p) <= 4:
            ifd += struct.pack("<HHI", tag, typ, count) + p.ljust(4, b"\0")
        else:
            ifd += struct.pack("<HHII", tag, typ, count, extra_at + len(blobs))
            blobs += p + (b"\0" if len(p) & 1 else b"")
    ifd += struct.pack("<I", 0)
    with open(path, "wb") as f:
        f.write(b"II*\0" + struct.pack("<I", ifd_at) + ifd + blobs)
        f.write(b"\0" * (data_at - f.tell()))
        for s in range(n_strips):
            part = a[s * rows_per_strip:(s + 1) * rows_per_strip]
            if bands == 3:
                part = part[:, :, ::-1]               # B, G, R -> R, G, B, this strip only
            f.write(np.ascontiguousarray(part, dtype=a.dtype.newbyteorder("<")).tobytes())
