""""Next" row N2 (SURVEY.md §8f): the input formats that feed the boundary, as the reference's loaders read them
(aerial_mapper_io/src/aerial-mapper-io.cc).  Host-side only; no compute.

    load_poses_from_file_standard   :103-121   text stream  x y z qw qx qy qz
    load_point_cloud_from_file      :309-347   text stream  x y z intensity, keeps z > -100
    load_images_from_file           :207-227   <prefix><i>.jpg, gray (IMREAD_GRAYSCALE) or colour (BGR)
    read_jpeg_files                            the same files undecoded, for OrthoBackwardGrid.process_jpeg
    load_camera_rig_from_file       :251-261   aslam NCamera YAML (camera 0: pinhole + distortion, T_B_C)

and the output side ("next" row N4):

    write_geotiff                   :349-509   toGeoTiff / writeDataToDEMGeoTiffColor, with the map's geotransform
    write_geotiff_strips                        the same tags around Deflate strips compressed on the device

and back in: read_geotiff, the DEM GeoTIFFs GDAL writes (GridMap.from_raster resamples them into a layer), and
read_geotiff_device, the same files decoded on a GPU (GridMap.from_geotiff imports them straight from the file).
"""
import ctypes as C
import math
import os
import struct
import zlib

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


def read_jpeg_files(filename_base, num_poses):
    """The raw bytes of filename_base + str(i) + ".jpg" for i in [0, num_poses), the names load_images_from_file reads,
    with its errors: for OrthoBackwardGrid.process_jpeg, which decodes the frames that contribute on the device."""
    files = []
    for i in range(int(num_poses)):
        name = "%s%d.jpg" % (filename_base, i)
        try:
            with open(name, "rb") as f:
                files.append(f.read())
        except OSError:
            raise IOError("cannot read %s" % name)
    if not files:
        raise ValueError("No images loaded.")
    return files


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


# ---- GeoTIFF (baseline TIFF 6.0 + GeoTIFF 1.0 tags), little-endian, uncompressed or Deflate strips ----
_SHORT, _ASCII, _LONG, _RATIONAL, _UNDEFINED, _DOUBLE = 3, 2, 4, 5, 7, 12
_TYPE_FMT = {_SHORT: "H", _LONG: "I", _RATIONAL: "I", _DOUBLE: "d"}
_STRIP_BYTES = 1 << 20


def _check_raster(a):
    """(bands, bits) of a raster write_geotiff accepts, else ValueError."""
    if a.ndim == 2 and a.dtype in (np.uint8, np.float32):
        bands = 1
    elif a.ndim == 3 and a.shape[2] == 3 and a.dtype == np.uint8:
        bands = 3
    else:
        raise ValueError("raster must be uint8 or float32 [H, W], or uint8 [H, W, 3] (B, G, R); got %s %r"
                         % (a.dtype, a.shape))
    if a.shape[0] < 1 or a.shape[1] < 1:
        raise ValueError("empty raster")
    return bands, (32 if a.dtype == np.float32 else 8)


def _north_up(geotransform):
    gt = [float(v) for v in geotransform]
    if len(gt) != 6 or gt[2] != 0.0 or gt[4] != 0.0 or not gt[1] > 0.0 or not gt[5] < 0.0:
        raise ValueError("a north-up geotransform (x0, res, 0, y0, 0, -res) is required, got %r" % (gt,))
    return gt


def _image_tags(width, height, bands, bits, predictor, layout, geo=None, subfile=None, compression=None,
                photometric=None, extra=()):
    """The tags of one image's IFD in ascending order: `layout` holds its strip or tile tags; predictor None for
    uncompressed data, else Compression 8 (Deflate) with that Predictor; geo (geotransform, epsg, nodata) adds the
    georeferencing; subfile, if given, NewSubfileType (0 full resolution, 1 reduced, 4 / 5 their masks).  compression
    and photometric, if given, replace those the predictor and the bands imply (JPEG, YCbCr, masks); extra: more tags."""
    if compression is None:
        compression = 1 if predictor is None else 8
    if photometric is None:
        photometric = 2 if bands == 3 else 1
    tags = [(256, _LONG, [width]), (257, _LONG, [height]), (258, _SHORT, [bits] * bands),
            (259, _SHORT, [compression]), (262, _SHORT, [photometric]),
            (277, _SHORT, [bands]), (284, _SHORT, [1]), (339, _SHORT, [3 if bits == 32 else 1] * bands)]
    tags += list(layout) + list(extra)
    if subfile is not None:
        tags.append((254, _LONG, [subfile]))
    if predictor is not None:
        tags.append((317, _SHORT, [predictor]))
    if geo is not None:
        gt, epsg, nodata = geo
        geokeys = [1, 1, 0, 3,                 # GeoKeyDirectory header: version 1.1.0, 3 keys
                   1024, 0, 1, 1,              # GTModelTypeGeoKey = ModelTypeProjected
                   1025, 0, 1, 1,              # GTRasterTypeGeoKey = RasterPixelIsArea
                   3072, 0, 1, int(epsg)]      # ProjectedCSTypeGeoKey
        tags += [(33550, _DOUBLE, [gt[1], -gt[5], 0.0]),                  # ModelPixelScale
                 (33922, _DOUBLE, [0.0, 0.0, 0.0, gt[0], gt[3], 0.0]),    # ModelTiepoint: pixel corner (0, 0) -> (west, north)
                 (34735, _SHORT, geokeys)]
        if nodata is not None:
            tags.append((42113, _ASCII, ("%s" % nodata).encode("ascii") + b"\0"))   # GDAL_NODATA
    return sorted(tags, key=lambda t: t[0])


def _payload(typ, vals):
    if typ in (_ASCII, _UNDEFINED):
        return bytes(vals)
    return struct.pack("<%d%s" % (len(vals), _TYPE_FMT[typ]), *vals)


def _count(typ, vals):
    """The TIFF count of `vals`: a RATIONAL is given as its numerator and denominator."""
    return len(vals) // 2 if typ == _RATIONAL else len(vals)


def _ifd_size(tags):
    """Bytes of the IFD of `tags` and its out-of-line values (each padded to an even length)."""
    return 2 + 12 * len(tags) + 4 + sum((len(_payload(t, v)) + 1) & ~1 for _, t, v in tags if len(_payload(t, v)) > 4)


def _set_tag(tags, tag, typ, vals):
    return [(k, typ, list(vals)) if k == tag else (k, t, v) for k, t, v in tags]


def _ifd(tags, at, next_ifd=0):
    """The IFD of `tags` at file offset `at`, pointing to the next IFD at `next_ifd` (0: the last), followed by its
    out-of-line values: _ifd_size(tags) bytes."""
    extra_at = at + 2 + 12 * len(tags) + 4
    ifd = struct.pack("<H", len(tags))
    blobs = b""
    for tag, typ, vals in tags:
        p = _payload(typ, vals)
        count = _count(typ, vals)
        if len(p) <= 4:
            ifd += struct.pack("<HHI", tag, typ, count) + p.ljust(4, b"\0")
        else:
            ifd += struct.pack("<HHII", tag, typ, count, extra_at + len(blobs))
            blobs += p + (b"\0" if len(p) & 1 else b"")
    return ifd + struct.pack("<I", next_ifd) + blobs


def _check_size(total):
    if total > 0xFFFFFFFF:
        raise ValueError("%d bytes: larger than a classic TIFF can address (4 GiB); BigTIFF is not supported" % total)


def _tiff_layout(width, height, bands, bits, rows_per_strip, strip_counts, geotransform, epsg, nodata,
                 predictor=None):
    """The file's bytes up to its first strip (header, the one IFD, its out-of-line values, zero padding to a 16-byte
    boundary), for strips of `strip_counts` bytes stored back to back after it.  predictor: None for uncompressed
    strips, else Compression 8 (Deflate) with that Predictor.  A file over 4 GiB raises ValueError (no BigTIFF)."""
    gt = _north_up(geotransform)
    n_strips = len(strip_counts)
    layout = [(273, _LONG, [0] * n_strips), (278, _LONG, [rows_per_strip]), (279, _LONG, list(strip_counts))]
    tags = _image_tags(width, height, bands, bits, predictor, layout, (gt, epsg, nodata))
    ifd_at = 8
    data_at = (ifd_at + _ifd_size(tags) + 15) & ~15
    _check_size(data_at + sum(strip_counts))
    offsets = np.concatenate([[0], np.cumsum(np.asarray(strip_counts, np.int64))[:-1]]) + data_at
    tags = _set_tag(tags, 273, _LONG, [int(v) for v in offsets])
    head = b"II*\0" + struct.pack("<I", ifd_at) + _ifd(tags, ifd_at)
    return head + b"\0" * (data_at - len(head))


def write_geotiff(path, raster, geotransform, epsg=32632, nodata=None):
    """io::AerialMapperIO::toGeoTiff (aerial-mapper-io.cc:349-509) with the map's own geotransform: a north-up raster
    whose GDAL-order `geotransform` is (west, res_x, 0, north, 0, -res_y) (GridMap.geotransform()), in the projected CRS
    `epsg` (default: the reference's hard-coded UTM zone 32N, :391-393).

    raster: uint8 or float32 [H, W] (one band; float32 is written with SampleFormat 3), or uint8 [H, W, 3] in B, G, R
    order (GridMap.to_raster(.., "bgr8")), stored as RGB one strip at a time.  nodata: GDAL_NODATA, e.g. "nan" for a DEM
    with NaN as no-data.  Uncompressed, no BigTIFF: a file over 4 GiB raises ValueError.  GridMap.to_geotiff writes
    Deflate-compressed files."""
    a = np.asarray(raster)
    bands, bits = _check_raster(a)
    height, width = a.shape[:2]
    row_bytes = width * bands * bits // 8
    rows_per_strip = max(1, min(height, _STRIP_BYTES // row_bytes))
    n_strips = (height + rows_per_strip - 1) // rows_per_strip
    strip_counts = [min(rows_per_strip, height - s * rows_per_strip) * row_bytes for s in range(n_strips)]
    head = _tiff_layout(width, height, bands, bits, rows_per_strip, strip_counts, geotransform, epsg, nodata)
    with open(path, "wb") as f:
        f.write(head)
        for s in range(n_strips):
            part = a[s * rows_per_strip:(s + 1) * rows_per_strip]
            if bands == 3:
                part = part[:, :, ::-1]               # B, G, R -> R, G, B, this strip only
            f.write(np.ascontiguousarray(part, dtype=a.dtype.newbyteorder("<")).tobytes())


def write_geotiff_strips(path, data, strip_bytes, width, height, fmt, rows_per_strip, geotransform, epsg=32632,
                         nodata=None):
    """Writes Deflate-compressed strips (GridMap.to_geotiff, deflate_strips; convention in include/aerial_mapper_b200.h,
    amb_deflate_strips_device) as a GeoTIFF with the tags write_geotiff writes, plus Compression 8 and Predictor 3 for
    fmt "f32", 2 for "gray8", "bgr8" and "mask8".  data: the strips back to back; strip_bytes: each strip's length."""
    bands, bits, predictor = _DEFLATE_FORMATS[fmt]
    data = memoryview(data).cast("B")
    counts = [int(v) for v in strip_bytes]
    rps = int(rows_per_strip)
    if width < 1 or height < 1 or rps < 1 or len(counts) != (height + rps - 1) // rps or sum(counts) != len(data):
        raise ValueError("write_geotiff_strips: %d strips of %d bytes in all do not fit a %d x %d raster in strips of %d "
                         "rows" % (len(counts), sum(counts), width, height, rps))
    head = _tiff_layout(int(width), int(height), bands, bits, min(rps, int(height)), counts, geotransform, epsg, nodata,
                        predictor)
    with open(path, "wb") as f:
        f.write(head)
        f.write(data)


_DEFLATE_FORMATS = {"f32": (1, 32, 3), "gray8": (1, 8, 2), "bgr8": (3, 8, 2), "mask8": (1, 8, 2)}  # bands, bits, predictor


def cog_layout(width, height, tile):
    """[(w_k, h_k)] of the levels of a Cloud-Optimized GeoTIFF (amb_cog_layout): level 0 first."""
    n = C.c_int32(0)
    lw, lh = (C.c_int32 * 32)(), (C.c_int32 * 32)()
    st = _lib.lib().amb_cog_layout(int(width), int(height), int(tile), C.byref(n), lw, lh)
    if st != _lib.AMB_OK:
        raise ValueError("no COG levels for a %r x %r raster in tiles of %r" % (width, height, tile))
    return [(lw[k], lh[k]) for k in range(n.value)]


def cog_nodata(fmt, nodata):
    """The GDAL_NODATA written for `nodata`, which must agree with the overviews' reduction: NaN for "f32" (NaN pixels
    are left out of the means), 0 for "mask8" (the maximum keeps 0 only where every child is 0), none for "gray8" and
    "bgr8" (their means would take a no-data value in).  Anything else raises ValueError."""
    if nodata is None:
        return None
    if fmt == "f32":
        if isinstance(nodata, str) and nodata.strip().lower() == "nan":
            return "nan"
        if isinstance(nodata, (float, np.floating)) and math.isnan(nodata):
            return "nan"
    elif fmt == "mask8":
        if not isinstance(nodata, (str, bool, np.bool_)) and isinstance(nodata, (int, float, np.integer, np.floating)) \
                and nodata == 0:
            return 0
    raise ValueError("COG nodata %r does not agree with the %r overviews: use %s" % (
        nodata, fmt, {"f32": "'nan'", "mask8": "0"}.get(fmt, "None")))


_JPEG_SAMPLING = {"420": (2, 2), "444": (1, 1)}


def write_cog(path, data, tile_bytes, width, height, fmt, tile, geotransform, epsg=32632, nodata=None,
              compress="deflate", jpeg_tables=None, sampling="420", mask=None):
    """Writes Cloud-Optimized GeoTIFF tiles (GridMap.to_cog, cog_tiles; convention in include/aerial_mapper_b200.h,
    amb_cog_tiles_device) as a classic TIFF: the header, the IFD of level 0 at offset 8 and then those of the overviews
    in decreasing size, each followed by its out-of-line values, then the tile data in file order (the smallest level
    first, row-major within a level).  Every IFD has TileWidth = TileLength = tile, Compression 8 and the predictor of
    write_geotiff_strips; level 0 has NewSubfileType 0 and the georeferencing and GDAL_NODATA, each overview
    NewSubfileType 1.  nodata: see cog_nodata.  data: the tiles back to back; tile_bytes: each tile's length.  A file
    over 4 GiB raises ValueError (no BigTIFF).

    compress="jpeg" (cog_jpeg_tiles; "gray8" and "bgr8" only, no nodata): Compression 7 with the JPEGTables stream
    `jpeg_tables` on every image IFD, no Predictor; "bgr8" as Photometric 6 (YCbCr) with YCbCrSubSampling 2, 2 for
    sampling "420" (1, 1 for "444") and ReferenceBlackWhite 0 255 128 255 128 255, "gray8" as Photometric 1.

    mask=(data, tile_bytes) (cog_mask_tiles; "gray8" and "bgr8" only) adds GDAL's internal mask: after each level's IFD
    the IFD of its mask, NewSubfileType 4 at level 0 and 5 on the overviews, Photometric 4, BitsPerSample 1, Compression
    8 without a predictor, the same tiling; in the data each image tile is followed by its mask tile."""
    if compress not in ("deflate", "jpeg"):
        raise ValueError("write_cog: compress must be 'deflate' or 'jpeg', got %r" % (compress,))
    jpeg = compress == "jpeg"
    if jpeg or mask is not None:
        if fmt not in ("gray8", "bgr8"):
            raise ValueError("write_cog: %s is for 'gray8' and 'bgr8' only, got %r"
                             % ("JPEG" if jpeg else "a mask", fmt))
    bands, bits, predictor = _DEFLATE_FORMATS[fmt]
    if jpeg:
        if nodata is not None:
            raise ValueError("write_cog: a JPEG COG has no no-data value (JPEG is lossy): give a mask instead")
        if sampling not in _JPEG_SAMPLING:
            raise ValueError("write_cog: sampling must be '420' or '444', got %r" % (sampling,))
        tables = bytes(jpeg_tables or b"")
        if tables[:4] != b"\xff\xd8\xff\xdb" or tables[-2:] != b"\xff\xd9":
            raise ValueError("write_cog: jpeg_tables must be a tables stream (SOI, DQT ..., DHT ..., EOI)")
    nd = cog_nodata(fmt, nodata)
    gt = _north_up(geotransform)
    data = memoryview(data).cast("B")
    counts = [int(v) for v in tile_bytes]
    levels = cog_layout(width, height, tile)
    n_tiles = [-(-w // tile) * -(-h // tile) for w, h in levels]
    if len(counts) != sum(n_tiles) or sum(counts) != len(data):
        raise ValueError("write_cog: %d tiles of %d bytes in all do not fit a %d x %d raster in tiles of %d (%d tiles)"
                         % (len(counts), sum(counts), width, height, tile, sum(n_tiles)))
    if mask is not None:
        mdata = memoryview(mask[0]).cast("B")
        mcounts = [int(v) for v in mask[1]]
        if len(mcounts) != len(counts) or sum(mcounts) != len(mdata):
            raise ValueError("write_cog: %d mask tiles of %d bytes in all do not match the %d image tiles"
                             % (len(mcounts), sum(mcounts), len(counts)))
    first = np.cumsum([0] + n_tiles[::-1])[::-1][1:]      # each level's first tile in file order (the smallest first)
    kw = {}
    if jpeg:
        extra = [(347, _UNDEFINED, list(tables))]
        if bands == 3:
            extra += [(530, _SHORT, list(_JPEG_SAMPLING[sampling])),
                      (532, _RATIONAL, [0, 1, 255, 1, 128, 1, 255, 1, 128, 1, 255, 1])]
        kw = {"compression": 7, "photometric": 6 if bands == 3 else 1, "extra": extra}
    tags, kinds = [], []                                  # kinds: 0 image, 1 mask
    for k, (w, h) in enumerate(levels):
        c = counts[first[k]:first[k] + n_tiles[k]]
        layout = [(322, _LONG, [tile]), (323, _LONG, [tile]), (324, _LONG, [0] * len(c)), (325, _LONG, c)]
        tags.append(_image_tags(w, h, bands, bits, None if jpeg else predictor, layout,
                                (gt, epsg, nd) if k == 0 else None, subfile=0 if k == 0 else 1, **kw))
        kinds.append(0)
        if mask is not None:
            mc = mcounts[first[k]:first[k] + n_tiles[k]]
            layout = [(322, _LONG, [tile]), (323, _LONG, [tile]), (324, _LONG, [0] * len(mc)), (325, _LONG, mc)]
            tags.append(_image_tags(w, h, 1, 1, None, layout, subfile=4 if k == 0 else 5, compression=8,
                                    photometric=4))
            kinds.append(1)
    ifd_at = [8]
    for t in tags:
        ifd_at.append(ifd_at[-1] + _ifd_size(t))
    data_at = (ifd_at[-1] + 15) & ~15
    total = len(data) + (len(mdata) if mask is not None else 0)
    _check_size(data_at + total)
    # file offsets of every tile (and mask tile), in file order: image tile i then its mask tile
    step = np.asarray(counts, np.int64) + (np.asarray(mcounts, np.int64) if mask is not None else 0)
    starts = np.concatenate([[0], np.cumsum(step)[:-1]]) + data_at
    head = b"II*\0" + struct.pack("<I", 8)
    for j, t in enumerate(tags):
        k = j // 2 if mask is not None else j
        s = starts[first[k]:first[k] + n_tiles[k]]
        if kinds[j]:
            s = s + np.asarray(counts[first[k]:first[k] + n_tiles[k]], np.int64)
        t = _set_tag(t, 324, _LONG, [int(v) for v in s])
        head += _ifd(t, ifd_at[j], ifd_at[j + 1] if j + 1 < len(tags) else 0)
    with open(path, "wb") as f:
        f.write(head + b"\0" * (data_at - len(head)))
        if mask is None:
            f.write(data)
        else:
            at = mat = 0
            for n, m in zip(counts, mcounts):
                f.write(data[at:at + n])
                f.write(mdata[mat:mat + m])
                at += n
                mat += m


# ---- GeoTIFF reader: the subset GDAL writes for DEMs ----
_TIFF_TYPES = {1: "B", 2: "s", 3: "H", 4: "I", 5: "II", 6: "b", 7: "B", 8: "h", 9: "i", 10: "ii", 11: "f", 12: "d"}
_SAMPLE_DTYPES = {(8, 1): np.uint8, (16, 2): np.int16, (16, 1): np.uint16, (32, 2): np.int32, (32, 3): np.float32,
                  (64, 3): np.float64}


def write_jpeg(path, data, geotransform=None):
    """Writes the JPEG file `data` (bytes from GridMap.to_jpeg or encode_jpeg) to `path`.  With a GDAL-order
    geotransform (GridMap.geotransform()) it also writes the ESRI world file next to it (`path` with the extension
    .jgw): x pixel size, the two rotation terms, y pixel size, then the centre of the top-left pixel (world files
    locate pixel centres, GDAL geotransforms pixel corners)."""
    data = bytes(data)
    if data[:2] != b"\xff\xd8" or data[-2:] != b"\xff\xd9":
        raise ValueError("write_jpeg: data is not a JPEG file (SOI ... EOI)")
    if geotransform is not None:
        gt = [float(v) for v in geotransform]
        if len(gt) != 6 or not all(math.isfinite(v) for v in gt):
            raise ValueError("write_jpeg: geotransform must be 6 finite numbers, got %r" % (geotransform,))
    with open(path, "wb") as f:
        f.write(data)
    if geotransform is not None:
        lines = (gt[1], gt[4], gt[2], gt[5], gt[0] + gt[1] / 2 + gt[2] / 2, gt[3] + gt[4] / 2 + gt[5] / 2)
        with open(os.path.splitext(path)[0] + ".jgw", "w") as f:
            f.write("".join("%r\n" % v for v in lines))


def _unsupported(tag, value, why):
    raise ValueError("read_geotiff: %s = %r is not supported (%s)" % (tag, value, why))


def _read_ifd(data, at=None):
    """Tag -> tuple of values (ASCII: str) of the IFD at offset `at` (by default the first) of a classic little-endian
    TIFF."""
    if len(data) < 8:
        raise ValueError("read_geotiff: not a TIFF file (%d bytes)" % len(data))
    if data[:2] == b"MM":
        _unsupported("byte order", "MM", "big-endian TIFF")
    if data[:2] != b"II":
        raise ValueError("read_geotiff: not a TIFF file (byte order mark %r)" % data[:2])
    magic = struct.unpack_from("<H", data, 2)[0]
    if magic == 43:
        _unsupported("version", 43, "BigTIFF")
    if magic != 42:
        raise ValueError("read_geotiff: not a TIFF file (version %d)" % magic)
    if at is None:
        at = struct.unpack_from("<I", data, 4)[0]
    n = struct.unpack_from("<H", data, at)[0]
    tags = {}
    for e in range(n):
        tag, typ, count, raw = struct.unpack_from("<HHI4s", data, at + 2 + 12 * e)
        if typ not in _TIFF_TYPES:
            _unsupported("type of tag %d" % tag, typ, "not a classic TIFF field type")
        fmt = _TIFF_TYPES[typ]
        size = struct.calcsize("<" + fmt) * count
        buf = raw if size <= 4 else data[struct.unpack("<I", raw)[0]:struct.unpack("<I", raw)[0] + size]
        if typ == 2:
            tags[tag] = buf[:count].split(b"\0")[0].decode("ascii", "replace")
        else:
            tags[tag] = struct.unpack_from("<%d%s" % (count * len(fmt), fmt[0]), buf)
    return tags


def _next_ifd(data, at):
    """The offset of the IFD after the one at `at` (0: none)."""
    return struct.unpack_from("<I", data, at + 2 + 12 * struct.unpack_from("<H", data, at)[0])[0]


def _overview_ifd(data, k):
    """The IFD of overview k >= 1: the k-th IFD after the first that is a reduced image (NewSubfileType bit 0) and not a
    mask (bit 2)."""
    first = struct.unpack_from("<I", data, 4)[0]
    seen, at, found = {first}, _next_ifd(data, first), 0
    while at and at not in seen and at + 2 <= len(data):
        seen.add(at)
        tags = _read_ifd(data, at)
        kind = tags.get(254, (0,))[0]
        if kind & 1 and not kind & 4:
            found += 1
            if found == k:
                return tags
        at = _next_ifd(data, at)
    raise ValueError("read_geotiff: overview %d requested, the file has %d" % (k, found))


def _geotransform(tags):
    if 34264 in tags:                                   # ModelTransformation, row-major 4 x 4
        m = tags[34264]
        if len(m) != 16:
            _unsupported("ModelTransformation", m, "16 values expected")
        if m[1] != 0.0 or m[4] != 0.0:
            _unsupported("ModelTransformation", m, "rotated geotransform")
        gt = [m[3], m[0], m[1], m[7], m[4], m[5]]
    elif 33550 in tags and 33922 in tags:               # ModelPixelScale + ModelTiepoint (I, J, K, X, Y, Z)
        sx, sy = tags[33550][0], tags[33550][1]
        tp = tags[33922]
        if len(tp) != 6:
            _unsupported("ModelTiepoint", tp, "exactly one tiepoint expected")
        i, j, x, y = tp[0], tp[1], tp[3], tp[4]
        gt = [x - i * sx, sx, 0.0, y + j * sy, 0.0, -sy]
    else:
        raise ValueError("read_geotiff: no georeferencing (ModelPixelScale + ModelTiepoint or ModelTransformation)")
    keys = _geokeys(tags)
    if keys.get(1025) == 2:                             # GTRasterTypeGeoKey = RasterPixelIsPoint: GDAL's half-pixel shift
        gt[0] -= 0.5 * gt[1] + 0.5 * gt[2]
        gt[3] -= 0.5 * gt[4] + 0.5 * gt[5]
    if not all(math.isfinite(v) for v in gt) or not gt[1] > 0.0 or not gt[5] < 0.0:
        _unsupported("geotransform", tuple(gt), "north-up (x0, res, 0, y0, 0, -res) only")
    return tuple(float(v) for v in gt)


def _geokeys(tags):
    """GeoKeyDirectory: key id -> SHORT value stored in the directory itself (the keys read here are all such)."""
    d = tags.get(34735, ())
    keys = {}
    for k in range(1, (len(d) // 4)):
        kid, loc, count, val = d[4 * k:4 * k + 4]
        if loc == 0 and count == 1:
            keys[kid] = val
    return keys


def _undo_predictor(chunk, predictor, dtype, rows, cols, spp):
    """chunk: the decoded bytes of `rows` rows of `cols` pixels of `spp` samples -> dtype [rows, cols, spp]."""
    item = np.dtype(dtype).itemsize
    raw = np.frombuffer(chunk, np.uint8, rows * cols * spp * item)
    if predictor == 3:                                  # byte planes, most significant first, differenced with stride spp
        b = raw.reshape(rows, cols, spp * item)
        b = np.cumsum(b.reshape(rows, cols * item, spp), axis=1, dtype=np.uint8).reshape(rows, item, cols * spp)
        be = np.ascontiguousarray(b.transpose(0, 2, 1))  # [rows, samples, bytes MSB..LSB]
        return be.view(np.dtype(dtype).newbyteorder(">")).reshape(rows, cols, spp).astype(dtype)
    a = raw.view(np.dtype(dtype).newbyteorder("<")).reshape(rows, cols, spp).astype(dtype)
    if predictor == 2:                                  # horizontal differencing, modulo the sample type
        a = np.cumsum(a, axis=1, dtype=dtype)
    return a


def read_geotiff(path, band=0, overview=0):
    """A band of a GeoTIFF as GDAL writes DEMs: (array [H, W] in the file's sample type, GDAL geotransform (west, res_x, 0,
    north, 0, -res_y), EPSG code or None, no-data value or None).

    Reads classic little-endian TIFF (first IFD, PlanarConfiguration 1), strips or tiles, uncompressed or Deflate,
    predictor 1, 2 (integer samples) or 3 (floating point), samples uint8, int16, uint16, int32, float32 or float64.  The
    geotransform comes from ModelPixelScale + ModelTiepoint (one tiepoint, at any raster point) or from a
    ModelTransformation without rotation; GTRasterTypeGeoKey = PixelIsPoint shifts it by half a pixel, as GDAL reads it.
    EPSG: ProjectedCSTypeGeoKey, else GeographicTypeGeoKey.  No-data: GDAL_NODATA as a float ("nan" included).  Anything
    else raises ValueError naming the tag and value (BigTIFF, big-endian, LZW, JPEG, rotated transforms ...).

    overview k >= 1 reads the k-th reduced-resolution IFD after the first (a COG's levels, GridMap.to_cog), whose
    geotransform is the first IFD's with its pixel sizes scaled by W / w_k and H / h_k (GDAL's rule); EPSG and no-data
    are the first IFD's.  An overview the file does not have raises ValueError.

    For GridMap.from_raster a DEM is converted with a.astype(np.float32), its no-data value passed along: that value must
    be exact in float32 (true of every int16 and uint16 value) or pixels holding it will not compare equal.

    read_geotiff_device reads the same files on a GPU."""
    with open(path, "rb") as f:
        data = f.read()
    t = tiff_layout(data, band, overview)
    out = np.empty((t.height, t.width), t.dtype)
    for (r0, c0, rows, cols), at, n in zip(t.grid, t.offsets, t.counts):
        if r0 >= t.height or c0 >= t.width:
            continue
        chunk = data[at:at + n]
        if t.compression != 1:
            chunk = zlib.decompress(chunk)
        a = _undo_predictor(chunk, t.predictor, t.dtype, rows, cols, t.spp)
        out[r0:r0 + rows, c0:c0 + cols] = a[:t.height - r0, :t.width - c0, band]
    return (out,) + t.georeferencing()


class TiffLayout(object):
    """One image of a TIFF as read_geotiff reads it (tiff_layout): its size, samples, compression and predictor, and its
    chunks: grid [(row, column, rows, columns)] of every strip or tile (full tiles at the edges, the last strip short),
    offsets and counts into the file.  base: the first IFD's tags, tags: the image's own."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def georeferencing(self):
        """(GDAL geotransform, EPSG code or None, no-data value or None) of the image, as read_geotiff returns them: an
        overview's pixel sizes are the first IFD's scaled by W / w_k and H / h_k."""
        base = self.base
        keys = _geokeys(base)
        epsg = keys.get(3072, keys.get(2048))
        nodata = base.get(42113)
        gt = _geotransform(base)
        if self.overview:
            sx, sy = base[256][0] / self.width, base[257][0] / self.height
            gt = (gt[0], gt[1] * sx, gt[2], gt[3], gt[4], gt[5] * sy)
        return gt, (None if epsg in (None, 0, 32767) else int(epsg)), (None if nodata is None else float(nodata.strip()))

    def c_layout(self):
        """The amb_tiff_layout of the image's grid of chunks (the arrays it points to live as long as the result)."""
        n = len(self.grid)
        if min(len(self.offsets), len(self.counts)) < n:
            raise ValueError("read_geotiff_device: %d chunk offsets and %d byte counts for a grid of %d chunks"
                             % (len(self.offsets), len(self.counts), n))
        offsets = np.asarray(self.offsets[:n], np.uint64)
        counts = np.asarray(self.counts[:n], np.uint64)
        L = _lib.TiffLayout(self.width, self.height, self.chunk_width, self.chunk_height, int(self.tiled), self.spp,
                            self.band, _lib.SAMPLE_TYPE[np.dtype(self.dtype).name], self.compression, self.predictor, n,
                            0, offsets.ctypes.data, counts.ctypes.data)
        L._keep = (offsets, counts)
        return L


def tiff_layout(data, band=0, overview=0):
    """The TiffLayout of band `band` of image `overview` of the TIFF file `data` (bytes), with read_geotiff's checks:
    anything it does not read raises ValueError naming the tag and value."""
    if isinstance(overview, bool) or not isinstance(overview, (int, np.integer)) or overview < 0:
        raise ValueError("read_geotiff: overview must be a non-negative integer, got %r" % (overview,))
    base = tags = _read_ifd(data)
    if overview:
        tags = _overview_ifd(data, int(overview))
    width, height = tags[256][0], tags[257][0]
    spp = tags.get(277, (1,))[0]
    planar = tags.get(284, (1,))[0]
    if planar != 1:
        _unsupported("PlanarConfiguration", planar, "chunky (1) only")
    bits = set(tags.get(258, (1,)))
    fmt = set(tags.get(339, (1,)))
    if len(bits) != 1 or len(fmt) != 1 or (bits.pop(), fmt.pop()) not in _SAMPLE_DTYPES:
        _unsupported("BitsPerSample / SampleFormat", (tags.get(258), tags.get(339)),
                     "uint8, int16, uint16, int32, float32 or float64 samples")
    dtype = _SAMPLE_DTYPES[(tags[258][0], tags.get(339, (1,))[0])]
    if not 0 <= band < spp:
        raise ValueError("read_geotiff: band %d of %d" % (band, spp))
    comp = tags.get(259, (1,))[0]
    if comp not in (1, 8, 32946):
        _unsupported("Compression", comp, "none (1) or Deflate (8, 32946) only")
    predictor = tags.get(317, (1,))[0]
    is_float = np.dtype(dtype).kind == "f"
    if predictor not in (1, 2, 3) or (predictor == 2 and is_float) or (predictor == 3 and not is_float):
        _unsupported("Predictor", predictor, "1, 2 for integer or 3 for floating-point samples")
    if 322 in tags:                                     # tiles
        tw, th = tags[322][0], tags[323][0]
        offsets, counts = tags[324], tags[325]
        across = (width + tw - 1) // tw
        grid = [((k // across) * th, (k % across) * tw, th, tw) for k in range(len(offsets))]
        tiled, cw, ch = True, tw, th
    elif 273 in tags:                                   # strips
        rps = min(tags.get(278, (height,))[0], height)
        offsets, counts = tags[273], tags[279]
        grid = [(k * rps, 0, min(rps, height - k * rps), width) for k in range(len(offsets))]
        tiled, cw, ch = False, width, rps
    else:
        raise ValueError("read_geotiff: neither strips nor tiles")
    n_grid = -(-height // ch) * (-(-width // cw) if tiled else 1)
    return TiffLayout(base=base, tags=tags, overview=int(overview), width=width, height=height, spp=spp, band=band,
                      dtype=dtype, compression=comp, predictor=predictor, tiled=tiled, chunk_width=cw, chunk_height=ch,
                      offsets=offsets, counts=counts, grid=grid[:n_grid] if len(grid) >= n_grid else grid)


class _FileBytes(object):
    """A TIFF file handed to the library without copying it: a path is read once, bytes and bytearray are used in
    place, any other bytes-like object is copied once."""

    def __init__(self, path_or_bytes):
        from .api import _JpegFile
        if isinstance(path_or_bytes, (str, os.PathLike)):
            with open(path_or_bytes, "rb") as f:
                path_or_bytes = f.read()
        elif not isinstance(path_or_bytes, (bytes, bytearray)):
            path_or_bytes = bytes(memoryview(path_or_bytes).cast("B"))
        self.data = path_or_bytes
        self.file = _JpegFile(path_or_bytes)


def _decode_device(f, t, device):
    """Image `t` (a TiffLayout of the file f, a _FileBytes) decoded on a GPU: torch CUDA float32 [H, W]."""
    import torch
    from .api import _jpeg_context
    dev = torch.device("cuda", int(device))
    out = torch.empty((t.height, t.width), dtype=torch.float32, device=dev)
    L = t.c_layout()
    ctx = _jpeg_context(int(device))
    torch.cuda.synchronize(dev)   # the output's allocation is ordered before the decode on the context's stream
    _lib.check(_lib.lib().amb_tiff_decode_device(ctx, C.c_void_p(f.file.ptr), f.file.size, C.byref(L), 0, t.height, 0,
                                                 t.width, C.c_void_p(out.data_ptr()), 4 * t.width), ctx)
    return out


def read_geotiff_device(path_or_bytes, band=0, overview=0, device=0):
    """read_geotiff on a GPU: (torch CUDA float32 [H, W], geotransform, EPSG code or None, no-data value or None), the
    array bit for bit read_geotiff(...)[0].astype(np.float32) (a NaN of a float64 file stays a NaN, its payload is not
    promised).  The file's chunks are inflated, unpredicted and converted on the device (convention in
    include/aerial_mapper_b200.h, amb_tiff_decode_device); the IFD is parsed here, with read_geotiff's ValueErrors.  A
    chunk that does not inflate raises AmbError(AMB_ERR_CORRUPT_DATA)."""
    f = _FileBytes(path_or_bytes)
    t = tiff_layout(f.data, band, overview)
    geo = t.georeferencing()
    return (_decode_device(f, t, device),) + geo
