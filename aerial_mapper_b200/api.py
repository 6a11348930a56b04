"""Python mirror of the reference's interface for the grid-mapping hot path, over the C ABI.

Same names, argument meaning and error behaviour as the reference's C++ classes, so the parity tests read like the
reference's callers (aerial_mapper_demos/src/dsm/main-dsm.cc:94-107,
src/ortho/main-ortho-backward-grid.cc:119-141, main-ortho-backward-grid-incremental.cc:99-163):

    settings = GridMapSettings(...);  map = AerialGridMap(settings)           # aerial-mapper-grid-map.h:23-54
    Dsm(DsmSettings(...), map.get_mutable()).process(point_cloud, map.get_mutable())     # dsm.h:25-47
    OrthoBackwardGrid(ncameras, OrthoSettings(...), map.get_mutable()).process(T_G_Bs, images, map.get_mutable())

The C++ drop-in headers with the literal reference signatures live in aerial_mapper_b200/shim/.

All compute happens in libaerial_mapper_b200.so on the GPU; there is no CPU path in this package.
"""
import ctypes as C
import os
import logging

import numpy as np

from . import _lib
from ._lib import AmbError, Camera, Geometry, LAYER_ID, LAYER_NAMES, check, lib

log = logging.getLogger("aerial_mapper_b200")

# Layers the hot path reads or writes (ortho-backward-grid.cc:133-138, dsm.cc:116).
HOT_LAYERS = ("ortho", "elevation", "elevation_angle", "observation_index", "colored_ortho")


class GridMapSettings(object):
    """grid_map::Settings (aerial-mapper-grid-map.h:23-29)."""

    def __init__(self, center_easting=0.0, center_northing=0.0, delta_easting=100.0, delta_northing=100.0,
                 resolution=1.0):
        self.center_easting = center_easting
        self.center_northing = center_northing
        self.delta_easting = delta_easting
        self.delta_northing = delta_northing
        self.resolution = resolution


class GridMap(object):
    """The slice of grid_map::GridMap the hot path uses: geometry + float32 column-major layers.

    `layers[name]` is a numpy float32 array of shape (rows, cols) in Fortran order — the memory layout of
    grid_map::Matrix (Eigen::MatrixXf): element (i, j) at i + j*rows, i <-> x / easting, j <-> y / northing.

    Host mode (default) keeps these arrays authoritative: every process() uploads what it reads and downloads what
    it writes, like the reference mutating the caller's map in place.  to_device() switches to resident mode: the
    layers live in HBM across process() calls (the incremental pipeline's access pattern) and come back with
    download().
    """

    def __init__(self, layer_names=LAYER_NAMES, pinned=False):
        self.layer_names = tuple(layer_names)
        self.pinned = bool(pinned)  # allocate the host layers in page-locked memory (full-rate PCIe copies)
        self._pinned_ptrs = []
        self.geometry = None
        self.layers = {}
        self.frame_id = ""
        self._ctx = None
        self._resident = False
        self._device = 0
        self._col_range = None

    # --- grid_map::GridMap surface used by the reference ---
    def setFrameId(self, frame_id):
        self.frame_id = frame_id

    def setGeometry(self, length, resolution, position=(0.0, 0.0)):
        g = Geometry()
        check(lib().amb_geometry_init(float(length[0]), float(length[1]), float(resolution), float(position[0]),
                                      float(position[1]), C.byref(g)))
        self.geometry = g
        self._free_pinned()
        self.layers = {}
        for name in self.layer_names:
            a = self._alloc_layer(g.rows, g.cols)
            a[...] = np.float32(np.nan)  # grid_map::GridMap::setGeometry -> clearAll()
            self.layers[name] = a
        self._release()

    def _alloc_layer(self, rows, cols):
        if not self.pinned:
            return np.empty((rows, cols), dtype=np.float32, order="F")
        p = C.c_void_p()
        nbytes = rows * cols * 4
        check(lib().amb_host_alloc(C.byref(p), nbytes))
        self._pinned_ptrs.append(p)
        buf = (C.c_float * (rows * cols)).from_address(p.value)
        return np.frombuffer(buf, dtype=np.float32).reshape((rows, cols), order="F")

    def _free_pinned(self):
        self.layers = {}
        for p in self._pinned_ptrs:
            lib().amb_host_free(p)
        self._pinned_ptrs = []

    def getSize(self):
        return (self.geometry.rows, self.geometry.cols)

    def getLength(self):
        return (self.geometry.length_x, self.geometry.length_y)

    def getResolution(self):
        return self.geometry.resolution

    def getPosition(self, index=None):
        if index is None:
            return (self.geometry.pos_x, self.geometry.pos_y)
        x, y = C.c_double(), C.c_double()
        check(lib().amb_geometry_position(C.byref(self.geometry), int(index[0]), int(index[1]), C.byref(x),
                                          C.byref(y)))
        return (x.value, y.value)

    def __getitem__(self, layer):
        return self.layers[layer]

    def __setitem__(self, layer, value):
        self.layers[layer][...] = value

    # --- device residency ---
    def context(self, device=None, col_range=None):
        if self._ctx is None:
            if device is not None:
                self._device = int(device)
            g = self.geometry
            c0, c1 = (0, g.cols) if col_range is None else col_range
            self._col_range = (int(c0), int(c1))
            ctx = C.c_void_p()
            check(lib().amb_create(C.byref(g), self._device, int(c0), int(c1), C.byref(ctx)))
            self._ctx = ctx
        return self._ctx

    def _slab(self, name):
        c0, c1 = self._col_range
        a = self.layers[name]
        assert a.dtype == np.float32 and a.flags.f_contiguous
        return a[:, c0:c1]  # contiguous in F order

    def upload(self, names=HOT_LAYERS):
        ctx = self.context()
        for name in names:
            slab = self._slab(name)
            check(lib().amb_upload_layer(ctx, LAYER_ID[name], slab.ctypes.data_as(C.c_void_p)), ctx)

    def download(self, names=HOT_LAYERS):
        ctx = self.context()
        for name in names:
            slab = self._slab(name)
            check(lib().amb_download_layer(ctx, LAYER_ID[name], slab.ctypes.data_as(C.c_void_p)), ctx)

    def download_async(self, names=HOT_LAYERS):
        """Enqueue device->host copies that overlap later work; sync() completes them (pinned layers recommended)."""
        ctx = self.context()
        for name in names:
            slab = self._slab(name)
            check(lib().amb_download_layer_async(ctx, LAYER_ID[name], slab.ctypes.data_as(C.c_void_p)), ctx)

    def set_mirrors(self, names=HOT_LAYERS, enable=True):
        """Register the host layers as mirrors (amb_set_host_mirror): process() streams every result layer back as
        soon as it is final, overlapping later stages; sync() completes the copies.  Use pinned layers."""
        ctx = self.context()
        # one-byte transport of `ortho` / `observation_index` (amb_set_host_mirror_compact; AMB_COMPACT_MIRRORS=0 turns it off)
        compact = os.environ.get("AMB_COMPACT_MIRRORS", "1") not in ("", "0")   # default on (exact-bits transport)
        for name in names:
            slab = self._slab(name)
            ptr = slab.ctypes.data_as(C.c_void_p) if enable else None
            check(lib().amb_set_host_mirror(ctx, LAYER_ID[name], ptr), ctx)
            if name in ("ortho", "observation_index"):
                check(lib().amb_set_host_mirror_compact(ctx, LAYER_ID[name], 1 if (enable and compact) else 0), ctx)

    def to_device(self, device=0, col_range=None, names=HOT_LAYERS):
        """Make the layers device-resident (uploads the current host values once)."""
        self._release()
        self.context(device, col_range)
        self.upload(names)
        self._resident = True
        return self

    def is_resident(self):
        return self._resident

    def sync(self):
        if self._ctx is not None:
            check(lib().amb_sync(self._ctx), self._ctx)

    # --- north-up raster export (convention: include/aerial_mapper_b200.h, amb_raster_format) ---
    def geotransform(self):
        """GDAL geotransform of the exported raster: (west, res, 0, north, 0, -res)."""
        gt = (C.c_double * 6)()
        check(lib().amb_raster_geotransform(C.byref(self.geometry), gt))
        return tuple(gt)

    def to_raster(self, name, fmt="f32", out=None):
        """The context's band of layer `name` as a north-up, row-major raster converted on the device: float32 or uint8
        [band_rows, rows], or uint8 [band_rows, rows, 3] (B, G, R) for "bgr8"; band_rows = col_end - col_begin, and image
        row r of the whole map is layer column r read backwards.  fmt: "f32", "gray8", "bgr8" or "mask8".  `out`: an
        optional C-contiguous array of that shape and dtype to write into (e.g. the context's rows of a full image, or
        page-locked memory)."""
        if not self._resident:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT,
                           "to_raster exports device-resident layers: call to_device() first")
        f = _lib.RASTER_FORMAT[fmt] if isinstance(fmt, str) else int(fmt)
        if f not in _lib.RASTER_BPP:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT, "raster format %r" % (fmt,))
        c0, c1 = self._col_range
        shape = (c1 - c0, self.geometry.rows) + ((3,) if f == _lib.RASTER_BGR8 else ())
        dtype = np.float32 if f == _lib.RASTER_F32 else np.uint8
        if out is None:
            out = np.empty(shape, dtype)
        elif out.shape != shape or out.dtype != dtype or not out.flags.c_contiguous:
            raise AmbError(_lib.AMB_ERR_SIZE_MISMATCH, "out must be C-contiguous %s %r" % (np.dtype(dtype).name, shape))
        ctx = self._ctx
        check(lib().amb_export_raster(ctx, LAYER_ID[name], f, out.ctypes.data_as(C.c_void_p)), ctx)
        return out

    def from_raster(self, name, band, geotransform, nodata=None, resample="bilinear"):
        """Resample a north-up float32 raster into the context's stripe of layer `name` on the device (convention:
        include/aerial_mapper_b200.h, amb_resample): band is float32 [H, W] with unit element stride (a row-sliced view
        is fine), geotransform its GDAL geotransform (west, res_x, 0, north, 0, -res_y) in the map's projected frame.
        NaN pixels, and pixels equal to `nodata` if given, are no-data; cells outside the raster or fed by no-data keep
        their value.  resample: "bilinear" or "nearest"; a raster on the map's own grid is copied bit for bit by both."""
        if not self._resident:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT,
                           "from_raster imports into device-resident layers: call to_device() first")
        r = _lib.RESAMPLE[resample] if isinstance(resample, str) else int(resample)
        a = np.asarray(band)
        if a.ndim != 2 or a.dtype != np.float32 or a.strides[1] != 4 or a.strides[0] < 4 * a.shape[1]:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT,
                           "band must be float32 [H, W] with unit element stride and increasing rows; got %s %r strides %r"
                           % (a.dtype, a.shape, a.strides))
        gt = (C.c_double * 6)(*[float(v) for v in geotransform])
        ctx = self._ctx
        check(lib().amb_import_raster(ctx, LAYER_ID[name], a.ctypes.data_as(C.c_void_p), a.shape[1], a.shape[0],
                                      a.strides[0], gt, 0 if nodata is None else 1,
                                      0.0 if nodata is None else float(nodata), r), ctx)

    def from_lonlat_raster(self, name, band, geotransform, map_epsg, nodata=None, resample="bilinear"):
        """from_raster of a longitude/latitude raster (WGS84, EPSG:4326; geotransform (lon0, dlon, 0, lat0, 0, -dlat) in
        degrees) into a map in the WGS84 UTM zone `map_epsg` (32601-32660 or 32701-32760): every cell is
        inverse-projected on the device, then resampled by from_raster's rule (convention: include/aerial_mapper_b200.h,
        amb_import_raster_lonlat).  Heights are imported as stored: no datum shift, no geoid correction."""
        if not self._resident:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT,
                           "from_lonlat_raster imports into device-resident layers: call to_device() first")
        r = _lib.RESAMPLE[resample] if isinstance(resample, str) else int(resample)
        a = np.asarray(band)
        if a.ndim != 2 or a.dtype != np.float32 or a.strides[1] != 4 or a.strides[0] < 4 * a.shape[1]:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT,
                           "band must be float32 [H, W] with unit element stride and increasing rows; got %s %r strides %r"
                           % (a.dtype, a.shape, a.strides))
        gt = (C.c_double * 6)(*[float(v) for v in geotransform])
        ctx = self._ctx
        check(lib().amb_import_raster_lonlat(ctx, LAYER_ID[name], a.ctypes.data_as(C.c_void_p), a.shape[1], a.shape[0],
                                             a.strides[0], gt, 0 if nodata is None else 1,
                                             0.0 if nodata is None else float(nodata), r, int(map_epsg)), ctx)

    def from_geotiff(self, name, path_or_bytes, band=0, overview=0, resample="bilinear", nodata="file", map_epsg=None):
        """from_raster of io.read_geotiff(path_or_bytes, band, overview) converted to float32, with its geotransform, bit
        for bit, decoded on the device: only the strips or tiles the context's stripe reads are copied and inflated
        (convention: include/aerial_mapper_b200.h, amb_import_tiff).  nodata: by default the file's GDAL_NODATA; None
        for none.  A chunk of that window that does not inflate raises AmbError(AMB_ERR_CORRUPT_DATA) and the layer is
        not written.
        map_epsg: None reads the file as in the map's frame, whatever its EPSG code.  Given (the map's UTM zone, e.g.
        32632), a file in EPSG:4326 is imported as from_lonlat_raster of its array, one in map_epsg as above, and any
        other file (another code, or none) raises ValueError."""
        if not self._resident:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT,
                           "from_geotiff imports into device-resident layers: call to_device() first")
        from . import io
        r = _lib.RESAMPLE[resample] if isinstance(resample, str) else int(resample)
        f = io._FileBytes(path_or_bytes)
        t = io.tiff_layout(f.data, band, overview)
        gt, file_epsg, file_nodata = t.georeferencing()
        lonlat = _lonlat_source(file_epsg, map_epsg)
        if isinstance(nodata, str) and nodata == "file":
            nodata = file_nodata
        L = t.c_layout()
        ctx = self._ctx
        args = (ctx, LAYER_ID[name], C.c_void_p(f.file.ptr), f.file.size, C.byref(L), (C.c_double * 6)(*gt),
                0 if nodata is None else 1, 0.0 if nodata is None else float(nodata), r)
        if lonlat:
            check(lib().amb_import_tiff_lonlat(*(args + (int(map_epsg),))), ctx)
        else:
            check(lib().amb_import_tiff(*args), ctx)

    def to_jpeg(self, name, quality=95, sampling="420", restart_interval=0, fmt=None):
        """The context's band of layer `name` as a baseline JPEG file (bytes), exported and encoded on the device
        (convention: include/aerial_mapper_b200.h, amb_jpeg_sampling), byte for byte cv2.imencode(".jpg", band, params)
        of the band to_raster(name, fmt) returns.  fmt: "gray8" or "bgr8"; by default "gray8" for `ortho` and "bgr8"
        for `colored_ortho`, required for any other layer.  sampling: "420" or "444"; restart_interval in MCUs."""
        if not self._resident:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT, "to_jpeg exports device-resident layers: call to_device() first")
        if fmt is None:
            fmt = {"ortho": "gray8", "colored_ortho": "bgr8"}.get(name)
            if fmt is None:
                raise ValueError("to_jpeg(%r): give fmt='gray8' or fmt='bgr8' for this layer" % (name,))
        if fmt not in ("gray8", "bgr8"):
            raise ValueError("to_jpeg: fmt must be 'gray8' or 'bgr8', got %r" % (fmt,))
        f = _lib.RASTER_FORMAT[fmt]
        channels = 3 if f == _lib.RASTER_BGR8 else 1
        args = _jpeg_args(self.geometry.rows, self._col_range[1] - self._col_range[0], channels, quality, sampling,
                          restart_interval)
        ctx = self._ctx
        return _jpeg_call(lambda buf, cap, size: lib().amb_export_jpeg(ctx, LAYER_ID[name], f, *args[3:], buf, cap, size),
                          args, ctx)

    def to_geotiff(self, path, name, fmt=None, epsg=32632, nodata=None, rows_per_strip=None):
        """Writes the context's band of layer `name` to `path` as a Deflate-compressed GeoTIFF, predicted and compressed
        on the device (convention: include/aerial_mapper_b200.h, amb_deflate_strips_device); reading it back gives
        to_raster(name, fmt) bit for bit.  fmt: "f32", "gray8", "bgr8" or "mask8"; by default "f32" for `elevation`,
        "gray8" for `ortho` and "bgr8" for `colored_ortho`, required for any other layer.  The geotransform is the
        band's own: a stripe context writes its rows of the map as a file of their own.  nodata: GDAL_NODATA, e.g.
        "nan".  rows_per_strip: by default libtiff's 8 KiB strips, max(1, 8192 // row_bytes)."""
        if not self._resident:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT,
                           "to_geotiff exports device-resident layers: call to_device() first")
        if fmt is None:
            fmt = {"elevation": "f32", "ortho": "gray8", "colored_ortho": "bgr8"}.get(name)
            if fmt is None:
                raise ValueError("to_geotiff(%r): give fmt='f32', 'gray8', 'bgr8' or 'mask8' for this layer" % (name,))
        if fmt not in _lib.RASTER_FORMAT:
            raise ValueError("to_geotiff: fmt must be 'f32', 'gray8', 'bgr8' or 'mask8', got %r" % (fmt,))
        f = _lib.RASTER_FORMAT[fmt]
        c0, c1 = self._col_range
        width, height = self.geometry.rows, c1 - c0
        rps = _deflate_rows(width * _lib.RASTER_BPP[f], height, rows_per_strip)
        ctx = self._ctx
        data, counts = _deflate_call(
            lambda buf, cap, size, sb: lib().amb_export_deflate_strips(ctx, LAYER_ID[name], f, rps, buf, cap, size, sb),
            width, height, f, rps, ctx)
        gt = list(self.geotransform())
        gt[3] += c0 * gt[5]        # the band's north edge
        from . import io
        io.write_geotiff_strips(path, data, counts, width, height, fmt, rps, gt, epsg, nodata)

    def to_cog(self, path, name, fmt=None, epsg=32632, nodata=None, tile_size=512, compress="deflate", quality=75,
               sampling="420", mask=None):
        """Writes the context's band of layer `name` to `path` as a Cloud-Optimized GeoTIFF: T x T Deflate tiles with
        internal overviews halved until one fits a tile, pyramid, tiles and compression on the device (convention:
        include/aerial_mapper_b200.h, amb_cog_tiles_device; layout: io.write_cog).  Level 0 reads back as to_raster(name,
        fmt) bit for bit.  fmt and the geotransform as to_geotiff.  nodata must agree with the overviews: "nan" (or NaN)
        for "f32", 0 for "mask8", none for "gray8" and "bgr8".  tile_size: a multiple of 16 in [16, 4096].

        compress="jpeg": JPEG tiles in YCbCr ("bgr8") or gray ("gray8") at `quality` (1..100) and `sampling` ("420" or
        "444"), encoded on the device (amb_cog_jpeg_tiles_device), GDAL's COMPRESS=JPEG layout; no nodata.
        mask: the name of a layer whose "mask8" export (valid where the layer is not NaN, e.g. "observation_index")
        becomes the file's internal 1-bit mask (amb_cog_mask_tiles_device), for "gray8" and "bgr8" with either
        compression: unobserved cells read as no-data instead of image content."""
        if not self._resident:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT, "to_cog exports device-resident layers: call to_device() first")
        if fmt is None:
            fmt = {"elevation": "f32", "ortho": "gray8", "colored_ortho": "bgr8"}.get(name)
            if fmt is None:
                raise ValueError("to_cog(%r): give fmt='f32', 'gray8', 'bgr8' or 'mask8' for this layer" % (name,))
        if fmt not in _lib.RASTER_FORMAT:
            raise ValueError("to_cog: fmt must be 'f32', 'gray8', 'bgr8' or 'mask8', got %r" % (fmt,))
        if compress not in ("deflate", "jpeg"):
            raise ValueError("to_cog: compress must be 'deflate' or 'jpeg', got %r" % (compress,))
        jpeg = compress == "jpeg"
        if (jpeg or mask is not None) and fmt not in ("gray8", "bgr8"):
            raise ValueError("to_cog: %s is for fmt 'gray8' and 'bgr8' only, got %r" % ("JPEG" if jpeg else "mask", fmt))
        if jpeg and nodata is not None:
            raise ValueError("to_cog: a JPEG COG takes no nodata (JPEG is lossy): give mask= instead")
        if mask is not None and mask not in LAYER_ID:
            raise ValueError("to_cog: mask must be a layer name, got %r" % (mask,))
        from . import io
        io.cog_nodata(fmt, nodata)
        tile = _cog_tile(tile_size)
        f = _lib.RASTER_FORMAT[fmt]
        c0, c1 = self._col_range
        width, height = self.geometry.rows, c1 - c0
        ctx = self._ctx
        tables = None
        if jpeg:
            q, s = _cog_jpeg_args(quality, sampling)
            data, counts = _cog_jpeg_call(
                lambda buf, cap, size, tb: lib().amb_export_cog_jpeg_tiles(ctx, LAYER_ID[name], f, tile, q, s, buf, cap,
                                                                           size, tb),
                width, height, f, tile, q, s, ctx)
            tables = cog_jpeg_tables(fmt, quality)
        else:
            data, counts = _cog_call(
                lambda buf, cap, size, tb: lib().amb_export_cog_tiles(ctx, LAYER_ID[name], f, tile, buf, cap, size, tb),
                width, height, f, tile, ctx)
        masks = None
        if mask is not None:
            masks = _cog_call(
                lambda buf, cap, size, tb: lib().amb_export_cog_mask_tiles(ctx, LAYER_ID[mask], tile, buf, cap, size, tb),
                width, height, _lib.RASTER_MASK8, tile, ctx, cap=lib().amb_cog_mask_max_size(width, height, tile))
        gt = list(self.geotransform())
        gt[3] += c0 * gt[5]        # the band's north edge
        io.write_cog(path, data, counts, width, height, fmt, tile, gt, epsg, nodata, compress=compress,
                     jpeg_tables=tables, sampling=sampling, mask=masks)

    def timings(self):
        t = _lib.Timings()
        check(lib().amb_get_timings(self.context(), C.byref(t)), self._ctx)
        return t.as_dict()

    def _release(self):
        if self._ctx is not None:
            lib().amb_destroy(self._ctx)
            self._ctx = None
        self._resident = False

    def __del__(self):
        try:
            self._release()
            self._free_pinned()
        except Exception:
            pass


def _lonlat_source(file_epsg, map_epsg):
    """Whether from_geotiff(map_epsg=...) reads a file of EPSG code file_epsg as a longitude/latitude raster."""
    if map_epsg is None:
        return False
    map_epsg = int(map_epsg)
    if not (32601 <= map_epsg <= 32660 or 32701 <= map_epsg <= 32760):
        raise ValueError("from_geotiff: map_epsg %d is not a WGS84 UTM zone (32601-32660, 32701-32760)" % map_epsg)
    if file_epsg == 4326:
        return True
    if file_epsg == map_epsg:
        return False
    raise ValueError("from_geotiff: the file is in EPSG:%s, the map in EPSG:%d; only EPSG:4326 files or files in the "
                     "map's own zone are imported" % ("none" if file_epsg is None else file_epsg, map_epsg))


class AerialGridMap(object):
    """grid_map::AerialGridMap (aerial-mapper-grid-map.cc:23-49) without the ROS publisher."""

    def __init__(self, settings, pinned=False, layer_names=LAYER_NAMES):
        self.settings_ = settings
        self.map_ = GridMap(layer_names, pinned=pinned)  # :25-28
        self.map_.setFrameId("world")
        self.map_.setGeometry((settings.delta_easting, settings.delta_northing), settings.resolution,
                              (settings.center_easting, settings.center_northing))  # :30-33
        self.reset()

    INITIAL_VALUES = {"ortho": 255.0, "elevation": np.nan, "elevation_angle": 0.0,
                      "elevation_angle_first_view": np.nan, "num_observations": 0.0, "observation_index": np.nan,
                      "observation_index_first": np.nan, "delta": np.nan, "colored_ortho": np.nan}

    def reset(self):
        """The setConstant() calls of AerialGridMap::initialize (aerial-mapper-grid-map.cc:40-48)."""
        for name in self.map_.layer_names:
            self.map_[name] = self.INITIAL_VALUES[name]

    def getMutable(self):
        return self.map_

    get_mutable = getMutable


class DsmSettings(object):
    """dsm::Settings (dsm.h:25-32).  interpolation_radius is an int compared against SQUARED distances (m^2)."""

    def __init__(self, interpolation_radius=1, adaptive_interpolation=False, center_easting=0.0,
                 center_northing=0.0, use_multi_threads=True):
        self.interpolation_radius = int(interpolation_radius)  # `int interpolation_radius = 1.0;`
        self.adaptive_interpolation = adaptive_interpolation   # never read by the reference (dsm.cc)
        self.center_easting = center_easting
        self.center_northing = center_northing
        self.use_multi_threads = use_multi_threads             # both reference twins compute the same values


class Dsm(object):
    """dsm::Dsm (dsm.h:34-72)."""

    def __init__(self, settings, map):
        if map is None:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT, "CHECK(map) (dsm.cc:22)")
        self.settings_ = settings
        self.debug = False
        self.last_debug = None
        # arithmetic of the gather's weights and sums (amb_dsm_set_precision): None = the library default ("f32":
        # float32 weights and sums, neighbour sets exact; the environment variable AMB_DSM_PRECISION=f64|f32, read by
        # the library itself, overrides that default process-wide — how the tests run both), or "f32" / "f64"
        self.precision = None
        # chunked evaluation + early mirroring of finished columns (amb_dsm_set_stream_chunks); 1 = off, default 4
        self.stream_chunks = max(1, int(os.environ.get("AMB_DSM_STREAM_CHUNKS", "4") or 4))

    def _configure(self, ctx):
        """This Dsm's debug, stream_chunks and precision onto the map's context, before each of its calls."""
        check(lib().amb_dsm_enable_debug(ctx, 1 if self.debug else 0), ctx)
        check(lib().amb_dsm_set_stream_chunks(ctx, int(self.stream_chunks)), ctx)
        if self.precision is not None:
            check(lib().amb_dsm_set_precision(ctx, _lib.DSM_F32 if self.precision == "f32" else _lib.DSM_F64), ctx)

    def process(self, point_cloud, map):
        """point_cloud: float64 [n, 3] (the AoS layout of std::vector<Eigen::Vector3d>).  Mutates map['elevation']."""
        pc = np.ascontiguousarray(point_cloud, dtype=np.float64)
        n = pc.size // 3
        if n == 0:
            log.warning("Passed empty point cloud to DSM module")  # dsm.cc:189-192
            return
        if map is None:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT, "CHECK(map) (dsm.cc:194)")
        ctx = map.context()
        s = self.settings_
        if not map.is_resident():
            map.upload(("elevation",))
        self._configure(ctx)
        check(lib().amb_dsm_process(ctx, pc.ctypes.data_as(C.c_void_p), n, int(s.interpolation_radius),
                                    float(s.center_easting), float(s.center_northing)), ctx)
        self._fetch_debug(map)
        if not map.is_resident():
            map.download(("elevation",))

    def process_device(self, d_xyz, n, map, d_ids=None):
        """Points already in HBM (device pointer as int); asynchronous — map.sync() before reading results.
        d_ids: optional device pointer to one uint64 id per point (a sharded cloud: global point ids)."""
        if n == 0:
            log.warning("Passed empty point cloud to DSM module")
            return
        ctx = map.context()
        s = self.settings_
        self._configure(ctx)
        if d_ids is None:
            check(lib().amb_dsm_process_device(ctx, C.c_void_p(int(d_xyz)), int(n), int(s.interpolation_radius),
                                               float(s.center_easting), float(s.center_northing)), ctx)
        else:
            check(lib().amb_dsm_process_device_ids(ctx, C.c_void_p(int(d_xyz)), C.c_void_p(int(d_ids)), int(n),
                                                   int(s.interpolation_radius), float(s.center_easting),
                                                   float(s.center_northing)), ctx)

    def process_sharded_device(self, d_xyz, d_ids, n_local, map, halo_capacity):
        """A cloud sharded by stripe, the exchange step included (amb_dsm_process_sharded_device): this rank's points
        and global ids (device pointers) -> border halo compaction -> one NCCL all-gather inside the library -> the
        stripe's elevation.  Collective over the communicator the map's context joined (sharding.init_comm);
        asynchronous — map.sync() before reading results."""
        ctx = map.context()
        s = self.settings_
        self._configure(ctx)
        check(lib().amb_dsm_process_sharded_device(ctx, C.c_void_p(int(d_xyz)), C.c_void_p(int(d_ids)), int(n_local),
                                                   int(s.interpolation_radius), float(s.center_easting),
                                                   float(s.center_northing), int(halo_capacity)), ctx)

    def process_sharded(self, point_cloud, ids, map, halo_capacity):
        """Same with this rank's points (float64 [n, 3]) and global ids (uint64 [n]) in host memory."""
        pc = np.ascontiguousarray(point_cloud, dtype=np.float64)
        idv = np.ascontiguousarray(ids, dtype=np.uint64)
        n = pc.size // 3
        ctx = map.context()
        s = self.settings_
        self._configure(ctx)
        check(lib().amb_dsm_process_sharded(ctx, pc.ctypes.data_as(C.c_void_p), idv.ctypes.data_as(C.c_void_p), n,
                                            int(s.interpolation_radius), float(s.center_easting),
                                            float(s.center_northing), int(halo_capacity)), ctx)

    def _fetch_debug(self, map):
        if not self.debug:
            self.last_debug = None
            return
        c0, c1 = map._col_range
        rows = map.geometry.rows
        cnt = np.empty((rows, c1 - c0), dtype=np.int32, order="F")
        lvl = np.empty((rows, c1 - c0), dtype=np.int8, order="F")
        check(lib().amb_dsm_download_debug(map.context(), cnt.ctypes.data_as(C.c_void_p),
                                           lvl.ctypes.data_as(C.c_void_p)), map.context())
        self.last_debug = (cnt, lvl)


def dsm_thresholds(interpolation_radius):
    buf = (C.c_double * 64)()
    n = lib().amb_dsm_thresholds(int(interpolation_radius), C.cast(buf, C.c_void_p), 64)
    if n < 0:
        raise AmbError(n)
    return [buf[k] for k in range(n)]


class OrthoSettings(object):
    """ortho::Settings of ortho-backward-grid.h:32-41.  Only colored_ortho affects results."""

    def __init__(self, show_orthomosaic_opencv=True, save_orthomosaic_jpg=True, orthomosaic_jpg_filename="",
                 orthomosaic_elevation_m=0.0, use_digital_elevation_map=True, colored_ortho=False,
                 use_multi_threads=True):
        self.show_orthomosaic_opencv = show_orthomosaic_opencv
        self.save_orthomosaic_jpg = save_orthomosaic_jpg
        self.orthomosaic_jpg_filename = orthomosaic_jpg_filename
        self.orthomosaic_elevation_m = orthomosaic_elevation_m
        self.use_digital_elevation_map = use_digital_elevation_map
        self.colored_ortho = colored_ortho
        self.use_multi_threads = use_multi_threads


class NCamera(object):
    """The part of aslam::NCamera the path uses: camera 0 (pinhole + distortion) and T_C_B(0)
    (ortho-backward-grid.cc:131,232)."""

    def __init__(self, width, height, fu, fv, cu, cv, dist_type=_lib.DIST_NONE, dist=(0.0, 0.0, 0.0, 0.0),
                 q_C_B=(1.0, 0.0, 0.0, 0.0), t_C_B=(0.0, 0.0, 0.0)):
        cam = Camera()
        cam.width, cam.height = int(width), int(height)
        cam.fu, cam.fv, cam.cu, cam.cv = float(fu), float(fv), float(cu), float(cv)
        cam.dist_type = int(dist_type)
        cam.dist = (C.c_double * 4)(*[float(d) for d in dist])
        cam.q_C_B = (C.c_double * 4)(*[float(d) for d in q_C_B])
        cam.t_C_B = (C.c_double * 3)(*[float(d) for d in t_C_B])
        self.camera = cam

    def imageWidth(self):
        return self.camera.width

    def imageHeight(self):
        return self.camera.height


class OrthoBackwardGrid(object):
    """ortho::OrthoBackwardGrid (ortho-backward-grid.h:43-71)."""

    def __init__(self, ncameras, settings, map=None):
        if ncameras is None:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT, "CHECK(ncameras_) (ortho-backward-grid.cc:27)")
        self.ncameras_ = ncameras
        self.settings_ = settings
        self.brute_force = False
        # per-tile dominance cull of the frame list (amb_ortho_set_dominance_cull; same output bits, fewer frames per
        # tile): on by default, AMB_ORTHO_DOMINANCE=0 selects the plain conservative list
        self.dominance_cull = os.environ.get("AMB_ORTHO_DOMINANCE", "1") not in ("", "0")

    def _layers_written(self):
        out = "colored_ortho" if self.settings_.colored_ortho else "ortho"
        return ("elevation_angle", "observation_index", out)

    def _configure(self, ctx):
        """This grid's brute_force and dominance_cull onto the map's context, before each of its calls."""
        check(lib().amb_ortho_set_brute_force(ctx, 1 if self.brute_force else 0), ctx)
        check(lib().amb_ortho_set_dominance_cull(ctx, 1 if self.dominance_cull else 0), ctx)

    @staticmethod
    def _poses(T_G_Bs, frames, empty=_lib.AMB_ERR_EMPTY):
        """T_G_Bs as float64 [n, 7] and n, one frame per pose (ortho-backward-grid.cc:225-226)."""
        T = np.ascontiguousarray(T_G_Bs, dtype=np.float64).reshape(-1, 7)
        n = T.shape[0]
        if n == 0:
            raise AmbError(empty, "CHECK(!T_G_Bs.empty()) (ortho-backward-grid.cc:225)")
        if n != len(frames):
            raise AmbError(_lib.AMB_ERR_SIZE_MISMATCH,
                           "CHECK(T_G_Bs.size() == images.size()) (ortho-backward-grid.cc:226)")
        return T, n

    def process(self, T_G_Bs, images, map):
        """T_G_Bs: float64 [n, 7] rows x y z qw qx qy qz; images: n uint8 arrays [H, W] (gray) or [H, W, 3] (BGR)."""
        T, n = self._poses(T_G_Bs, images)
        if map is None:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT, "CHECK(map) (ortho-backward-grid.cc:227)")
        colored = bool(self.settings_.colored_ortho)
        channels = 3 if colored else 1
        cam = self.ncameras_.camera
        imgs = []
        for im in images:
            im = np.ascontiguousarray(im, dtype=np.uint8)
            ok = im.shape[:2] == (cam.height, cam.width) and (
                (im.ndim == 3 and im.shape[2] == 3) if colored else im.ndim == 2)
            if not ok:
                raise AmbError(_lib.AMB_ERR_SIZE_MISMATCH, "image shape %r" % (im.shape,))
            imgs.append(im)
        row_step = cam.width * channels
        ptrs = (C.c_void_p * n)(*[im.ctypes.data for im in imgs])
        ctx = map.context()
        if not map.is_resident():
            map.upload(("elevation",) + self._layers_written())
        self._configure(ctx)
        check(lib().amb_ortho_process(ctx, C.byref(cam), T.ctypes.data_as(C.c_void_p), C.cast(ptrs, C.c_void_p), n,
                                      channels, row_step, 1 if colored else 0), ctx)
        if not map.is_resident():
            map.download(self._layers_written())

    def process_jpeg(self, T_G_Bs, jpeg_files, map):
        """process() with the frames as JPEG files (a sequence of bytes-like objects, e.g. io.read_jpeg_files) in place
        of decoded images: the frames that contribute are decoded on the device, pixel for pixel what cv2.imread
        returns (amb_ortho_process_jpeg).  A corrupt scan of a contributing frame raises AmbError(AMB_ERR_CORRUPT_DATA)
        after elevation_angle and observation_index have been written; the ortho layer is then left as it was."""
        T, n = self._poses(T_G_Bs, jpeg_files)
        if map is None:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT, "CHECK(map) (ortho-backward-grid.cc:227)")
        files = [_JpegFile(f) for f in jpeg_files]   # no copy of the files' bytes
        colored = bool(self.settings_.colored_ortho)
        ptrs = (C.c_void_p * n)(*[f.ptr for f in files])
        sizes = (C.c_size_t * n)(*[f.size for f in files])
        ctx = map.context()
        if not map.is_resident():
            map.upload(("elevation",) + self._layers_written())
        self._configure(ctx)
        st = lib().amb_ortho_process_jpeg(ctx, C.byref(self.ncameras_.camera), T.ctypes.data_as(C.c_void_p), ptrs,
                                          sizes, n, 1 if colored else 0)
        if st == _lib.AMB_ERR_CORRUPT_DATA and not map.is_resident():
            map.download(self._layers_written()[:2])
        check(st, ctx)
        if not map.is_resident():
            map.download(self._layers_written())

    def process_device(self, T_G_Bs, d_image_ptrs, row_step, map):
        """Frames already in HBM: d_image_ptrs is a sequence of device pointers (ints).  Asynchronous."""
        T, n = self._poses(T_G_Bs, d_image_ptrs, empty=_lib.AMB_ERR_SIZE_MISMATCH)
        colored = bool(self.settings_.colored_ortho)
        ptrs = (C.c_void_p * n)(*[int(p) for p in d_image_ptrs])
        ctx = map.context()
        self._configure(ctx)
        check(lib().amb_ortho_process_device(ctx, C.byref(self.ncameras_.camera), T.ctypes.data_as(C.c_void_p),
                                             C.cast(ptrs, C.c_void_p), n, 3 if colored else 1, int(row_step),
                                             1 if colored else 0), ctx)


class OrthoFromPclSettings(object):
    """ortho::Settings of ortho-from-pcl.h:28-35 ("next" row N1)."""

    def __init__(self, show_orthomosaic_opencv=False, interpolation_radius=2, use_adaptive_interpolation=False,
                 save_orthomosaic_jpg=False, orthomosaic_jpg_filename=""):
        self.show_orthomosaic_opencv = show_orthomosaic_opencv
        self.interpolation_radius = int(interpolation_radius)
        self.use_adaptive_interpolation = use_adaptive_interpolation
        self.save_orthomosaic_jpg = save_orthomosaic_jpg
        self.orthomosaic_jpg_filename = orthomosaic_jpg_filename


class OrthoFromPcl(object):
    """ortho::OrthoFromPcl (ortho-from-pcl.h:37-52): IDW of point intensities into map['ortho']."""

    def __init__(self, settings):
        self.settings_ = settings

    def process(self, pointcloud, intensities, map):
        pc = np.ascontiguousarray(pointcloud, dtype=np.float64)
        n = pc.size // 3
        if n == 0:
            raise AmbError(_lib.AMB_ERR_EMPTY, "CHECK(!pointcloud.empty()) (ortho-from-pcl.cc:23)")
        if map is None:
            raise AmbError(_lib.AMB_ERR_INVALID_ARGUMENT, "CHECK(map) (ortho-from-pcl.cc:24)")
        inten = np.ascontiguousarray(intensities, dtype=np.int32)
        if inten.size < n:
            raise AmbError(_lib.AMB_ERR_SIZE_MISMATCH, "CHECK(i < intensities.size()) (ortho-from-pcl.cc:32)")
        ctx = map.context()
        s = self.settings_
        if not map.is_resident():
            map.upload(("ortho",))
        check(lib().amb_ortho_from_pcl_process(ctx, pc.ctypes.data_as(C.c_void_p), inten.ctypes.data_as(C.c_void_p),
                                               n, int(s.interpolation_radius),
                                               1 if s.use_adaptive_interpolation else 0), ctx)
        if not map.is_resident():
            map.download(("ortho",))

    def process_device(self, d_xyz, d_intensities, n, map, d_ids=None):
        """Points (float64 [n, 3]) and intensities (int32 [n]) already in HBM (device pointers as ints); asynchronous —
        map.sync() before reading results.  d_ids: optional device pointer to one uint64 global id per point (a sharded
        cloud), the canonical summation order instead of the array position."""
        if n == 0:
            raise AmbError(_lib.AMB_ERR_EMPTY, "CHECK(!pointcloud.empty()) (ortho-from-pcl.cc:23)")
        ctx = map.context()
        s = self.settings_
        adaptive = 1 if s.use_adaptive_interpolation else 0
        if d_ids is None:
            check(lib().amb_ortho_from_pcl_process_device(ctx, C.c_void_p(int(d_xyz)), C.c_void_p(int(d_intensities)),
                                                          int(n), int(s.interpolation_radius), adaptive), ctx)
        else:
            check(lib().amb_ortho_from_pcl_process_device_ids(ctx, C.c_void_p(int(d_xyz)),
                                                              C.c_void_p(int(d_intensities)), C.c_void_p(int(d_ids)),
                                                              int(n), int(s.interpolation_radius), adaptive), ctx)

    def _no_adaptive_when_sharded(self):
        if self.settings_.use_adaptive_interpolation:
            raise AmbError(_lib.AMB_ERR_UNSUPPORTED,
                           "adaptive interpolation needs the whole cloud, which no rank of a sharded cloud holds")

    def process_sharded_device(self, d_xyz, d_intensities, d_ids, n_local, map, halo_capacity):
        """A cloud sharded by stripe, the exchange step included (amb_ortho_from_pcl_process_sharded_device): this
        rank's points, intensities and global ids (device pointers) -> the stripe's `ortho`.  Collective over the
        communicator the map's context joined (sharding.init_comm); asynchronous — map.sync() before reading results."""
        self._no_adaptive_when_sharded()
        ctx = map.context()
        check(lib().amb_ortho_from_pcl_process_sharded_device(ctx, C.c_void_p(int(d_xyz)), C.c_void_p(int(d_intensities)),
                                                              C.c_void_p(int(d_ids)), int(n_local),
                                                              int(self.settings_.interpolation_radius),
                                                              int(halo_capacity)), ctx)

    def process_sharded(self, pointcloud, intensities, ids, map, halo_capacity):
        """Same with this rank's points (float64 [n, 3]), intensities (int32 [n]) and global ids (uint64 [n]) in host
        memory."""
        self._no_adaptive_when_sharded()
        pc = np.ascontiguousarray(pointcloud, dtype=np.float64)
        n = pc.size // 3
        inten = np.ascontiguousarray(intensities, dtype=np.int32)
        idv = np.ascontiguousarray(ids, dtype=np.uint64)
        if inten.size < n or idv.size < n:
            raise AmbError(_lib.AMB_ERR_SIZE_MISMATCH, "one intensity and one id per point")
        ctx = map.context()
        check(lib().amb_ortho_from_pcl_process_sharded(ctx, pc.ctypes.data_as(C.c_void_p),
                                                       inten.ctypes.data_as(C.c_void_p), idv.ctypes.data_as(C.c_void_p),
                                                       n, int(self.settings_.interpolation_radius),
                                                       int(halo_capacity)), ctx)


K_MAX_INVALID_DISPARITY = 1  # stereo::Densifier::kMaxInvalidDisparity (densifier.h:49)


def compute_point_cloud(disparity_map, image_left, K, baseline, R_G_C, t_G_C1, device=0,
                        max_invalid_disparity=K_MAX_INVALID_DISPARITY):
    """stereo::Densifier::computePointCloud (densifier.cpp:25-108; "next" row N3): disparity map (float32 [H, W]) +
    left rectified image (uint8 [H, W]) -> (point_cloud_eigen float64 [n, 3], point_cloud_intensities int32 [n]) in
    raster order.  K is the 3x3 camera matrix of the rectified pair (or (fx, fy, cx, cy))."""
    disp = np.ascontiguousarray(disparity_map, dtype=np.float32)
    img = np.ascontiguousarray(image_left, dtype=np.uint8)
    h, w = disp.shape
    if img.shape != (h, w):
        raise AmbError(_lib.AMB_ERR_SIZE_MISMATCH, "CHECK_EQ(image_resolution_, disparity_map.size())")
    K = np.asarray(K, dtype=np.float64)
    k4 = np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]]) if K.shape == (3, 3) else K.reshape(4).copy()
    R = np.ascontiguousarray(R_G_C, dtype=np.float64).reshape(9)
    t = np.ascontiguousarray(t_G_C1, dtype=np.float64).reshape(3)
    cap = h * w
    xyz = np.empty((cap, 3), dtype=np.float64)
    inten = np.empty(cap, dtype=np.int32)
    n = C.c_size_t(0)
    check(lib().amb_stereo_reproject(int(device), disp.ctypes.data_as(C.c_void_p), w, img.ctypes.data_as(C.c_void_p),
                                     w, w, h, k4.ctypes.data_as(C.c_void_p), float(baseline),
                                     R.ctypes.data_as(C.c_void_p), t.ctypes.data_as(C.c_void_p),
                                     float(max_invalid_disparity), xyz.ctypes.data_as(C.c_void_p),
                                     inten.ctypes.data_as(C.c_void_p), cap, C.byref(n)))
    return xyz[:n.value].copy(), inten[:n.value].copy()


def rectify_stereo_setup(K, R_G_C1, R_G_C2, t_G_C1, t_G_C2):
    """Host half of stereo::Rectifier::rectifyStereoPair (rectifier.cpp:43-79; "next" row N3): Fusiello's compact
    rectification.  Returns (baseline, R_G_C_rect float64 [3, 3], T1_inv float32 [3, 3], T2_inv float32 [3, 3])."""
    a = [np.ascontiguousarray(m, dtype=np.float64).reshape(n) for m, n in
         ((K, 9), (R_G_C1, 9), (R_G_C2, 9), (t_G_C1, 3), (t_G_C2, 3))]
    baseline = C.c_double(0.0)
    R = np.zeros(9, np.float64)
    T1 = np.zeros(9, np.float32)
    T2 = np.zeros(9, np.float32)
    p = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
    check(lib().amb_stereo_rectify_setup(p(a[0]), p(a[1]), p(a[2]), p(a[3]), p(a[4]), C.byref(baseline), p(R), p(T1),
                                         p(T2)))
    return baseline.value, R.reshape(3, 3), T1.reshape(3, 3), T2.reshape(3, 3)


def rectify_stereo_maps(T1_inv, T2_inv, width, height, device=0):
    """Device half (rectifier.cpp:80-104): the four CV_32FC1 rectification maps cv::remap consumes.
    Returns (map_rectify_1_x, map_rectify_1_y, map_rectify_2_x, map_rectify_2_y), float32 [H, W] each."""
    T1 = np.ascontiguousarray(T1_inv, dtype=np.float32).reshape(9)
    T2 = np.ascontiguousarray(T2_inv, dtype=np.float32).reshape(9)
    maps = [np.empty((int(height), int(width)), np.float32) for _ in range(4)]
    p = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
    check(lib().amb_stereo_rectify_maps(int(device), p(T1), p(T2), int(width), int(height), int(width), p(maps[0]),
                                        p(maps[1]), p(maps[2]), p(maps[3])))
    return tuple(maps)


# ---- baseline JPEG (amb_jpeg_encode_device, amb_export_jpeg) ----------------------------------------------------------
JPEG_SAMPLING = {"420": 0, "444": 1}


def _jpeg_args(width, height, channels, quality, sampling, restart_interval):
    """Checks the supported parameter set (ValueError otherwise); returns the C arguments."""
    if sampling not in JPEG_SAMPLING:
        raise ValueError("JPEG sampling must be '420' or '444', got %r" % (sampling,))
    for what, v, lo, hi in (("quality", quality, 1, 100), ("restart_interval", restart_interval, 0, 65535),
                            ("width", width, 1, 65535), ("height", height, 1, 65535)):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not lo <= v <= hi:
            raise ValueError("JPEG %s must be an integer in [%d, %d], got %r" % (what, lo, hi, v))
    return (int(width), int(height), channels, int(quality), JPEG_SAMPLING[sampling], int(restart_interval))


def _jpeg_call(call, args, ctx):
    """Runs `call(buffer, capacity, size)`, first with a buffer the size of the raw image, again at the size the library
    reports if the file is larger (incompressible content); returns the file's bytes."""
    width, height, channels = args[:3]
    cap = width * height * channels + 4096
    for _ in range(2):
        buf = np.empty(cap, np.uint8)
        size = C.c_size_t(0)
        st = call(buf.ctypes.data_as(C.c_void_p), cap, C.byref(size))
        if st == _lib.AMB_ERR_SIZE_MISMATCH and size.value > cap:
            cap = size.value
            continue
        check(st, ctx)
        return buf[:size.value].tobytes()
    raise AmbError(_lib.AMB_ERR_SIZE_MISMATCH, "JPEG size changed between two encodes of the same image")


_jpeg_contexts = {}


def _jpeg_context(device):
    """A context per device for encode_jpeg and deflate_strips: only its stream and its scratch are used (a 1 x 1 map,
    no layers)."""
    ctx = _jpeg_contexts.get(device)
    if ctx is None:
        g = Geometry()
        check(lib().amb_geometry_init(1.0, 1.0, 1.0, 0.0, 0.0, C.byref(g)))
        ctx = C.c_void_p()
        check(lib().amb_create(C.byref(g), int(device), 0, 1, C.byref(ctx)))
        _jpeg_contexts[device] = ctx
    return ctx


def encode_jpeg(image, quality=95, sampling="420", restart_interval=0):
    """Baseline JPEG (bytes) of a torch CUDA uint8 tensor, H x W (gray) or H x W x 3 (B, G, R), encoded on its device:
    byte for byte cv2.imencode(".jpg", image, params).  Rows may be padded (a row-sliced view), pixels must be packed.
    Waits for the work queued on the current torch stream before reading the image."""
    import torch
    if not isinstance(image, torch.Tensor) or not image.is_cuda or image.dtype != torch.uint8:
        raise ValueError("encode_jpeg: expected a torch CUDA uint8 tensor")
    if image.dim() == 2:
        channels = 1
    elif image.dim() == 3 and image.shape[2] == 3:
        channels = 3
    else:
        raise ValueError("encode_jpeg: expected H x W or H x W x 3, got %s" % (tuple(image.shape),))
    h, w = int(image.shape[0]), int(image.shape[1])
    inner = (1,) if channels == 1 else (3, 1)
    if tuple(image.stride())[1:] != inner or (h > 1 and image.stride(0) < w * channels):
        raise ValueError("encode_jpeg: pixels must be packed along rows, got strides %s" % (tuple(image.stride()),))
    args = _jpeg_args(w, h, channels, quality, sampling, restart_interval)
    device = image.device.index if image.device.index is not None else torch.cuda.current_device()
    ctx = _jpeg_context(device)
    torch.cuda.current_stream(image.device).synchronize()
    stride = image.stride(0) if h > 1 else w * channels
    return _jpeg_call(lambda buf, cap, size: lib().amb_jpeg_encode_device(ctx, C.c_void_p(image.data_ptr()), args[0],
                                                                          args[1], stride, *args[2:], buf, cap, size),
                      args, ctx)


# ---- JPEG frames decoded on the device (amb_jpeg_info, amb_jpeg_decode_device) ---------------------------------------
JPEG_SAMPLING_NAME = {0: "420", 1: "444", 2: "422"}


class _JpegFile(object):
    """A JPEG file handed to the library without copying it: `ptr` is the address of its `size` bytes, valid while this
    object lives.  bytes are used in place (read only); bytearray, writable memoryviews and contiguous uint8 arrays
    likewise; a read-only or strided view is copied once."""

    def __init__(self, data):
        if isinstance(data, np.ndarray):
            if data.dtype != np.uint8:
                raise ValueError("a JPEG file as an array must be uint8, got %s" % data.dtype)
            self.keep = np.ascontiguousarray(data).reshape(-1)
            self.ptr, self.size = self.keep.ctypes.data, self.keep.size
            return
        if isinstance(data, memoryview):
            data = data if data.contiguous and not data.readonly else bytes(data)
        if isinstance(data, bytes):
            self.keep = data
            self.ptr, self.size = C.cast(C.c_char_p(data), C.c_void_p).value, len(data)   # the bytes' own storage
        elif isinstance(data, (bytearray, memoryview)):
            n = data.nbytes if isinstance(data, memoryview) else len(data)
            self.keep = (C.c_char * max(n, 1)).from_buffer(data) if n else C.create_string_buffer(1)
            self.ptr, self.size = C.addressof(self.keep), n
        else:
            raise ValueError("a JPEG file must be bytes-like, got %s" % type(data).__name__)


def _jpeg_info(f):
    w, h, c, s, r = C.c_int32(), C.c_int32(), C.c_int(), C.c_int(), C.c_int32()
    check(lib().amb_jpeg_info(C.c_void_p(f.ptr), f.size, C.byref(w), C.byref(h), C.byref(c), C.byref(s), C.byref(r)))
    return {"width": w.value, "height": h.value, "components": c.value, "sampling": JPEG_SAMPLING_NAME[s.value],
            "restart_interval": r.value}


def jpeg_info(data):
    """The header of a JPEG file (host only, no GPU): dict width, height, components (1 or 3), sampling ('444',
    '422' or '420'; '444' for gray) and restart_interval.  AmbError(AMB_ERR_UNSUPPORTED) for a file outside the set the
    device decoder takes, AmbError(AMB_ERR_INVALID_ARGUMENT) for one that is not a well-formed JPEG."""
    return _jpeg_info(_JpegFile(data))


def decode_jpeg(data_or_list, channels=3, device=0):
    """JPEG file(s) decoded on a GPU: torch CUDA uint8 [H, W, 3] (B, G, R) for channels=3, [H, W] for channels=1, pixel
    for pixel cv2.imread(path, IMREAD_COLOR / IMREAD_GRAYSCALE).  A list of files returns a list of tensors (decoded
    together).  Raises AmbError with the status of the first file that cannot be decoded (AMB_ERR_UNSUPPORTED,
    AMB_ERR_INVALID_ARGUMENT, AMB_ERR_CORRUPT_DATA)."""
    import torch
    if channels not in (1, 3):
        raise ValueError("decode_jpeg: channels must be 1 or 3, got %r" % (channels,))
    single = not isinstance(data_or_list, (list, tuple))
    files = [_JpegFile(d) for d in ([data_or_list] if single else data_or_list)]
    n = len(files)
    if n == 0:
        return []
    infos = [_jpeg_info(f) for f in files]
    dev = torch.device("cuda", int(device))
    outs = [torch.empty((i["height"], i["width"], 3) if channels == 3 else (i["height"], i["width"]), dtype=torch.uint8,
                        device=dev) for i in infos]
    ctx = _jpeg_context(int(device))
    torch.cuda.synchronize(dev)   # the outputs' allocation is ordered before the decode on the context's stream
    ptrs = (C.c_void_p * n)(*[f.ptr for f in files])
    sizes = (C.c_size_t * n)(*[f.size for f in files])
    outp = (C.c_void_p * n)(*[o.data_ptr() for o in outs])
    steps = (C.c_size_t * n)(*[i["width"] * channels for i in infos])
    status = (C.c_int * n)()
    check(lib().amb_jpeg_decode_device(ctx, ptrs, sizes, n, channels, outp, steps, status), ctx)
    return outs[0] if single else outs


# ---- Deflate strips of a GeoTIFF (amb_deflate_strips_device, amb_export_deflate_strips) -------------------------------
def _deflate_rows(row_bytes, height, rows_per_strip):
    """rows_per_strip, by default libtiff's 8 KiB strip max(1, 8192 // row_bytes), capped at the height."""
    if rows_per_strip is None:
        return max(1, min(height, 8192 // row_bytes))
    if isinstance(rows_per_strip, bool) or not isinstance(rows_per_strip, (int, np.integer)) or rows_per_strip < 1:
        raise ValueError("rows_per_strip must be a positive integer, got %r" % (rows_per_strip,))
    return int(min(rows_per_strip, height, 0x7FFFFFFF))


def _deflate_call(call, width, height, fmt, rps, ctx):
    """Runs `call(buffer, capacity, size, strip_bytes)` with a buffer of amb_deflate_max_size bytes; returns the strips
    (bytes) and their lengths (uint32 array)."""
    cap = lib().amb_deflate_max_size(width, height, fmt, rps)
    if cap == 0:
        raise AmbError(_lib.AMB_ERR_UNSUPPORTED, "a %d x %d raster in strips of %d rows" % (width, height, rps))
    buf = np.empty(cap, np.uint8)
    counts = np.zeros((height + rps - 1) // rps, np.uint32)
    size = C.c_size_t(0)
    check(call(buf.ctypes.data_as(C.c_void_p), cap, C.byref(size), counts.ctypes.data_as(C.c_void_p)), ctx)
    return buf[:size.value].tobytes(), counts


_DEFLATE_DTYPES = {"f32": "float32", "gray8": "uint8", "mask8": "uint8", "bgr8": "uint8"}


def _device_raster(image, fmt, what):
    """Checks a torch CUDA raster of format `fmt` for deflate_strips / cog_tiles (ValueError otherwise); returns (h, w,
    format id, row stride in bytes, the device's context) once the work queued on the current torch stream is done."""
    import torch
    if fmt not in _DEFLATE_DTYPES:
        raise ValueError("%s: fmt must be 'f32', 'gray8', 'bgr8' or 'mask8', got %r" % (what, fmt))
    if not isinstance(image, torch.Tensor) or not image.is_cuda or \
            image.dtype != getattr(torch, _DEFLATE_DTYPES[fmt]):
        raise ValueError("%s: expected a torch CUDA %s tensor for %r" % (what, _DEFLATE_DTYPES[fmt], fmt))
    channels = 3 if fmt == "bgr8" else 1
    if image.dim() != (3 if channels == 3 else 2) or (channels == 3 and image.shape[2] != 3):
        raise ValueError("%s: expected %s for %r, got %s"
                         % (what, "H x W x 3" if channels == 3 else "H x W", fmt, tuple(image.shape)))
    h, w = int(image.shape[0]), int(image.shape[1])
    inner = (1,) if channels == 1 else (3, 1)
    if h < 1 or w < 1 or tuple(image.stride())[1:] != inner or (h > 1 and image.stride(0) < w * channels):
        raise ValueError("%s: pixels must be packed along rows, got shape %s strides %s"
                         % (what, tuple(image.shape), tuple(image.stride())))
    f = _lib.RASTER_FORMAT[fmt]
    device = image.device.index if image.device.index is not None else torch.cuda.current_device()
    ctx = _jpeg_context(device)
    torch.cuda.current_stream(image.device).synchronize()
    stride = image.stride(0) * image.element_size() if h > 1 else w * _lib.RASTER_BPP[f]
    return h, w, f, stride, ctx


def deflate_strips(image, fmt, rows_per_strip=None):
    """The Deflate-compressed GeoTIFF strips of a torch CUDA raster, compressed on its device (convention:
    include/aerial_mapper_b200.h, amb_deflate_strips_device): returns (strips as bytes, uint32 length of each strip,
    rows_per_strip), ready for io.write_geotiff_strips.  image: float32 H x W for fmt "f32", uint8 H x W for "gray8" and
    "mask8", uint8 H x W x 3 (B, G, R) for "bgr8".  Rows may be padded (a row-sliced view), pixels must be packed.  Waits
    for the work queued on the current torch stream before reading the image."""
    h, w, f, stride, ctx = _device_raster(image, fmt, "deflate_strips")
    rps = _deflate_rows(w * _lib.RASTER_BPP[f], h, rows_per_strip)
    data, counts = _deflate_call(
        lambda buf, cap, size, sb: lib().amb_deflate_strips_device(ctx, C.c_void_p(image.data_ptr()), w, h, stride, f,
                                                                   rps, buf, cap, size, sb), w, h, f, rps, ctx)
    return data, counts, rps


# ---- Cloud-Optimized GeoTIFF tiles (amb_cog_tiles_device, amb_export_cog_tiles) ------------------------------------------
def _cog_tile(tile_size):
    if isinstance(tile_size, bool) or not isinstance(tile_size, (int, np.integer)) or not 16 <= tile_size <= 4096 or \
            tile_size % 16:
        raise ValueError("tile_size must be a multiple of 16 in [16, 4096], got %r" % (tile_size,))
    return int(tile_size)


def _cog_call(call, width, height, fmt, tile, ctx, cap=None):
    """Runs `call(buffer, capacity, size, tile_bytes)` with a buffer of `cap` bytes (by default amb_cog_max_size);
    returns the tiles in file order (bytes) and their lengths (uint32 array)."""
    if cap is None:
        cap = lib().amb_cog_max_size(width, height, fmt, tile)
    if cap == 0:
        raise AmbError(_lib.AMB_ERR_UNSUPPORTED, "a %d x %d raster in tiles of %d" % (width, height, tile))
    from . import io
    n_tiles = sum(-(-w // tile) * -(-h // tile) for w, h in io.cog_layout(width, height, tile))
    buf = np.empty(cap, np.uint8)
    counts = np.zeros(n_tiles, np.uint32)
    size = C.c_size_t(0)
    check(call(buf.ctypes.data_as(C.c_void_p), cap, C.byref(size), counts.ctypes.data_as(C.c_void_p)), ctx)
    return buf[:size.value].tobytes(), counts


def cog_tiles(image, fmt, tile_size=512):
    """The tiles of a Cloud-Optimized GeoTIFF of a torch CUDA raster: overview pyramid, tiling and Deflate on its device
    (convention: include/aerial_mapper_b200.h, amb_cog_tiles_device).  Returns (tiles as bytes in file order, uint32
    length of each tile), ready for io.write_cog.  image and fmt as for deflate_strips; tile_size a multiple of 16 in
    [16, 4096].  Waits for the work queued on the current torch stream before reading the image."""
    tile = _cog_tile(tile_size)
    h, w, f, stride, ctx = _device_raster(image, fmt, "cog_tiles")
    return _cog_call(
        lambda buf, cap, size, tb: lib().amb_cog_tiles_device(ctx, C.c_void_p(image.data_ptr()), w, h, stride, f, tile,
                                                              buf, cap, size, tb), w, h, f, tile, ctx)


# ---- JPEG and mask tiles of a Cloud-Optimized GeoTIFF (amb_cog_jpeg_tiles_device, amb_cog_mask_tiles_device) ------------
def _cog_jpeg_args(quality, sampling):
    """Checks quality and sampling (ValueError otherwise); returns their C values."""
    if sampling not in JPEG_SAMPLING:
        raise ValueError("JPEG sampling must be '420' or '444', got %r" % (sampling,))
    if isinstance(quality, bool) or not isinstance(quality, (int, np.integer)) or not 1 <= quality <= 100:
        raise ValueError("JPEG quality must be an integer in [1, 100], got %r" % (quality,))
    return int(quality), JPEG_SAMPLING[sampling]


def _cog_jpeg_call(call, width, height, fmt, tile, quality, sampling, ctx):
    """Runs `call(buffer, capacity, size, tile_bytes)`, first with a buffer the size of the raw stacked tiles, again at
    the size the library reports if the tiles are larger (incompressible content); returns the tiles in file order
    (bytes) and their lengths (uint32 array)."""
    if lib().amb_cog_jpeg_max_size(width, height, fmt, tile, quality, sampling) == 0:
        raise AmbError(_lib.AMB_ERR_UNSUPPORTED, "JPEG tiles of a %d x %d raster in tiles of %d" % (width, height, tile))
    from . import io
    n_tiles = sum(-(-w // tile) * -(-h // tile) for w, h in io.cog_layout(width, height, tile))
    cap = n_tiles * (tile * tile * _lib.RASTER_BPP[fmt] + 64)
    for _ in range(2):
        buf = np.empty(cap, np.uint8)
        counts = np.zeros(n_tiles, np.uint32)
        size = C.c_size_t(0)
        st = call(buf.ctypes.data_as(C.c_void_p), cap, C.byref(size), counts.ctypes.data_as(C.c_void_p))
        if st == _lib.AMB_ERR_SIZE_MISMATCH and size.value > cap:
            cap = size.value
            continue
        check(st, ctx)
        return buf[:size.value].tobytes(), counts
    raise AmbError(_lib.AMB_ERR_SIZE_MISMATCH, "JPEG tiles changed size between two encodes of the same raster")


def cog_jpeg_tables(fmt, quality=75):
    """The JPEGTables stream (bytes: SOI, DQT ..., DHT ..., EOI, what cv2.imencode writes) of the JPEG tiles of a "gray8"
    or "bgr8" raster at `quality`; host only (amb_cog_jpeg_tables)."""
    if fmt not in ("gray8", "bgr8"):
        raise ValueError("cog_jpeg_tables: fmt must be 'gray8' or 'bgr8', got %r" % (fmt,))
    q, _ = _cog_jpeg_args(quality, "420")
    buf = np.empty(1024, np.uint8)
    size = C.c_size_t(0)
    check(lib().amb_cog_jpeg_tables(3 if fmt == "bgr8" else 1, q, buf.ctypes.data_as(C.c_void_p), len(buf),
                                    C.byref(size)))
    return buf[:size.value].tobytes()


def cog_jpeg_tiles(image, fmt, tile_size=512, quality=75, sampling="420"):
    """The JPEG tiles of a Cloud-Optimized GeoTIFF of a torch CUDA "gray8" or "bgr8" raster: overview pyramid, tiling and
    JPEG on its device (convention: include/aerial_mapper_b200.h, amb_cog_jpeg_tiles_device).  Returns (tiles as bytes
    in file order, uint32 length of each tile, the JPEGTables stream), ready for io.write_cog(..., compress="jpeg").
    image as for cog_tiles; quality 1..100, sampling "420" or "444" (ignored for gray)."""
    if fmt not in ("gray8", "bgr8"):
        raise ValueError("cog_jpeg_tiles: fmt must be 'gray8' or 'bgr8', got %r" % (fmt,))
    tile = _cog_tile(tile_size)
    q, s = _cog_jpeg_args(quality, sampling)
    h, w, f, stride, ctx = _device_raster(image, fmt, "cog_jpeg_tiles")
    data, counts = _cog_jpeg_call(
        lambda buf, cap, size, tb: lib().amb_cog_jpeg_tiles_device(ctx, C.c_void_p(image.data_ptr()), w, h, stride, f,
                                                                   tile, q, s, buf, cap, size, tb), w, h, f, tile, q, s,
        ctx)
    return data, counts, cog_jpeg_tables(fmt, q)


def cog_mask_tiles(image, tile_size=512):
    """The 1-bit mask tiles of a Cloud-Optimized GeoTIFF of a torch CUDA uint8 H x W "mask8" raster (non-zero = valid):
    its MASK8 pyramid, tiled, packed to bits and deflated on its device (convention: include/aerial_mapper_b200.h,
    amb_cog_mask_tiles_device).  Returns (tiles as bytes in file order, uint32 length of each tile), the `mask` of
    io.write_cog."""
    tile = _cog_tile(tile_size)
    h, w, f, stride, ctx = _device_raster(image, "mask8", "cog_mask_tiles")
    return _cog_call(
        lambda buf, cap, size, tb: lib().amb_cog_mask_tiles_device(ctx, C.c_void_p(image.data_ptr()), w, h, stride, tile,
                                                                   buf, cap, size, tb), w, h, f, tile, ctx,
        cap=lib().amb_cog_mask_max_size(w, h, tile))
