"""ctypes binding of libaerial_mapper_b200.so (the C ABI declared in include/aerial_mapper_b200.h).

There is no CPU fallback: if the CUDA library is missing this module raises at load time, and every compute entry
point fails with AMB_ERR_NO_DEVICE when no GPU is visible.
"""
import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libaerial_mapper_b200.so")
if os.environ.get("AMB_LIB_PATH"):   # development only: an alternative build of the SAME library (kernel tuning variants)
    LIB_PATH = os.environ["AMB_LIB_PATH"]
CSRC = os.path.join(_HERE, "csrc")

AMB_OK = 0
AMB_ERR_EMPTY = -1
AMB_ERR_SIZE_MISMATCH = -2
AMB_ERR_COINCIDENT_POINT = -3
AMB_ERR_CUDA = -4
AMB_ERR_INVALID_ARGUMENT = -5
AMB_ERR_CHECK_FAILED = -6
AMB_ERR_NO_DEVICE = -7
AMB_ERR_UNSUPPORTED = -8
AMB_ERR_CORRUPT_DATA = -9

LAYER_NAMES = ("ortho", "elevation", "elevation_angle", "num_observations", "elevation_angle_first_view", "delta",
               "observation_index", "observation_index_first", "colored_ortho")
LAYER_ID = {name: k for k, name in enumerate(LAYER_NAMES)}

DIST_NONE, DIST_RADTAN, DIST_EQUIDISTANT, DIST_FOV = 0, 1, 2, 3
DSM_F64, DSM_F32 = 0, 1
# amb_raster_format: pixel formats of amb_export_raster, and their bytes per pixel
RASTER_F32, RASTER_GRAY8, RASTER_BGR8, RASTER_MASK8 = 0, 1, 2, 3
RASTER_FORMAT = {"f32": RASTER_F32, "gray8": RASTER_GRAY8, "bgr8": RASTER_BGR8, "mask8": RASTER_MASK8}
RASTER_BPP = {RASTER_F32: 4, RASTER_GRAY8: 1, RASTER_BGR8: 3, RASTER_MASK8: 1}
# amb_resample: resampling of amb_import_raster
RESAMPLE = {"nearest": 0, "bilinear": 1}


class Geometry(C.Structure):
    _fields_ = [("rows", C.c_int32), ("cols", C.c_int32), ("resolution", C.c_double),
                ("length_x", C.c_double), ("length_y", C.c_double), ("pos_x", C.c_double), ("pos_y", C.c_double)]


class Camera(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("fu", C.c_double), ("fv", C.c_double),
                ("cu", C.c_double), ("cv", C.c_double), ("dist_type", C.c_int32), ("reserved_", C.c_int32),
                ("dist", C.c_double * 4), ("q_C_B", C.c_double * 4), ("t_C_B", C.c_double * 3)]


# amb_sample_type of amb_tiff_layout, by numpy dtype name
SAMPLE_TYPE = {"uint8": 0, "int16": 1, "uint16": 2, "int32": 3, "float32": 4, "float64": 5}


class TiffLayout(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("chunk_width", C.c_int32), ("chunk_height", C.c_int32),
                ("tiled", C.c_int32), ("spp", C.c_int32), ("band", C.c_int32), ("sample", C.c_int32),
                ("compression", C.c_int32), ("predictor", C.c_int32), ("n_chunks", C.c_uint32),
                ("reserved_", C.c_uint32), ("offsets", C.c_void_p), ("byte_counts", C.c_void_p)]


class Timings(C.Structure):
    _fields_ = [("dsm_h2d_ms", C.c_float), ("dsm_bin_ms", C.c_float), ("dsm_gather_ms", C.c_float),
                ("dsm_fill_ms", C.c_float), ("dsm_total_ms", C.c_float), ("ortho_h2d_ms", C.c_float),
                ("ortho_kernel_ms", C.c_float), ("ortho_total_ms", C.c_float),
                ("dsm_kernel_launches", C.c_int32), ("ortho_kernel_launches", C.c_int32),
                ("dsm_points_binned", C.c_int64), ("dsm_cells_empty", C.c_int64),
                ("ortho_h2d_bytes", C.c_int64)]

    def as_dict(self):
        return {name: getattr(self, name) for name, _ in self._fields_}


# every symbol include/aerial_mapper_b200.h declares: name -> (restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    "amb_abi_version": (C.c_int, []),
    "amb_status_string": (C.c_char_p, [C.c_int]),
    "amb_last_error": (C.c_char_p, [_P]),
    "amb_device_count": (C.c_int, []),
    "amb_geometry_init": (C.c_int, [C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.POINTER(Geometry)]),
    "amb_geometry_position": (C.c_int, [C.POINTER(Geometry), C.c_int32, C.c_int32, C.POINTER(C.c_double),
                                        C.POINTER(C.c_double)]),
    "amb_create": (C.c_int, [C.POINTER(Geometry), C.c_int, C.c_int32, C.c_int32, C.POINTER(_P)]),
    "amb_destroy": (None, [_P]),
    "amb_sync": (C.c_int, [_P]),
    "amb_stream": (_P, [_P]),
    "amb_init_layers": (C.c_int, [_P]),
    "amb_upload_layer": (C.c_int, [_P, C.c_int, _P]),
    "amb_download_layer": (C.c_int, [_P, C.c_int, _P]),
    "amb_upload_layer_device": (C.c_int, [_P, C.c_int, _P]),
    "amb_download_layer_async": (C.c_int, [_P, C.c_int, _P]),
    "amb_set_host_mirror": (C.c_int, [_P, C.c_int, _P]),
    "amb_set_host_mirror_compact": (C.c_int, [_P, C.c_int, C.c_int]),
    "amb_layer_device_ptr": (C.c_int, [_P, C.c_int, C.POINTER(_P)]),
    "amb_dsm_process": (C.c_int, [_P, _P, C.c_size_t, C.c_int32, C.c_double, C.c_double]),
    "amb_dsm_process_device": (C.c_int, [_P, _P, C.c_size_t, C.c_int32, C.c_double, C.c_double]),
    "amb_dsm_process_device_ids": (C.c_int, [_P, _P, _P, C.c_size_t, C.c_int32, C.c_double, C.c_double]),
    "amb_dsm_set_density_hint": (C.c_int, [_P, C.c_double]),
    "amb_stripe_y_interval": (C.c_int, [C.POINTER(Geometry), C.c_int32, C.c_int32, C.POINTER(C.c_double),
                                        C.POINTER(C.c_double)]),
    "amb_dsm_set_stream_chunks": (C.c_int, [_P, C.c_int]),
    "amb_dsm_set_precision": (C.c_int, [_P, C.c_int]),
    "amb_dsm_halo_reach": (C.c_double, [C.POINTER(Geometry), C.c_int32]),
    "amb_dsm_extract_halo": (C.c_int, [_P, _P, _P, C.c_size_t, C.c_double, C.c_double, C.c_double, C.c_double, _P,
                                       _P, C.c_uint32, _P]),
    "amb_comm_unique_id": (C.c_int, [_P]),
    "amb_comm_init": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "amb_comm_destroy": (C.c_int, [_P]),
    "amb_comm_set_exchange": (C.c_int, [_P, C.c_int]),
    "amb_comm_last_exchange": (C.c_int, [_P]),
    "amb_comm_size": (C.c_int, [_P]),
    "amb_comm_rank": (C.c_int, [_P]),
    "amb_dsm_process_sharded_device": (C.c_int, [_P, _P, _P, C.c_size_t, C.c_int32, C.c_double, C.c_double,
                                                 C.c_uint32]),
    "amb_dsm_process_sharded": (C.c_int, [_P, _P, _P, C.c_size_t, C.c_int32, C.c_double, C.c_double, C.c_uint32]),
    "amb_dsm_enable_debug": (C.c_int, [_P, C.c_int]),
    "amb_dsm_download_debug": (C.c_int, [_P, _P, _P]),
    "amb_dsm_download_bins": (C.c_int, [_P, _P, _P, _P, _P]),
    "amb_dsm_thresholds": (C.c_int, [C.c_int32, _P, C.c_int32]),
    "amb_ortho_from_pcl_process": (C.c_int, [_P, _P, _P, C.c_size_t, C.c_int32, C.c_int32]),
    "amb_ortho_from_pcl_process_device": (C.c_int, [_P, _P, _P, C.c_size_t, C.c_int32, C.c_int32]),
    "amb_ortho_from_pcl_process_device_ids": (C.c_int, [_P, _P, _P, _P, C.c_size_t, C.c_int32, C.c_int32]),
    "amb_ortho_from_pcl_extract_halo": (C.c_int, [_P, _P, _P, _P, C.c_size_t, C.c_double, C.c_double, C.c_double, _P,
                                                  _P, _P, C.c_uint32, _P]),
    "amb_ortho_from_pcl_process_sharded_device": (C.c_int, [_P, _P, _P, _P, C.c_size_t, C.c_int32, C.c_uint32]),
    "amb_ortho_from_pcl_process_sharded": (C.c_int, [_P, _P, _P, _P, C.c_size_t, C.c_int32, C.c_uint32]),
    "amb_stereo_reproject": (C.c_int, [C.c_int, _P, C.c_size_t, _P, C.c_size_t, C.c_int32, C.c_int32, _P, C.c_double,
                                       _P, _P, C.c_float, _P, _P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "amb_stereo_reproject_device": (C.c_int, [C.c_int, _P, _P, C.c_size_t, _P, C.c_size_t, C.c_int32, C.c_int32, _P,
                                              C.c_double, _P, _P, C.c_float, _P, _P, C.c_size_t, _P, _P]),
    "amb_stereo_rectify_setup": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "amb_stereo_rectify_maps": (C.c_int, [C.c_int, _P, _P, C.c_int32, C.c_int32, C.c_size_t, _P, _P, _P, _P]),
    "amb_stereo_rectify_maps_device": (C.c_int, [C.c_int, _P, _P, _P, C.c_int32, C.c_int32, C.c_size_t, _P, _P, _P, _P,
                                                 _P]),
    "amb_ortho_process": (C.c_int, [_P, C.POINTER(Camera), _P, _P, C.c_size_t, C.c_int32, C.c_size_t, C.c_int32]),
    "amb_ortho_process_device": (C.c_int, [_P, C.POINTER(Camera), _P, _P, C.c_size_t, C.c_int32, C.c_size_t,
                                           C.c_int32]),
    "amb_ortho_set_brute_force": (C.c_int, [_P, C.c_int]),
    "amb_ortho_set_dominance_cull": (C.c_int, [_P, C.c_int]),
    "amb_multi_create": (C.c_int, [C.POINTER(Geometry), C.c_int, C.POINTER(_P)]),
    "amb_multi_destroy": (None, [_P]),
    "amb_multi_size": (C.c_int, [_P]),
    "amb_multi_context": (_P, [_P, C.c_int]),
    "amb_multi_last_error": (C.c_char_p, [_P]),
    "amb_multi_init_layers": (C.c_int, [_P]),
    "amb_multi_upload_layer": (C.c_int, [_P, C.c_int, _P]),
    "amb_multi_download_layer": (C.c_int, [_P, C.c_int, _P]),
    "amb_multi_set_host_mirror": (C.c_int, [_P, C.c_int, _P]),
    "amb_multi_sync": (C.c_int, [_P]),
    "amb_multi_dsm_process": (C.c_int, [_P, _P, C.c_size_t, C.c_int32, C.c_double, C.c_double]),
    "amb_multi_ortho_process": (C.c_int, [_P, C.POINTER(Camera), _P, _P, C.c_size_t, C.c_int32, C.c_size_t, C.c_int32]),
    "amb_multi_ortho_from_pcl_process": (C.c_int, [_P, _P, _P, C.c_size_t, C.c_int32, C.c_int32]),
    "amb_raster_geotransform": (C.c_int, [C.POINTER(Geometry), C.POINTER(C.c_double)]),
    "amb_export_raster": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "amb_export_raster_device": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "amb_multi_export_raster": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "amb_import_raster": (C.c_int, [_P, C.c_int, _P, C.c_int32, C.c_int32, C.c_size_t, C.POINTER(C.c_double), C.c_int,
                                    C.c_float, C.c_int]),
    "amb_import_raster_device": (C.c_int, [_P, C.c_int, _P, C.c_int32, C.c_int32, C.c_size_t, C.POINTER(C.c_double),
                                           C.c_int, C.c_float, C.c_int]),
    "amb_multi_import_raster": (C.c_int, [_P, C.c_int, _P, C.c_int32, C.c_int32, C.c_size_t, C.POINTER(C.c_double),
                                          C.c_int, C.c_float, C.c_int]),
    "amb_raster_import_tables": (C.c_int, [C.POINTER(Geometry), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                           C.POINTER(C.c_double), C.c_int, _P, _P, _P, _P]),
    "amb_tiff_decode_device": (C.c_int, [_P, _P, C.c_size_t, C.POINTER(TiffLayout), C.c_int32, C.c_int32, C.c_int32,
                                         C.c_int32, _P, C.c_size_t]),
    "amb_import_tiff": (C.c_int, [_P, C.c_int, _P, C.c_size_t, C.POINTER(TiffLayout), C.POINTER(C.c_double), C.c_int,
                                  C.c_float, C.c_int]),
    "amb_multi_import_tiff": (C.c_int, [_P, C.c_int, _P, C.c_size_t, C.POINTER(TiffLayout), C.POINTER(C.c_double),
                                        C.c_int, C.c_float, C.c_int]),
    "amb_import_raster_lonlat": (C.c_int, [_P, C.c_int, _P, C.c_int32, C.c_int32, C.c_size_t, C.POINTER(C.c_double),
                                           C.c_int, C.c_float, C.c_int, C.c_int32]),
    "amb_import_raster_lonlat_device": (C.c_int, [_P, C.c_int, _P, C.c_int32, C.c_int32, C.c_size_t,
                                                  C.POINTER(C.c_double), C.c_int, C.c_float, C.c_int, C.c_int32]),
    "amb_multi_import_raster_lonlat": (C.c_int, [_P, C.c_int, _P, C.c_int32, C.c_int32, C.c_size_t,
                                                 C.POINTER(C.c_double), C.c_int, C.c_float, C.c_int, C.c_int32]),
    "amb_import_tiff_lonlat": (C.c_int, [_P, C.c_int, _P, C.c_size_t, C.POINTER(TiffLayout), C.POINTER(C.c_double),
                                         C.c_int, C.c_float, C.c_int, C.c_int32]),
    "amb_multi_import_tiff_lonlat": (C.c_int, [_P, C.c_int, _P, C.c_size_t, C.POINTER(TiffLayout),
                                               C.POINTER(C.c_double), C.c_int, C.c_float, C.c_int, C.c_int32]),
    "amb_lonlat_import_window": (C.c_int, [C.POINTER(Geometry), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                           C.POINTER(C.c_double), _P]),
    "amb_lonlat_positions_device": (C.c_int, [_P, C.c_int32, _P]),
    "amb_jpeg_max_size": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int, C.c_int, C.c_int, C.c_int32]),
    "amb_jpeg_encode_device": (C.c_int, [_P, _P, C.c_int32, C.c_int32, C.c_size_t, C.c_int, C.c_int, C.c_int,
                                         C.c_int32, _P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "amb_export_jpeg": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int32, _P, C.c_size_t,
                                  C.POINTER(C.c_size_t)]),
    "amb_jpeg_info": (C.c_int, [_P, C.c_size_t, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int),
                                C.POINTER(C.c_int), C.POINTER(C.c_int32)]),
    "amb_jpeg_decode_device": (C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_size_t), C.c_size_t, C.c_int, C.POINTER(_P),
                                         C.POINTER(C.c_size_t), C.POINTER(C.c_int)]),
    "amb_ortho_process_jpeg": (C.c_int, [_P, C.POINTER(Camera), _P, C.POINTER(_P),
                                         C.POINTER(C.c_size_t), C.c_size_t, C.c_int32]),
    "amb_deflate_max_size": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int, C.c_int32]),
    "amb_deflate_strips_device": (C.c_int, [_P, _P, C.c_int32, C.c_int32, C.c_size_t, C.c_int, C.c_int32, _P,
                                            C.c_size_t, C.POINTER(C.c_size_t), _P]),
    "amb_export_deflate_strips": (C.c_int, [_P, C.c_int, C.c_int, C.c_int32, _P, C.c_size_t, C.POINTER(C.c_size_t),
                                            _P]),
    "amb_cog_layout": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, _P, _P, _P]),
    "amb_cog_max_size": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int, C.c_int32]),
    "amb_cog_tiles_device": (C.c_int, [_P, _P, C.c_int32, C.c_int32, C.c_size_t, C.c_int, C.c_int32, _P, C.c_size_t,
                                       C.POINTER(C.c_size_t), _P]),
    "amb_export_cog_tiles": (C.c_int, [_P, C.c_int, C.c_int, C.c_int32, _P, C.c_size_t, C.POINTER(C.c_size_t), _P]),
    "amb_cog_jpeg_max_size": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int, C.c_int32, C.c_int, C.c_int]),
    "amb_cog_jpeg_tables": (C.c_int, [C.c_int, C.c_int, _P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "amb_cog_jpeg_tiles_device": (C.c_int, [_P, _P, C.c_int32, C.c_int32, C.c_size_t, C.c_int, C.c_int32, C.c_int,
                                            C.c_int, _P, C.c_size_t, C.POINTER(C.c_size_t), _P]),
    "amb_export_cog_jpeg_tiles": (C.c_int, [_P, C.c_int, C.c_int, C.c_int32, C.c_int, C.c_int, _P, C.c_size_t,
                                            C.POINTER(C.c_size_t), _P]),
    "amb_cog_mask_max_size": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    "amb_cog_mask_tiles_device": (C.c_int, [_P, _P, C.c_int32, C.c_int32, C.c_size_t, C.c_int32, _P, C.c_size_t,
                                            C.POINTER(C.c_size_t), _P]),
    "amb_export_cog_mask_tiles": (C.c_int, [_P, C.c_int, C.c_int32, _P, C.c_size_t, C.POINTER(C.c_size_t), _P]),
    "amb_get_timings": (C.c_int, [_P, C.POINTER(Timings)]),
    "amb_host_alloc": (C.c_int, [C.POINTER(_P), C.c_size_t]),
    "amb_host_free": (C.c_int, [_P]),
}


def build(force=False, verbose=False):
    """Compile the CUDA library in-tree for sm_90a (H100) (nvcc cross-compiles without a GPU)."""
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cc", ".h", ".cuh", ".inc", "Makefile"))]
    srcs.append(os.path.join(_HERE, "..", "include", "aerial_mapper_b200.h"))
    need = force or not os.path.exists(LIB_PATH)
    if not need:
        t = os.path.getmtime(LIB_PATH)
        need = any(os.path.getmtime(s) > t for s in srcs)
    if need:
        out = None if verbose else subprocess.DEVNULL
        subprocess.check_call(["make", "-C", CSRC, "-j", "8", "all"], stdout=out)
    return LIB_PATH


_lib = None


def lib():
    """Load the product library; raises loudly if it is absent (no fallback path exists)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "aerial_mapper_b200: %s is missing — build it with `python -c 'import __graft_entry__ as g; "
                "g.build()'` (there is no CPU fallback)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SYMBOLS.items():
            fn = getattr(L, name)  # AttributeError if the library does not export a declared symbol
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = L
    return _lib


class AmbError(RuntimeError):
    def __init__(self, status, detail=""):
        self.status = status
        msg = lib().amb_status_string(status).decode()
        super().__init__("amb status %d: %s%s" % (status, msg, (" — " + detail) if detail else ""))


def check(status, ctx=None):
    if status != AMB_OK:
        detail = lib().amb_last_error(ctx).decode() if ctx else ""
        raise AmbError(status, detail)
    return status
