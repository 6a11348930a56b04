"""aerial_mapper_b200 — H100-native grid-mapping hot path of ethz-asl/aerial_mapper (DSM rasteriser + grid
orthomosaic back-projection) behind the reference's own class API.  See DESIGN.md / INTEGRATION.md.

The compute lives in libaerial_mapper_b200.so (hand-written sm_90a CUDA, C ABI in include/aerial_mapper_b200.h).
"""
from ._lib import (AMB_OK, AmbError, Camera, Geometry, LAYER_ID, LAYER_NAMES, DIST_EQUIDISTANT, DIST_NONE,
                   DIST_RADTAN, LIB_PATH, build, check, lib)
from .api import (AerialGridMap, Dsm, DsmSettings, GridMap, GridMapSettings, HOT_LAYERS, NCamera,
                  OrthoBackwardGrid, OrthoFromPcl, OrthoFromPclSettings, OrthoSettings, compute_point_cloud,
                  cog_jpeg_tables, cog_jpeg_tiles, cog_mask_tiles, cog_tiles, decode_jpeg, deflate_strips, dsm_thresholds, encode_jpeg, jpeg_info, rectify_stereo_maps,
                  rectify_stereo_setup)

__all__ = ["AMB_OK", "AmbError", "Camera", "Geometry", "LAYER_ID", "LAYER_NAMES", "DIST_EQUIDISTANT", "DIST_NONE",
           "DIST_RADTAN", "LIB_PATH", "build", "check", "lib", "AerialGridMap", "Dsm", "DsmSettings", "GridMap",
           "GridMapSettings", "HOT_LAYERS", "NCamera", "OrthoBackwardGrid", "OrthoFromPcl", "OrthoFromPclSettings", "OrthoSettings", "cog_jpeg_tables", "cog_jpeg_tiles", "cog_mask_tiles", "cog_tiles", "compute_point_cloud", "decode_jpeg", "deflate_strips", "dsm_thresholds", "encode_jpeg", "jpeg_info",
           "rectify_stereo_maps", "rectify_stereo_setup"]
