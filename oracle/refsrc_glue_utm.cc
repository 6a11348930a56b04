/*
 * refsrc_glue_utm.cc — C entry point around the REFERENCE'S OWN UTM::UTMtoLL (TEST INFRASTRUCTURE; see amb_oracle.h).
 *
 *   /root/reference/aerial_mapper_thirdparty/include/aerial-mapper-thirdparty/gps-conversions.h, verbatim (found through
 *   -I$(REF_ROOT)/aerial_mapper_thirdparty/include).  tests/golden/make_utm_golden.py builds it into
 *   _ref/libamb_refsrc_utm.so and records its results in tests/golden/utm_reference.json, so no test needs the build.
 */
#include <aerial-mapper-thirdparty/gps-conversions.h>

#define AMB_EXPORT extern "C" __attribute__((visibility("default")))

// zone: e.g. "32N" (band letter N or later: northern hemisphere) or "33M" (southern); degrees out
AMB_EXPORT void ambo_ref_utm_to_ll(double northing, double easting, const char* zone, double* lat, double* lon) {
  UTM::UTMtoLL(northing, easting, zone, *lat, *lon);
}
