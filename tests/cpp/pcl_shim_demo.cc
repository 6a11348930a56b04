// pcl_shim_demo.cc — the call sequence of the reference's OrthoFromPcl demo (main-ortho-from-pcl.cc:122-136): caller code
// that only uses the reference's public API, built against the DROP-IN headers (aerial_mapper_b200/shim, -DAMB_SHIM_MINI
// stand-ins) by tests/test_ortho_from_pcl_stripes.py.  AMB_SHIM_GPUS=N in the environment spreads the map's column stripes
// over N GPUs of this process.
// Reads a scenario file written by the test, writes the resulting `ortho` layer back.
#include <aerial-mapper-ortho/ortho-from-pcl.h>

#include <cstdio>
#include <fstream>

template <typename T>
static void rd(std::ifstream& f, T* p, size_t n) {
  f.read(reinterpret_cast<char*>(p), sizeof(T) * n);
}

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  std::ifstream f(argv[1], std::ios::binary);
  double geo[5];  // delta_easting, delta_northing, resolution, center_easting, center_northing
  rd(f, geo, 5);
  int64_t hdr[3];  // n_points, interpolation_radius, use_adaptive_interpolation
  rd(f, hdr, 3);
  AlignedType<std::vector, Eigen::Vector3d>::type cloud(static_cast<size_t>(hdr[0]));
  rd(f, &cloud[0](0), 3 * cloud.size());
  std::vector<int> intensities(static_cast<size_t>(hdr[0]));
  rd(f, intensities.data(), intensities.size());

  // AerialGridMap::initialize (aerial-mapper-grid-map.cc:23-49)
  grid_map::GridMap map({"ortho", "elevation", "elevation_angle", "num_observations", "elevation_angle_first_view",
                         "delta", "observation_index", "observation_index_first", "colored_ortho"});
  map.setFrameId("world");
  grid_map::Length len;
  len(0) = geo[0];
  len(1) = geo[1];
  grid_map::Position pos;
  pos(0) = geo[3];
  pos(1) = geo[4];
  map.setGeometry(len, geo[2], pos);
  map["ortho"].setConstant(255);

  ortho::Settings settings;  // main-ortho-from-pcl.cc:122-131
  settings.interpolation_radius = static_cast<int>(hdr[1]);
  settings.use_adaptive_interpolation = hdr[2] != 0;
  ortho::OrthoFromPcl mosaic(settings);
  mosaic.process(cloud, intensities, &map);

  std::ofstream o(argv[2], std::ios::binary);
  o.write(reinterpret_cast<const char*>(map["ortho"].data()), sizeof(float) * map["ortho"].rows() * map["ortho"].cols());
  std::printf("pcl_shim_demo ok %d x %d\n", map.getSize()(0), map.getSize()(1));
  return 0;
}
