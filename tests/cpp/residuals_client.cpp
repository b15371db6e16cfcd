// A client of NanoGICP::getFitnessScore(max_range) (pcl::Registration::getFitnessScore): LoopClosure's configuration
// (loop_closure.cpp:9-16), one align, then the score at every range given on the command line.  stdout is one JSON line:
// the fp32 final transformation (row-major), lastResult().fitness, the number of rows lastResiduals() holds and the score
// at each range, every double printed with 17 significant digits (it reads back bit for bit).
// usage: residuals_client src.bin dst.bin r...   (bin = n x 4 float32: x y z intensity; r parsed by strtod: "nan", "inf")
#define B200REG_HOST_IMPLEMENTATION
#include <nano_gicp/nano_gicp.hpp>
#include <nano_gicp/point_type_nano_gicp.hpp>

#if defined(B200REG_EXPECT_PCL) && !defined(B200REG_HAVE_PCL)
#error "the PCL/Eigen configuration of the facade was requested but b200reg_compat.hpp did not select it"
#endif

#include <cstdio>
#include <cstdlib>
#include <fstream>

static pcl::PointCloud<PointType> load(const char* path) {
  pcl::PointCloud<PointType> c;
  std::ifstream f(path, std::ios::binary);
  float v[4];
  while (f.read(reinterpret_cast<char*>(v), sizeof(v))) {
    PointType p;
    p.x = v[0];
    p.y = v[1];
    p.z = v[2];
    p.intensity = v[3];
    c.push_back(p);
  }
  return c;
}

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  pcl::PointCloud<PointType>::Ptr src(new pcl::PointCloud<PointType>(load(argv[1])));
  pcl::PointCloud<PointType>::Ptr dst(new pcl::PointCloud<PointType>(load(argv[2])));
  nano_gicp::NanoGICP<PointType, PointType> gicp;
  gicp.setNumThreads(0);
  gicp.setCorrespondenceRandomness(15);
  gicp.setMaximumIterations(32);
  gicp.setMaxCorrespondenceDistance(52.5);
  gicp.setTransformationEpsilon(0.01);
  gicp.setInputSource(src);
  gicp.setInputTarget(dst);
  pcl::PointCloud<PointType> aligned;
  gicp.align(aligned);
  if (!gicp.hasConverged()) std::fprintf(stderr, "not converged\n");
  const b200reg_result& r = gicp.lastResult();
  std::printf("{\"Tf\": [");
  for (int i = 0; i < 16; i++) std::printf("%s%.9g", i ? ", " : "", r.Tf[i]);
  std::printf("], \"fitness\": %.17g, \"rows\": %zu, \"nn_rows\": %zu, \"scores\": [", r.fitness, gicp.lastResiduals().d2.size(),
              gicp.lastResiduals().nn.size());
  for (int a = 3; a < argc; a++) {
    const double s = gicp.getFitnessScore(std::strtod(argv[a], nullptr));
    std::printf("%s%.17g", a > 3 ? ", " : "", s);
  }
  std::printf("]}\n");
  return 0;
}
