// A client of NanoGICP::setCorrespondenceRandomness with k > 32: LoopClosure's configuration (loop_closure.cpp:9-16) but 48
// neighbours per covariance, one align.  Prints one JSON line: converged, fitness, the covariance count of both clouds and
// getFinalTransformation().
// usage: large_k_client src.bin dst.bin   (bin = n x 4 float32: x y z intensity)
#define B200REG_HOST_IMPLEMENTATION
#include <nano_gicp/nano_gicp.hpp>
#include <nano_gicp/point_type_nano_gicp.hpp>

#if defined(B200REG_EXPECT_PCL) && !defined(B200REG_HAVE_PCL)
#error "the PCL/Eigen configuration of the facade was requested but b200reg_compat.hpp did not select it"
#endif

#include <cstdio>
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
  gicp.setCorrespondenceRandomness(48);
  gicp.setMaximumIterations(32);
  gicp.setMaxCorrespondenceDistance(52.5);
  gicp.setTransformationEpsilon(0.01);
  gicp.setInputSource(src);
  gicp.setInputTarget(dst);
  pcl::PointCloud<PointType> aligned;
  gicp.align(aligned);
  const double score = gicp.getFitnessScore();
  const Eigen::Matrix4f T = gicp.getFinalTransformation();
  std::printf("{\"converged\": %d, \"score\": %.17g, \"n_cov\": [%zu, %zu], \"T\": [", gicp.hasConverged() ? 1 : 0, score,
              gicp.getSourceCovariances().size(), gicp.getTargetCovariances().size());
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) std::printf("%.9g%s", T(i, j), (i == 3 && j == 3) ? "" : ", ");
  std::printf("]}\n");
  return 0;
}
