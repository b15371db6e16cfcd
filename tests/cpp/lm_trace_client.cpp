// A client of NanoGICP::setDebugPrint (lsq_registration.hpp:92): LoopClosure's configuration (loop_closure.cpp:9-16), debug
// print on, one align.  stdout carries the reference's LM table (lsq_registration_impl.hpp:95-99, 183-189), then one line
// "records <n> iterations <nr_iterations> lm_failed <0|1>" from lastLmTrace() / lastResult().
// usage: lm_trace_client src.bin dst.bin   (bin = n x 4 float32: x y z intensity)
#define B200REG_HOST_IMPLEMENTATION
#include <nano_gicp/nano_gicp.hpp>
#include <nano_gicp/point_type_nano_gicp.hpp>

#if defined(B200REG_EXPECT_PCL) && !defined(B200REG_HAVE_PCL)
#error "the PCL/Eigen configuration of the facade was requested but b200reg_compat.hpp did not select it"
#endif

#include <cstdio>
#include <fstream>
#include <iostream>

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
  gicp.setDebugPrint(true);
  gicp.setInputSource(src);
  gicp.setInputTarget(dst);
  pcl::PointCloud<PointType> aligned;
  gicp.align(aligned);
  std::cout << "records " << gicp.lastLmTrace().size() << " iterations " << gicp.nr_iterations() << " lm_failed "
            << gicp.lastResult().lm_failed << std::endl;
  return 0;
}
