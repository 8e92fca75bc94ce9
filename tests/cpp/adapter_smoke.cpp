// C++ smoke test of include/b200reg_pcl.hpp (stand-alone mode, no PCL): reads like apps/align.cpp:18-40 of the
// reference — setInputTarget, setInputSource, align, getFitnessScore. Built by tests/test_host_logic.py on CPU (where it
// must fail loudly for lack of a GPU) and run by tests/test_gpu_parity.py on the H100.
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <stdexcept>

#include "b200reg_pcl.hpp"

static float frand(unsigned& s) {
  s = s * 1664525u + 1013904223u;
  return (float)((s >> 8) & 0xffffff) / 16777216.0f;
}

int main() {
  try {
    b200reg::NormalDistributionsTransform ndt;
    ndt.setResolution(2.0f);
    ndt.setTransformationEpsilon(0.01);
    ndt.setNeighborhoodSearchMethod(b200reg::DIRECT7);
    b200reg::PointCloud target, source, aligned;
    unsigned seed = 7;
    for (int i = 0; i < 40000; i++) {  // a floor and two walls
      b200reg::PointXYZI p;
      float u = 40.f * frand(seed) - 20.f, v = 40.f * frand(seed) - 20.f;
      int kind = i % 3;
      if (kind == 0) { p.x = u; p.y = v; p.z = 0.02f * frand(seed); }
      else if (kind == 1) { p.x = u; p.y = 10.f + 0.02f * frand(seed); p.z = 4.f * frand(seed); }
      else { p.x = 15.f + 0.02f * frand(seed); p.y = v; p.z = 4.f * frand(seed); }
      target.points.push_back(p);
      if (i % 4 == 0) {  // source = target shifted by (-0.3, 0.2, 0)
        b200reg::PointXYZI q = p;
        q.x -= 0.3f;
        q.y += 0.2f;
        source.points.push_back(q);
      }
    }
    ndt.setInputTarget(target);
    ndt.setInputSource(source);
    ndt.align(aligned);
    b200reg::Matrix4f T = ndt.getFinalTransformation();
    std::printf("converged=%d iterations=%d t=(%.4f %.4f %.4f) fitness=%.6f aligned=%zu\n", (int)ndt.hasConverged(),
                ndt.getFinalNumIteration(), T[12], T[13], T[14], ndt.getFitnessScore(), aligned.size());
    bool ok = ndt.hasConverged() && std::fabs(T[12] - 0.3f) < 0.05f && std::fabs(T[13] + 0.2f) < 0.05f;

    // frontend session (scanmatcher_component.cpp cloud callback): frame 0 initialises the map from `target` at the
    // identity pose, frame 1 is the same world seen from a sensor moved by (+2.0, 0, 0): the session must report that
    // pose, trigger a map update (>= trans_for_mapupdate = 1.5 m) and keep two submaps on the device.
    b200reg::NormalDistributionsTransform reg;
    reg.setResolution(2.0f);
    reg.setTransformationEpsilon(0.01);
    reg.setNeighborhoodSearchMethod(b200reg::DIRECT7);
    b200reg::ScanMatcherSession session;
    session.setParams(0.5f, 0.4f, 10, 1.5);
    double pose[7];
    float fin[16];
    bool upd0 = session.receiveCloud(reg.handle(), &target.points[0].x, target.size(), sizeof(b200reg::PointXYZI),
                                     offsetof(b200reg::PointXYZI, intensity), pose, fin);
    b200reg::PointCloud moved = target;
    for (auto& p : moved.points) p.x -= 0.4f;  // sensor moved +0.4 m in x per frame
    bool upd = false;
    int frames_until_update = 0;
    for (int k = 1; k <= 6 && !upd; k++) {
      for (auto& p : moved.points) p.x = target.points[&p - &moved.points[0]].x - 0.4f * k;
      upd = session.receiveCloud(reg.handle(), &moved.points[0].x, moved.size(), sizeof(b200reg::PointXYZI),
                                 offsetof(b200reg::PointXYZI, intensity), pose, fin);
      frames_until_update = k;
    }
    std::printf("session: first update after %d frames, pose x=%.3f y=%.3f, submaps=%zu\n", frames_until_update, pose[0], pose[1],
                session.numSubmaps());
    ok = ok && !upd0 && upd && frames_until_update == 4 && std::fabs(pose[0] - 1.6) < 0.1 && std::fabs(pose[1]) < 0.1 &&
         session.numSubmaps() == 2;
    return ok ? 0 : 2;
  } catch (const std::exception& e) {
    std::printf("no GPU: %s\n", e.what());
    return 3;  // expected on a CPU-only box: the engine has no CPU fallback
  }
}
