import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np
import lidarslam_ros2_b200 as m
import oracle
from lidarslam_ros2_b200 import synth
cfg, res = sys.argv[1], float(sys.argv[2])
src, tgt, _ = synth.registration_pair(cfg, res)
o = oracle.NDT(resolution=res, transformation_epsilon=0.01); o.set_target(tgt); o.set_source(src); To = o.align()
print("oracle iters", o.iterations)
g = m.NormalDistributionsTransform(); g.setResolution(res); g.setTransformationEpsilon(0.01)
g.setInputTarget(tgt); g.setInputSource(src)
for k in range(4):
    T = g.align()
    print(k, "iters", g.getFinalNumIteration(), "evals", g.stats()["evaluations"], "err", synth.pose_error(T, To))
