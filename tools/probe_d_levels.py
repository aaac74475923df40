"""How much of config D's step is the single 200x256 level chain?  (graph replay time of the step for subsets of the levels)"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench_configs as bc
from benchkit import capture, replay_ms
dev = torch.device('cuda:0')
for levels in ([(200, 256)], [(200, 256), (200, 256)], [(100, 128)], [(50, 64)], bc.LEVELS_D):
    bc.LEVELS_D = list(levels)
    step, info = bc.build_D(dev, 1234)
    for _ in range(2):
        step()
    print(levels, f'{replay_ms(capture(step), 10):.3f} ms per step', flush=True)
