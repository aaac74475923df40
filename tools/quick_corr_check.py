"""Ten-second check of bxs_corr_solve on the GPU box: the regularised tables of the three golden cases against the reference's own
(tests/golden/corr.npz, scaled max difference) and the device time of one call replayed from a CUDA graph.
      python tools/quick_corr_check.py"""
import numpy as np, torch, sys
sys.path.insert(0, '.')
from benchkit import graph_us
from boxinstseg_b200.models.dense_heads.disco_corr import SemanticCorrSolver
from oracle.make_golden_corr import SOLVER, FEAT
g = np.load('tests/golden/corr.npz')
s = SemanticCorrSolver(**SOLVER)
dev = 'cuda:0'
worst = 0.0
for seed in (0, 1, 2):
    Cu = torch.from_numpy(g[f's{seed}_Cu']).to(dev)
    T = s.votes(Cu, FEAT, FEAT)
    ref = g[f's{seed}_T']
    worst = max(worst, float(np.abs(T.cpu().numpy() - ref).max() / np.abs(ref).max()))
print('solve vs reference golden, max scaled diff:', worst)
print('corr_solve graph us:', graph_us(lambda: s.votes(Cu, FEAT, FEAT), 20, per_graph=4))
