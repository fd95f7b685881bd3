import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from path_optimizer_b200 import synth
from path_optimizer_b200.solver import BatchPathSolver
b = synth.curvy_corridors(1024, 100)
s = BatchPathSolver(max_batch=1024, max_total_points=1024 * 100)
r = s.solve(b, "K")
print("K kernel_ms", r["stats"].kernel_ms)
