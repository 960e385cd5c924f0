"""Small MPM run for a profiler (config 3 scene, non-graph launches). Usage: python scripts/profile_mpm.py [substeps]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from scripts.gpu_mpm_perf import make

if __name__ == "__main__":
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 12
    s = make()
    s.p2g2p_n(n, 1e-4)
    torch.cuda.synchronize()
