"""Clock breakdown of the tensor-core neighbour pass tile: builds a -DB200_TC_TIMING copy of the library (clock64() around
the parts of the tile loop of simTensorKernel<count>), runs the bench's Butina step on it at 4 x 2 superposition without
the pilot and prints clocks per tile for each part.   python tools/pair_pass_timing.py [n_centres] [cluster variant]
The clock reads change the schedule a little: the figures attribute time, the pass time of this build is not a benchmark."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

os.environ["B200_NO_CORE"] = "1"  # bind the instrumented library through ctypes, not the pybind module of the main one

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
out = os.environ.get("B200_TIMING_LIB") or os.path.join(ROOT, "nvmolkit_b200", "lib", "libb200mol_tctiming.so")
if not os.environ.get("B200_TIMING_LIB"):
    subprocess.run(["make", "-C", os.path.join(ROOT, "nvmolkit_b200", "csrc"), "-j", "8", "-s", "tctiming"], check=True)
from nvmolkit_b200 import _lib, synthetic  # noqa: E402

_lib.LIB_PATH = out
import torch  # noqa: E402

import bench  # noqa: E402
from nvmolkit_b200.clustering import fused_butina_device  # noqa: E402

n_centres = int(sys.argv[1]) if len(sys.argv) > 1 else 20000
torch.cuda.set_device(0)
_lib.profile_enable(True)
_lib.set_option("similarity_superpose_auto", 0)
_lib.set_option("similarity_superpose", 4)
_lib.set_option("similarity_superpose_cols", 2)
if len(sys.argv) > 2:
    _lib.set_option("similarity_tensor_cluster", int(sys.argv[2]))
L = _lib.load()
buf = (C.c_ulonglong * 8)()
fp = synthetic.clustered_fingerprints(n_centres, 50, seed=synthetic.SEED)
x = torch.from_numpy(fp.view(np.int32)).cuda()
fused_butina_device(x, bench.CUTOFF)  # warm-up
torch.cuda.synchronize()
L.b200mol_debug_clocks_tc(buf)  # reset
fused_butina_device(x, bench.CUTOFF)
torch.cuda.synchronize()
L.b200mol_debug_clocks_tc(buf)
v = np.array(list(buf), dtype=np.float64)
warp_tiles = max(v[5], 1.0)
tiles = warp_tiles / 8  # eight consumer warps per CTA
print({"n": fp.shape[0], "neighbor_pass_tc_ms": _lib.profile_read("neighbor_pass_tc"),
       "verify_candidates_ms": _lib.profile_read("verify_candidates"),
       "pairs_per_accumulator": _lib.get_option("similarity_superpose_last"),
       "candidates": _lib.get_option("similarity_candidates_last"), "tiles": int(tiles),
       "device": torch.cuda.get_device_name(0)})
labels = ["tile metadata wait", "fullBar wait", "wgmma wait", "pre-filter", "candidates"]
loop = v[6] / warp_tiles
print(f"consumer warp, clk/tile (of {loop:.0f}):")
for k, name in enumerate(labels):
    print(f"   {name:22s} {v[k] / warp_tiles:9.0f}   {100 * v[k] / v[6]:5.1f} %")
rest = v[6] - v[:5].sum()
print(f"   {'everything else':22s} {rest / warp_tiles:9.0f}   {100 * rest / v[6]:5.1f} %")
print(f"producer, emptyBar wait clk/tile {v[7] / tiles:9.0f}")
