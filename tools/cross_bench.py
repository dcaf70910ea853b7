"""Materialised cross-similarity timings (BASELINE config 1 = 1k x 1k, and larger squares): kernel time from the library's
CUDA events, algorithmic bytes 8 B/pair + 256 B/fingerprint (SURVEY.md 8d).   python tools/cross_bench.py [sizes ...]"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from nvmolkit_b200 import _lib, synthetic  # noqa: E402
from nvmolkit_b200.similarity import crossTanimotoSimilarity  # noqa: E402

sizes = [int(a) for a in sys.argv[1:]] or [1000, 4096, 16384, 32768]
_lib.profile_enable(True)
if os.environ.get("B200_MIN_PAIRS"):  # e.g. 0: the tensor tile for every size (default: from 2^24 pairs up)
    _lib.set_option("similarity_tensor_min_pairs", int(os.environ["B200_MIN_PAIRS"]))
peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 6650.0
for n in sizes:
    a = torch.from_numpy(synthetic.random_fingerprints(n, seed=1, near_dups=n // 8).view(np.int32)).cuda()
    b = torch.from_numpy(synthetic.random_fingerprints(n, seed=2, near_dups=n // 8).view(np.int32)).cuda()
    for _ in range(3):
        out = crossTanimotoSimilarity(a, b)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 10
    e0.record()
    for _ in range(reps):
        out = crossTanimotoSimilarity(a, b)
    e1.record()
    torch.cuda.synchronize()
    ms_call = e0.elapsed_time(e1) / reps
    try:
        ms_k, phase = _lib.profile_read("cross_tc"), "cross_tc (wgmma u8 tensor-core tile)"
    except ValueError:
        ms_k, phase = ms_call, "whole call (SIMT popcount tile; below similarity_tensor_min_pairs)"
    bytes_ = 8.0 * n * n + 512.0 * n
    print(json.dumps({"shape": [n, n], "ms_per_call": ms_call, "kernel_ms": ms_k, "timed": phase, "pairs_per_s": n * n / (ms_call * 1e-3),
                      "algorithmic_GBps_call": bytes_ / (ms_call * 1e-3) / 1e9, "algorithmic_GBps_kernel": bytes_ / (ms_k * 1e-3) / 1e9,
                      "frac_of_hbm_kernel": bytes_ / (ms_k * 1e-3) / 1e9 / peak}))
    del out
