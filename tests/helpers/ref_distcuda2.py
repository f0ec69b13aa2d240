"""Run with a stack's PYTHONPATH (tests/scripts_harness.py): distCUDA2 from that stack's `simple_knn._C` on every [P,3] array of an
.npz, written to another .npz under the same keys, plus
"__module__": the file the extension module was loaded from.  Under the stock stack this is the reference's own extension."""
import sys

import numpy as np
import torch

import simple_knn._C
from simple_knn._C import distCUDA2

src, dst = sys.argv[1], sys.argv[2]
out = {"__module__": np.array(simple_knn._C.__file__)}
with np.load(src) as f:
    for k in f.files:
        out[k] = distCUDA2(torch.from_numpy(f[k]).cuda()).cpu().numpy()
np.savez(dst, **out)
