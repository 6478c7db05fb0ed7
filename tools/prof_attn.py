"""Runs the L0 spatial attention (with reference-KV concat) a few times -- target of `ncu -k regex:attn_tc`."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hallo_b200 import ops  # noqa: E402

C, L, frames = int(os.environ.get("C", 320)), int(os.environ.get("L", 4096)), int(os.environ.get("FRAMES", 32))
dev = "cuda"
qkv = torch.randn(frames * L, 3 * C, device=dev, dtype=torch.float16)
kvr = torch.randn(2 * L, 2 * C, device=dev, dtype=torch.float16)
o = torch.empty(frames * L, C, device=dev, dtype=torch.float16)
ridx = torch.tensor([-1] * (frames // 2) + [n % 2 for n in range(frames // 2)], dtype=torch.int32, device=dev)
for _ in range(int(os.environ.get("REPS", 3))):
    ops.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], o, heads=8, L=L, kref=kvr[:, :C], vref=kvr[:, C:],
                  ref_index=ridx)
torch.cuda.synchronize()
print("done")
