"""Development helper for torch.profiler: train steps of a bench workload with eager launches (no CUDA graph).
usage: python tools/one_step.py [batch] [steps] [config]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from bench import WORKLOADS, WEIGHTS, workload_inputs
from deepsvg_b200 import SVGLoss, SVGTransformer, _lib
from deepsvg_b200.config import Hierarchical, OneStageOneShot
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
name = sys.argv[3] if len(sys.argv) > 3 else "hier"
wl = WORKLOADS[name]
B = int(sys.argv[1]) if len(sys.argv) > 1 and int(sys.argv[1]) > 0 else wl["batch"]
dev = "cuda:0"
cfg = (Hierarchical if wl["kind"] == "hierarchical" else OneStageOneShot)(**wl["over"])
torch.manual_seed(0)
model = SVGTransformer(cfg, precision=os.environ.get("DSVG_PRECISION", "bf16"), graphs=False).to(dev).train()
loss_fn = SVGLoss(cfg).to(dev)
c, a, lab = workload_inputs(wl, B, seed=1)
c, a = c.to(dev), a.to(dev)
lab = lab.to(dev) if lab is not None else None
for i in range(steps):
    l0 = _lib.launch_count()
    model.zero_grad(set_to_none=True)
    out = model(c, a, c, a, label=lab, params={})
    ls = loss_fn(out, None, weights=WEIGHTS)
    ls["loss"].backward()
    torch.cuda.synchronize()
    print("step", i, "launches", _lib.launch_count() - l0, "loss", ls["loss"].item(), flush=True)
