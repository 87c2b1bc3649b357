"""compute-sanitizer target: one reduced C4 bottom-up step (256x256 frames, the C4 network) with the fused first block
on and off, in precision 0 and in the split-fp16 precision 2, so that every hand-written mbarrier / TMA / wgmma pipeline,
the split stores and k_head_1x1 run under memcheck / racecheck in minutes.  `quick`: the fused block in precision 0 only.
Usage: compute-sanitizer --tool memcheck python tools/sanitize_step.py [quick]"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = r'''
import os, sys
sys.path.insert(0, %r)
import numpy as np
import bench
from sleap_b200.nn import architectures as A
from sleap_b200.nn.inference import BottomUpPredictor
from sleap_b200.nn.model import DeviceModel
spec = bench.c4_spec()
w = A.make_synthetic_weights(A.compile_model(spec, 1), bench.SEED)
m = DeviceModel(spec, w, input_channels=1, precision=int(os.environ.get("SB_SAN_PRECISION", "0")))
fr = np.random.default_rng(0).integers(0, 256, size=(2, 256, 256, 1), dtype=np.uint8)
cms, _ = m.forward(fr)
p = BottomUpPredictor(m, bench.NODES, bench.EDGES, peak_threshold=float(np.quantile(cms, 0.999)), batch_size=2,
                      max_peaks_per_sample=2048, max_node_peaks=64, max_instances_per_frame=64)
out = p.predict(np.concatenate([fr, fr]), make_labels=False)
print("conv01", os.environ.get("SB_FORCE_CONV01"), "precision", os.environ.get("SB_SAN_PRECISION", "0"),
      "ok", int(sum(o["n_valid"].sum() for o in out)))
''' % ROOT

if __name__ == "__main__":
    quick = len(sys.argv) > 1 and sys.argv[1] == "quick"
    combos = [("1", "0")] if quick else [("1", "0"), ("0", "0"), ("0", "2")]
    for c, prec in combos:
        env = dict(os.environ, SB_FORCE_CONV01=c, SB_SAN_PRECISION=prec)
        r = subprocess.run([sys.executable, "-c", CHILD], env=env)
        if r.returncode:
            sys.exit(r.returncode)
