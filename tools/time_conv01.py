"""Configure the C4 model (autotune prints the fused first block's time with SB_DEBUG=1)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import bench
from sleap_b200.nn import architectures as A
from sleap_b200.nn.model import DeviceModel
spec = bench.c4_spec()
w = A.make_synthetic_weights(A.compile_model(spec, 1), bench.SEED)
m = DeviceModel(spec, w, input_channels=1, precision=0)
m.configure(8, 1024, 1024, 1)
