"""Per-launch times of the depthwise-separable c-DCSCN x4 graph (BASELINE.json configs[4]), 256 tiles of 48x48."""
import os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "dcscn-super-resolution_b200"))
from helper import engine as E, tf_bundle
r = tf_bundle.BundleReader(os.path.join(ROOT, "tests", "golden", "models", "dcscn_L7_F32to8_G1.20_Sc4_NIN_A24_B8_PS_DS_R1F32.ckpt"))
eng = E.Engine(E.make_config(scale=4, layers=7, filters=32, min_filters=8, filters_decay_gamma=1.2, nin_filters=24, nin_filters2=8,
                             reconstruct_layers=0, pixel_shuffler_filters=1, depthwise_separable=1))
eng.set_params({k: r.get_tensor(k) for k in r.keys()})
g = torch.Generator().manual_seed(2)
x = (torch.rand(256, 48, 48, 1, generator=g) * 255).cuda(); x2 = (torch.rand(256, 192, 192, 1, generator=g) * 255).cuda()
y = torch.empty_like(x2)
eng.set_option("timing", 1)
for _ in range(2):
    for _ in range(3): eng.forward(x, x2, y)
    torch.cuda.synchronize()
    tm = eng.timings()
    print("total %.3f ms  " % sum(t for _, t in tm) + " ".join("%s=%.3f" % (name, t) for name, t in tm))
