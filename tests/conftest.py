import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "dcscn-super-resolution_b200")
for p in (PKG, os.path.join(ROOT, "oracle"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (select with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


def load_golden_weights(name):
    from helper import tf_bundle
    r = tf_bundle.BundleReader(os.path.join(GOLDEN, "models", name + ".ckpt"))
    return {k: r.get_tensor(k) for k in r.keys()}


MODEL_FLAGS = {
    # model name -> (oracle/engine config kwargs)
    "dcscn_L12_F196to48_NIN_A64_PS_R1F32": dict(),
    "dcscn_L12_F196to48_Sc4_NIN_A64_PS_R1F32": dict(scale=4),
    "dcscn_L12_F196to48_Sc3_NIN_A64_PS_R1F32": dict(scale=3),
    "dcscn_L8_F96to48_NIN_A64_PS_R1F32": dict(layers=8, filters=96),
    "dcscn_L8_F96to48_Sc3_NIN_A64_PS_R1F32": dict(scale=3, layers=8, filters=96),
    "dcscn_L8_F96to48_Sc4_NIN_A64_PS_R1F32": dict(scale=4, layers=8, filters=96),
    "dcscn_L7_F32to8_G1.20_NIN_A24_B8_PS_R1F32": dict(
        scale=2, layers=7, filters=32, min_filters=8, filters_decay_gamma=1.2, nin_filters=24, nin_filters2=8,
        reconstruct_layers=0, pixel_shuffler_filters=1),
    "dcscn_L7_F32to8_G1.20_Sc3_NIN_A24_B8_PS_R1F32": dict(
        scale=3, layers=7, filters=32, min_filters=8, filters_decay_gamma=1.2, nin_filters=24, nin_filters2=8,
        reconstruct_layers=0, pixel_shuffler_filters=1),
    "dcscn_L7_F32to8_G1.20_Sc4_NIN_A24_B8_PS_R1F32": dict(
        scale=4, layers=7, filters=32, min_filters=8, filters_decay_gamma=1.2, nin_filters=24, nin_filters2=8,
        reconstruct_layers=0, pixel_shuffler_filters=1),
    "dcscn_L7_F32to8_G1.20_Sc4_NIN_A24_B8_PS_DS_R1F32": dict(
        scale=4, layers=7, filters=32, min_filters=8, filters_decay_gamma=1.2, nin_filters=24, nin_filters2=8,
        reconstruct_layers=0, pixel_shuffler_filters=1, depthwise_separable=True),
}
