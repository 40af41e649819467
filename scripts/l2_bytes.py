"""L2 -> shared-memory bytes of the tensor-core conv launches of one bench.py headline step (DCSCN L12 x2, 256 tiles of
48 x 48, f16x3 = two fp16 planes, 64-channel chunks), counted from the shapes the engine plans: activations and weights,
per layer, before (one 128-pixel box per (tap, chunk), column tiles up to 128 wide) and after (one TW x (TH + 2)-pixel
box per (chunk, kx) serving all three ky taps, column tiles up to 112 wide).  usage: python scripts/l2_bytes.py"""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import dcscn_oracle as O  # noqa: E402

N_IMG, H, W = 256, 48, 48
TH, TW = 8, 16                 # choose_patch's tile for 48 x 48
KC, PLANES, EL = 64, 2, 2      # channels per chunk, hi/lo planes, bytes per fp16


def pad16(x):
    return (x + 15) // 16 * 16


def tiling(cols, cap, unit=0):
    """Column tiles of a layer (engine.cu choose_tiling; the last pixel shuffler keeps whole sub-pixels per tile)."""
    c = pad16(cols)
    nt = (c + cap - 1) // cap
    np_ = pad16((c + nt - 1) // nt)
    if unit and cols % unit == 0 and np_ % unit:
        np_ = cap // unit * unit
        nt = (cols + np_ - 1) // np_
    return nt, np_


def main():
    cfg = O.OracleConfig()
    feat = O.feature_filters(cfg)

    def layers(cap):
        rows = []
        for i in range(1, len(feat)):
            rows.append(("CNN%d" % (i + 1), 3, pad16(feat[i - 1]), tiling(feat[i], cap)))
        rows.append(("A1+B1", 1, sum(pad16(f) for f in feat), tiling(cfg.nin_filters + cfg.nin_filters2, cap)))
        rows.append(("B2", 3, pad16(cfg.nin_filters2), tiling(cfg.nin_filters2, cap)))
        cin = cfg.nin_filters + cfg.nin_filters2
        rows.append(("Up-PS", 3, pad16(cin), tiling(cfg.scale * cfg.scale * cin, cap, unit=cin)))
        return rows

    tiles = N_IMG * ((H + TH - 1) // TH) * ((W + TW - 1) // TW)
    print("%-7s %3s %5s %10s %10s %10s %10s %10s" % ("layer", "k", "cin", "tiles", "A before", "W before", "A after",
                                                     "W after"))
    tot = [0.0] * 4
    for (name, k, cin_pad, (nt0, np0)), (_, _, _, (nt1, np1)) in zip(layers(128), layers(112)):
        chunks = (cin_pad + KC - 1) // KC
        a0 = tiles * nt0 * k * k * chunks * PLANES * TH * TW * KC * EL
        w0 = tiles * nt0 * k * k * chunks * PLANES * np0 * KC * EL
        a1 = tiles * nt1 * k * chunks * PLANES * TW * (TH + k - 1) * KC * EL
        w1 = tiles * nt1 * k * k * chunks * PLANES * np1 * KC * EL
        for j, v in enumerate((a0, w0, a1, w1)):
            tot[j] += v
        print("%-7s %3d %5d %4d x %3d %7.2f GB %7.2f GB %7.2f GB %7.2f GB" % (name, k, cin_pad, nt1, np1, a0 / 1e9, w0 / 1e9,
                                                                          a1 / 1e9, w1 / 1e9))
    print("%-7s %20s %7.2f GB %7.2f GB %7.2f GB %7.2f GB" % ("sum", "", *(v / 1e9 for v in tot)))
    print("total L2->SM per step: before %.1f GB, after %.1f GB" % ((tot[0] + tot[1]) / 1e9, (tot[2] + tot[3]) / 1e9))


if __name__ == "__main__":
    main()
