"""L2 -> shared-memory bytes of the tensor-core conv launches of one bench.py headline step (DCSCN L12 x2, 256 tiles of
48 x 48, f16x3 = two fp16 planes, 64-channel chunks), counted from the shapes the engine plans: activations and weights,
per layer, before (one 8 x 16-pixel patch's TW x (TH + 2) box per (chunk, kx) serving the three ky taps) and after
(one (TW + 2) x (TH + 2) box of a 16 x 8 patch per chunk serving all nine taps, where two such boxes fit beside three
weight tiles: engine.cu tc_chunk_box).  usage: python scripts/l2_bytes.py"""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import dcscn_oracle as O  # noqa: E402

N_IMG, H, W = 256, 48, 48
TH, TW = 8, 16                 # choose_patch's tile for 48 x 48 without a chunk box
CTH, CTW = 16, 8               # and with one
KC, PLANES, EL = 64, 2, 2      # channels per chunk, hi/lo planes, bytes per fp16
CAP = 112                      # column tile cap (kMaxTileN)


def chunk_box(k, n_pad):
    """engine.cu tc_chunk_box at f16x3: two chunk boxes beside three weight tiles in the ring budget."""
    if k == 1:
        return False
    budget = 227 * 1024 - 1024 - (2 * (4 + 12) + 2) * 8 - 128 * (n_pad + 8) * 4
    plane = ((CTW + k - 1) * (CTH + k - 1) * KC * EL + 1023) // 1024 * 1024
    return 2 * PLANES * plane + 3 * PLANES * n_pad * KC * EL <= budget


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

    rows = []
    for i in range(1, len(feat)):
        rows.append(("CNN%d" % (i + 1), 3, pad16(feat[i - 1]), tiling(feat[i], CAP)))
    rows.append(("A1+B1", 1, sum(pad16(f) for f in feat), tiling(cfg.nin_filters + cfg.nin_filters2, CAP)))
    rows.append(("B2", 3, pad16(cfg.nin_filters2), tiling(cfg.nin_filters2, CAP)))
    cin = cfg.nin_filters + cfg.nin_filters2
    rows.append(("Up-PS", 3, pad16(cin), tiling(cfg.scale * cfg.scale * cin, CAP, unit=cin)))

    print("%-7s %3s %5s %10s %4s %10s %10s %10s" % ("layer", "k", "cin", "tiles", "box", "A before", "A after", "W"))
    tot = [0.0] * 3
    for name, k, cin_pad, (nt, np_) in rows:
        chunks = (cin_pad + KC - 1) // KC
        tiles = N_IMG * ((H + TH - 1) // TH) * ((W + TW - 1) // TW)
        a0 = tiles * nt * k * chunks * PLANES * TW * (TH + k - 1) * KC * EL
        cb = chunk_box(k, np_)
        if cb:
            ctiles = N_IMG * ((H + CTH - 1) // CTH) * ((W + CTW - 1) // CTW)
            a1 = ctiles * nt * chunks * PLANES * (CTW + k - 1) * (CTH + k - 1) * KC * EL
        else:
            a1 = a0
        w = tiles * nt * k * k * chunks * PLANES * np_ * KC * EL
        for j, v in enumerate((a0, a1, w)):
            tot[j] += v
        print("%-7s %3d %5d %4d x %3d %4s %7.2f GB %7.2f GB %7.2f GB" % (name, k, cin_pad, nt, np_, "yes" if cb else "-",
                                                                     a0 / 1e9, a1 / 1e9, w / 1e9))
    print("%-7s %25s %7.2f GB %7.2f GB %7.2f GB" % ("sum", "", *(v / 1e9 for v in tot)))
    print("total L2->SM per step: before %.1f GB, after %.1f GB" % ((tot[0] + tot[2]) / 1e9, (tot[1] + tot[2]) / 1e9))


if __name__ == "__main__":
    main()
