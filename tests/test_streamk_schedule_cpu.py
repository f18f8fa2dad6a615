"""Host logic of the stream-K schedule of csrc/conv2d_tc.cu (no GPU): the partition of the tile-major (tile, K-step) list into one
contiguous range per cluster, through the library's own rule (dvd_conv2d_streamk_bounds = SegIter::bound on the host).

Invariants the kernel's exchange protocol relies on:
  * ranges are monotone, cover every K-step of every tile exactly once, and range boundaries within 1/8 of a tile boundary snap to it;
  * a cluster delivers at most ONE partial tile (the first segment of its range, when that range starts inside a tile);
  * the cluster that owns the first K-steps of a split tile finds exactly the clusters whose ranges BEGIN inside that tile as its
    contributors (the kernel counts them with the same rule), so every raised flag is consumed and lowered in the same launch."""
import ctypes
import random

import pytest


def _bounds(ntiles, ksteps, n):
    from dvd_b200 import _lib
    out = (ctypes.c_long * (n + 1))()
    _lib.check(_lib.load().dvd_conv2d_streamk_bounds(ntiles, ksteps, n, out), 'bounds')
    return list(out)


def _check(ntiles, ksteps, n):
    b = _bounds(ntiles, ksteps, n)
    total = ntiles * ksteps
    assert b[0] == 0 and b[-1] == total and all(b[i] <= b[i + 1] for i in range(n))
    for u in b:
        r = u % ksteps
        assert r == 0 or (r * 8 >= ksteps and (ksteps - r) * 8 >= ksteps), (u, ksteps)       # slivers are snapped away
    flags, owners, cover = {}, [], {}
    for c in range(n):
        u, u1 = b[c], b[c + 1]
        first = True
        while u < u1:
            t, k0 = divmod(u, ksteps)
            k1 = min(ksteps, k0 + (u1 - u))
            cover.setdefault(t, []).append((k0, k1))
            if k0 > 0:
                assert first and c not in flags     # only the first segment of a range can be a partial tile
                flags[c] = t
            elif k1 < ksteps:
                npart = 0
                while c + 1 + npart < n and b[c + 1 + npart] < (t + 1) * ksteps:
                    npart += 1
                owners.append((c, t, npart))
            u += k1 - k0
            first = False
    for c, t, npart in owners:
        assert npart >= 1
        for p in range(npart):
            assert flags.pop(c + 1 + p) == t
    assert not flags
    for t in range(ntiles):
        pos = 0
        for k0, k1 in sorted(cover[t]):
            assert k0 == pos
            pos = k1
        assert pos == ksteps


# (tiles, K-steps, CTAs). The H100 launch runs one CTA per SM (up to 132) and at most max(8, K-steps / 4) K-steps per range:
#   layer4_rn (3x3, 2048 -> 256, one 256-channel tile per image) at the bench batch 16 x 7 x 12: 16 tiles over 64 CTAs;
#   at the 1 x 12 / 12 x 1 layer4 grids of 32 x 384 / 384 x 32 images (one tile per image): 2 tiles over 8 CTAs;
#   at the 1 x 1 grid of a 32 x 32 image: 1 tile over 4 CTAs (4 images: 4 tiles over 16);
#   layer3_rn (3x3, 1024 -> 256) at the bench batch 16 x 14 x 24: 48 tiles, 288 K-steps over 132 CTAs;
#   the data gradient of a 3x3 256 -> 2048 convolution at a 1 x 1 grid (2048 input channels): 1 tile over 4 CTAs.
H100_LAYERS = [(16, 576, 64), (2, 576, 8), (1, 576, 4), (4, 576, 16), (48, 288, 132), (132, 576, 132), (133, 1152, 132)]


@pytest.mark.parametrize('shape', [(84, 32, 74), (6, 576, 74), (24, 288, 74), (1, 64, 4), (48, 64, 74), (168, 16, 74), (11, 8, 11),
                                   (3, 9, 2)] + H100_LAYERS)
def test_partition_of_the_layers_of_the_depth_net(shape):
    _check(*shape)


def test_partition_invariants_on_random_shapes():
    rnd = random.Random(0)
    done = 0
    while done < 3000:
        ks, n, nt = rnd.randint(1, 1152), rnd.randint(1, 132), rnd.randint(1, 400)
        if nt * ks < n:
            continue
        _check(nt, ks, n)
        done += 1
