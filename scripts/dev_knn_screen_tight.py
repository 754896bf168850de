"""How tight the kNN tile screen's bound u(q) is, and what it saves, on the bench workload's own X_pca (1.3M x 50, k = 15).

u(q) comes from a cold short sweep of each query block over SB2_KNN_NEAR consecutive tiles of the kd order; 8, 16,
32 and 64 (the default) are compared.  Per setting:
  - the kept fraction of (block, tile) pairs (the screen's lists, sb2_knn_debug_screen_f32);
  - from one SB2_KNN_STAMPS=1 run: the screen's line (ms of each part) and the sweep's (cycles per tile, insertions per row);
  - pass1_ms (CUDA events around the whole kNN first pass, screen included) over --rounds alternated rounds, and that
    (idx, dist) are bit-identical between the settings.
Then, for the default's u(q), the screen's keep test restated in float64 (exact tile means and radii, no
rounding slack) at 128-row and at 64-row granularity: (block, tile) pairs against (half-block, tile) pairs, the halves
taken as they are now (each 64-row half of a 128-point leaf is in index order, so a random half) and as 64-point leaves
(each leaf split at the median of its own largest-variance coordinate).  The 64-row lists are worth building only if
the halves visit clearly fewer tiles than 2 x the blocks.
Last, --rounds of pass1_ms on unclustered data (uniform and Gaussian, --n x 50) with 8 and 64 near tiles: where the
screen gives up (too few tiles skipped) the wider short sweep is pure cost.  Prints the card name and power limit.

    python scripts/dev_knn_screen_tight.py [--n 1300000] [--rounds 3]
"""
import argparse
import os
import re
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402

from dev_knn_screen import card, stamped  # noqa: E402
from scanpy_b200 import _abi, _ops  # noqa: E402
from scanpy_b200._synth import synth_scipy  # noqa: E402

SETTINGS = {
    "near8": {"SB2_KNN_NEAR": "8"},
    "near16": {"SB2_KNN_NEAR": "16"},
    "near32": {"SB2_KNN_NEAR": "32"},
    "near64": {},
}


def use(env):
    for key in ("SB2_KNN_NEAR", "SB2_KNN_STAMPS"):
        os.environ.pop(key, None)
    os.environ.update(env)


def debug_screen(ctx, xp, k):
    n, d = xp.shape
    nb = (n + 127) // 128
    perm = torch.empty(n, dtype=torch.int32, device="cuda")
    lists = torch.empty(nb * nb, dtype=torch.int32, device="cuda")
    lens = torch.empty(nb, dtype=torch.int32, device="cuda")
    ub = torch.empty(n, dtype=torch.float32, device="cuda")
    _ops.check(ctx.lib.sb2_knn_debug_screen_f32(ctx.handle, n, d, _ops.ptr(xp), k, _ops.ptr(perm), _ops.ptr(lists),
                                                _ops.ptr(lens), _ops.ptr(ub)))
    del lists
    return perm.long(), lens, ub


def halves_kept(xp, perm, ub, chunk_blocks=32):
    """float64 restatement of the keep test |q - mu_t| - r_t <= u(q): kept (block, tile) pairs, kept (half, tile) pairs
    with the halves of the current order, and with 64-point leaves"""
    n, d = xp.shape
    nb = (n + 127) // 128
    x = xp.double()[perm]
    pad = nb * 128 - n
    xt = torch.cat([x, x[-1:].expand(pad, d)]) if pad else x            # the tiles: padding repeats the last point
    cnt = torch.full((nb,), 128, device="cuda", dtype=torch.float64)
    cnt[-1] = 128 - pad
    valid = (torch.arange(nb * 128, device="cuda") < n).view(nb, 128)
    mu = (xt.view(nb, 128, d) * valid[..., None]).sum(1) / cnt[:, None]
    rad = (((xt.view(nb, 128, d) - mu[:, None, :]) ** 2).sum(-1).sqrt() * valid).amax(1)
    mu2 = (mu ** 2).sum(1)
    # 64-point leaves: each 128-point leaf of the query order split at the median of its largest-variance coordinate
    xb = xt.view(nb, 128, d)
    var = ((xb - mu[:, None, :]) ** 2 * valid[..., None]).sum(1)
    axis = var.argmax(1)
    key = torch.gather(xb, 2, axis[:, None, None].expand(nb, 128, 1))[..., 0]
    key = torch.where(valid, key, torch.full_like(key, float("inf")))   # padding rows last
    leaf = torch.sort(key, dim=1, stable=True).indices                   # row order within each block
    u = torch.cat([ub.double(), torch.full((pad,), float("-inf"), device="cuda", dtype=torch.float64)])
    k128 = k64 = k64l = 0
    for b0 in range(0, nb, chunk_blocks):
        b1 = min(nb, b0 + chunk_blocks)
        q = xt[b0 * 128:b1 * 128]
        d2 = (q ** 2).sum(1)[:, None] + mu2[None, :] - 2.0 * q @ mu.T
        keep = (d2.clamp_min(0).sqrt() - rad[None, :]) <= u[b0 * 128:b1 * 128, None]
        nbc = b1 - b0
        kb = keep.view(nbc, 128, nb)
        k128 += int(kb.any(1).sum())
        k64 += int(kb.view(nbc, 2, 64, nb).any(2).sum())
        kl = torch.gather(kb, 1, leaf[b0:b1, :, None].expand(nbc, 128, nb))
        k64l += int(kl.view(nbc, 2, 64, nb).any(2).sum())
    return nb, k128, k64, k64l


def timed_rounds(ctx, xp, k, settings, rounds):
    ms = {s: [] for s in settings}
    ref = {}
    for r in range(rounds + 1):        # round 0 warms every setting up
        for s in settings:
            use(SETTINGS[s])
            idx, dist, info = _ops.knn_device(ctx, xp, k)
            torch.cuda.synchronize()
            if r == 0:
                ref[s] = (idx.clone(), dist.clone())
            else:
                ms[s].append(info["pass1_ms"])
    i0, d0 = ref[settings[0]]
    same = all(torch.equal(i0, ref[s][0]) and torch.equal(d0, ref[s][1]) for s in settings)
    return ms, same


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=1_300_000)
    p.add_argument("--genes", type=int, default=2000)
    p.add_argument("--k", type=int, default=15)
    p.add_argument("--rounds", type=int, default=3)
    a = p.parse_args()
    print("card:", card(), flush=True)
    x, _ = synth_scipy(a.n, a.genes, device="cuda")
    ctx = _abi.default_context()
    ip, ix, dat = _ops.csr_to_device(x)
    xp = _ops.pca_csr_device(ctx, ip, ix, dat, a.n, a.genes, 50, solver=1)["X_pca"].contiguous()
    print(f"X_pca {tuple(xp.shape)}", flush=True)
    names = list(SETTINGS)
    for s in names:
        use(SETTINGS[s])
        perm, lens, ub = debug_screen(ctx, xp, a.k)
        nb = lens.numel()
        print(f"{s}: kept (block, tile) pairs {float(lens.double().sum()) / nb / nb:.4f}, median u {float(ub.median()):.4f}",
              flush=True)
        for ln in stamped(ctx, xp, a.k):
            m = re.search(r"(\d+) cycles/tile.*insertions/row ([\d.]+)", ln)
            print(f"{s} {ln}" + (f"  => cycles/tile {m.group(1)}, insertions/row {m.group(2)}" if m else ""), flush=True)
        if s == "near64":
            nb, k128, k64, k64l = halves_kept(xp, perm, ub)
            print(f"{s} float64 keep test: (block, tile) kept {k128 / nb / nb:.4f}; (64-row half, tile) visits / (2 x block visits): "
                  f"current halves {k64 / (2 * k128):.4f}, 64-point leaves {k64l / (2 * k128):.4f}", flush=True)
    ms, same = timed_rounds(ctx, xp, a.k, names, a.rounds)
    for s in names:
        v = np.array(ms[s])
        print(f"{s}: pass1_ms median {np.median(v):.1f} min {v.min():.1f} max {v.max():.1f} over {len(v)} rounds", flush=True)
    print(f"(idx, dist) bit-identical across {names}: {same}", flush=True)
    rs = torch.Generator(device="cuda").manual_seed(0)
    for kind in ("uniform", "gauss"):
        shape = (a.n, 50)
        y = (torch.rand(shape, generator=rs, device="cuda") * 2 - 1) if kind == "uniform" else torch.randn(shape, generator=rs, device="cuda")
        yms, ysame = timed_rounds(ctx, y.contiguous(), a.k, ["near8", "near64"], a.rounds)
        use(SETTINGS["near64"])
        line = [ln for ln in stamped(ctx, y.contiguous(), a.k) if ln.startswith("[sb2 knn screen]")]
        print(f"{kind} {a.n} x 50: 8 near tiles median {np.median(yms['near8']):.1f} ms, 64 median {np.median(yms['near64']):.1f} ms "
              f"(min {min(yms['near8']):.1f} / {min(yms['near64']):.1f}); identical {ysame}; {line[0] if line else ''}", flush=True)
        assert ysame
    use({})
    print("card:", card(), flush=True)
    assert same


if __name__ == "__main__":
    main()
