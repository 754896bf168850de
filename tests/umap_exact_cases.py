"""The cases on which the device UMAP layout is compared with its float64 restatement (tests/test_gpu_umap_exact.py) and
on which the comparison tolerance is shown to reject a wrong schedule (tests/test_umap_schedule_cpu.py): one table, so
every device case is also a mutation case.

The layout is chaotic at the default learning rate: a rounding difference grows by orders of magnitude per epoch.  So
runs at initial_alpha = 1 stop at 3 epochs, 5-epoch runs use 0.2 and longer runs 0.01 or less."""
from functools import lru_cache

import numpy as np

from oracle import umap_schedule as us

A, B = 0.5830300, 1.3341669  # find_ab_params(1.0, 0.5), sc.tl.umap's defaults
GRAPHS = {"small": (400, 0), "mid": (2000, 300), "big": (12000, 600)}  # (n, hub degree); "big": n > 10000


def _case(cid, graph="mid", dim=2, init_seed=2, const_col=None, **kw):
    kw = dict(dict(n_epochs=3, gamma=1.0, initial_alpha=1.0, negative_sample_rate=5, seed=7), **kw)
    return dict(id=cid, graph=graph, dim=dim, init_seed=init_seed, const_col=const_col, kw=kw)


CASES = (
    [_case(f"dim={d}", graph="small", dim=d, init_seed=d) for d in range(1, 17)]
    + [_case(f"{g} n_epochs={ne}", graph=g, n_epochs=ne, initial_alpha=0.2 if ne == 5 else 1.0)
       for g in ("mid", "big") for ne in (0, 1, 2, 3, 5)]
    # 70 owes 69-70 negatives per sample; the kernel clamps to 64 (a deliberate bound that umap does not have)
    + [_case(f"negative_sample_rate={r}", negative_sample_rate=r) for r in (0, 1, 5, 70)]
    # rate 7 over 91 epochs reaches the arcs of eps 5 (epochs 45, 90) and eps 10 (epoch 90) where epoch * rate / eps is
    # an integer that epoch * (rate / eps) rounds below
    + [_case("negative_sample_rate=7 91 epochs alpha=0.003", negative_sample_rate=7, n_epochs=91, initial_alpha=0.003)]
    + [_case("gamma=2.5 alpha=0.5", gamma=2.5, initial_alpha=0.5),
       _case("gamma=0.3 alpha=0.01 50 epochs", gamma=0.3, initial_alpha=0.01, n_epochs=50),
       _case("seed=2**32+99", seed=2**32 + 99),
       _case("seed=99", seed=99),
       _case("constant column, 1 epoch", dim=3, const_col=1, n_epochs=1),
       _case("constant column, 3 epochs", dim=3, const_col=1, n_epochs=3)]
)
IDS = [c["id"] for c in CASES]


@lru_cache(maxsize=None)
def graph(name):
    n, hub = GRAPHS[name]
    return us.edge_case_graph(n, seed=0, hub_degree=hub)


def init(case):
    x = np.random.default_rng(case["init_seed"]).normal(size=(GRAPHS[case["graph"]][0], case["dim"])).astype(np.float32)
    if case["const_col"] is not None:
        x[:, case["const_col"]] = 4.25  # the rescale maps a constant column to 0
    return x


def restated(case, dtype=np.float64, **mutation):
    return us.umap_layout(graph(case["graph"]), init(case), a=A, b=B, dtype=dtype, **case["kw"], **mutation)
