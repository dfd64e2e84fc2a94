"""Small, fixed workloads to capture with ncu (one kernel family per invocation, few launches):
    ncu --set full --clock-control none --import-source on -k regex:<kernel> -c <n> -o gpurun_out/<name> python tools/prof_targets.py <target>
targets: hogwild (C2), hogwild_large (1M x 2M items), score_c2, score_c5, vae (C3 step: gemm_tc_kernel at the three I-sized shapes,
vae_softmax_kernel), reconcile (single GPU, 2 replicas).  Not the bench contract; numbers printed here are not bench values."""
import sys

import torch

sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
from elliot_b200 import ops                                                            # noqa: E402

dev = "cuda:0"
what = sys.argv[1] if len(sys.argv) > 1 else "hogwild"
HP = (0.05, 0.0025, 0.0, 0.0025, 0.00025)


def csr(nu, ni, per, seed):
    g = torch.Generator(device=dev); g.manual_seed(seed)
    cand = (torch.rand(nu, per, device=dev, generator=g) ** 2 * ni).to(torch.int32).clamp_(max=ni - 1)
    cand, _ = torch.sort(cand, dim=1)
    keep = torch.ones_like(cand, dtype=torch.bool); keep[:, 1:] = cand[:, 1:] != cand[:, :-1]
    indptr = torch.zeros(nu + 1, dtype=torch.int64, device=dev); indptr[1:] = torch.cumsum(keep.sum(1), 0)
    return indptr, cand[keep].contiguous()


if what in ("hogwild", "hogwild_large"):
    nu, ni, d, B = 1_000_000, (100_000 if what == "hogwild" else 2_000_000), 64, 1 << 22
    U = torch.randn(nu, d, device=dev) * 0.1; V = torch.randn(ni, d, device=dev) * 0.1; b = torch.zeros(ni, device=dev)
    ip, ix = csr(nu, ni, 100, 100)
    f = ops.bloom_build(ip, ix, nu) if what == "hogwild_large" else None      # as in bench.py: signatures only on the large catalogue
    for s in range(5):
        ops.bpr_step_sampled_f32(U, V, b, d, nu, ni, ip, ix, B, 42, s * B, *HP, filter=f)
    torch.cuda.synchronize()
elif what in ("score_c2", "score_c5"):
    nu = 132 * 128 * 2
    ni, d = (100_000, 64) if what == "score_c2" else (2_000_000, 128)
    U = torch.randn(nu, d, device=dev) * 0.1; V = torch.randn(ni, d, device=dev) * 0.1; b = torch.randn(ni, device=dev) * 0.05
    ip, ix = csr(nu, ni, 100, 5)
    for _ in range(3):
        _, _, st = ops.score_topk_tc(U, V, b, d, 10, ip, ix)
    torch.cuda.synchronize()
    print(what, st)
elif what == "vae":
    from elliot_b200.recommender.multi_vae import VariationalAutoEncoder
    nu, ni, B = 138_493, 26_744, 512
    ip, ix = csr(nu, ni, 144, 900)
    m = VariationalAutoEncoder(ni, 600, 200, 1e-3, 0.5, 0.01, 42, ip, ix, dev)
    rows = torch.randperm(nu, device=dev)[:B].to(torch.int32)
    for _ in range(3):
        m.train_step(rows, 0.1)
    torch.cuda.synchronize()
elif what == "reconcile":
    n = 100_000 * 65
    reps = [torch.randn(n, device=dev) for _ in range(2)]
    prev = reps[0].clone(); reps[1].copy_(reps[0])
    for _ in range(3):
        for t in reps:
            t.add_(1e-3)
        ops.table_reconcile_peer_f32([t.data_ptr() for t in reps], prev, 0.5)
    torch.cuda.synchronize()
print("done", what)
if what == "neumf":
    from elliot_b200.recommender.neumf_sharded import ShardedNeuMFModel
    B = 1 << 20
    sh = ShardedNeuMFModel(2_500_000, 1_000_000, 64, 1e-3, 42, dev, full_init=False)
    u = torch.randint(0, 2_500_000, (B,), device=dev, dtype=torch.int32); it = torch.randint(0, 1_000_000, (B,), device=dev, dtype=torch.int32)
    y = (torch.arange(B, device=dev) % 5 == 0).float()
    for _ in range(3):
        sh.train_step((u, it, y))
    torch.cuda.synchronize()
    print("done neumf")
