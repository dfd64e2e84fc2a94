"""Times the tensor-core scoring kernel on C2- and C5-shaped inputs (not the bench contract)."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from elliot_b200 import ops
dev = "cuda:0"
def run(nu, ni, d, k, per_user, label):
    g = torch.Generator(device=dev); g.manual_seed(0)
    ld = ops.padded_dim(d)
    U = torch.zeros((nu, ld), device=dev); V = torch.zeros((ni, ld), device=dev)
    U[:, :d] = torch.randn(nu, d, device=dev, generator=g) * 0.1; V[:, :d] = torch.randn(ni, d, device=dev, generator=g) * 0.1
    b = torch.randn(ni, device=dev, generator=g) * 0.05
    cand = (torch.rand(nu, per_user, device=dev, generator=g) ** 2 * ni).to(torch.int32).clamp_(max=ni - 1)
    cand, _ = torch.sort(cand, dim=1); keep = torch.ones_like(cand, dtype=torch.bool); keep[:, 1:] = cand[:, 1:] != cand[:, :-1]
    indptr = torch.zeros(nu + 1, dtype=torch.int64, device=dev); indptr[1:] = torch.cumsum(keep.sum(1), 0); indices = cand[keep].contiguous()
    for _ in range(2): i1, v1, st = ops.score_topk_tc(U, V, b, d, k, indptr, indices)
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record(); reps = 3
    for _ in range(reps): i1, v1, st = ops.score_topk_tc(U, V, b, d, k, indptr, indices)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    kp = st["kp"]; fl = 2.0 * kp * ni * nu
    print(f"{label}: {nu} users x {ni} items d={d} kp={kp}: {ms:.2f} ms  {nu/ms*1e3/1e6:.3f} M users/s  {fl/ms/1e9:.1f} TFLOP/s (padded K)  {2.0*d*ni*nu/ms/1e9:.1f} TFLOP/s (algorithmic)  rechecked {st['rechecked']}  prof {st.get('prof')}")
    # spot-check vs exact kernel on 512 users
    i0, v0 = ops.score_topk(U, V, b, d, k, indptr, indices, user_begin=0, n_sel=512)
    print("   identical to exact kernel on 512 users:", torch.equal(i0, i1[:512]), torch.equal(v0, v1[:512]))
if len(sys.argv) > 1 and sys.argv[1] == "ab":
    # A/B of the epilogue layouts; EB_TC_DEBUG=3 certifies everything (no re-check) so the main kernel is timed alone;
    # EB_TC_PROF=1 adds warp 0's cycle counters (stage wait, MMA + staging, scan, compaction, re-rank; counts)
    os.environ["EB_TC_PROF"] = "1"
    for ng in ("1", "2"):
        for dbg in ("0", "3"):
            os.environ["EB_TC_NG"] = ng; os.environ["EB_TC_DEBUG"] = dbg
            run(132 * 128 * 2, 100_000, 64, 10, 100, f"C2 ng={ng} dbg={dbg}")
            run(132 * 128 * 2, 2_000_000, 128, 10, 100, f"C5 ng={ng} dbg={dbg}")
    sys.exit(0)
if len(sys.argv) > 1 and sys.argv[1] == "pair":
    # single CTAs against CTA pairs (clusters of two, each item tile fetched half by each CTA and multicast to both)
    os.environ["EB_TC_PROF"] = "1"; os.environ["EB_TC_NG"] = "2"
    for pair in ("0", "1"):
        for dbg in ("0", "1"):
            os.environ["EB_TC_PAIR"] = pair; os.environ["EB_TC_DEBUG"] = dbg
            run(132 * 128 * 2, 100_000, 64, 10, 100, f"C2 pair={pair} dbg={dbg}")
            run(132 * 128 * 2, 2_000_000, 128, 10, 100, f"C5 pair={pair} dbg={dbg}")
    sys.exit(0)
if len(sys.argv) > 1 and sys.argv[1] == "atm":
    # the user block in shared memory against the user block in registers (wgmma A operand)
    os.environ["EB_TC_PROF"] = "1"; os.environ["EB_TC_NG"] = "2"; os.environ["EB_TC_PAIR"] = "0"
    for atm in ("0", "1"):
        for dbg in ("0", "1"):
            os.environ["EB_TC_ATM"] = atm; os.environ["EB_TC_DEBUG"] = dbg
            run(132 * 128 * 2, 100_000, 64, 10, 100, f"C2 atm={atm} dbg={dbg}")
            run(132 * 128 * 2, 2_000_000, 128, 10, 100, f"C5 atm={atm} dbg={dbg}")
    sys.exit(0)
if len(sys.argv) > 1 and sys.argv[1] == "feed":
    # EB_TC_DEBUG=1: the epilogue only reads the accumulators and takes the max (no inserts): the TMA/MMA pipeline's own pace
    os.environ["EB_TC_PROF"] = "1"
    for ng in ("1", "2"):
        for dbg in ("1", "2"):
            os.environ["EB_TC_NG"] = ng; os.environ["EB_TC_DEBUG"] = dbg
            run(132 * 128 * 2, 100_000, 64, 10, 100, f"C2 ng={ng} dbg={dbg}")
            run(132 * 128 * 2, 2_000_000, 128, 10, 100, f"C5 ng={ng} dbg={dbg}")
    sys.exit(0)
run(132 * 128 * 4, 100_000, 64, 10, 100, "C2-shape")
run(132 * 128 * 2, 2_000_000, 128, 10, 100, "C5-shape(per-GPU slice)")
run(6040, 3706, 64, 10, 130, "C1-shape")
