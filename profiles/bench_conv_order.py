"""Per-shape cost of the sparse-convolution kernel under tile orders (pcb_conv_tile_order): every tensor-core forward and data-gradient
launch of one C1 training step (Res16UNet34C, 4 synthetic ScanNet-shape pairs at 2.5 cm, both views stacked), timed with CUDA events
over windows of at least `--seconds` after warm-up, in the identity order and in the window-sorted order for each window of the sweep.
Per shape it reports the kernel time, the kernel offsets a 128-row tile stages (of K) and the share of MMA rows that carry a real
neighbour pair; `per_step_ms` weights each shape by how many units of the step issue it.  Offset-split launches (small levels) always run
in the identity order and are left out.  Per shape `pool` describes how often the identity order's tiles read the same input row:
distinct input rows per tile, gathers (entries with a neighbour) per distinct row, the largest row span of a tile, and the share of
tiles that a shared-memory pool of POOL_ROWS distinct rows within POOL_SPAN rows could not hold (the pool measured in DESIGN.md
section 7).  The `wgrad` block times every `pcb_conv_wgrad_split` shape of the same step (weight-gradient kernel plus its reduce, in the
executor's orientation and accumulating into dW, as the step issues it) the same way, with a CRC of the dW one non-accumulating call
returns, so two builds can be compared for bits; its `per_step_ms` weights each shape by its launches per step.  `--parts` picks the
blocks to run.  Prints one JSON line, with the card's name, power limit and SM clock.

    python profiles/bench_conv_order.py [--seconds 1.0] [--windows 4096,8192,16384,0] [--parts conv,wgrad]
"""
import argparse
import json
import os
import subprocess
import sys
import zlib

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from pointcontrast_b200 import _lib, fused, me, synth  # noqa: E402
from pointcontrast_b200._lib import check, lib, ptr, stream  # noqa: E402
from pointcontrast_b200.config import default_config  # noqa: E402
from pointcontrast_b200.data import to_torch  # noqa: E402
from pointcontrast_b200.model import load_model  # noqa: E402

BM = 128
WINDOWS = "4096,8192,16384,0"             # 0: the whole level is one window
POOL_ROWS, POOL_SPAN = 512, 4096          # one 32-channel chunk of 512 rows, hi and lo planes: 64 KB of shared memory


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), (v.strip() for v in out.splitlines()[torch.cuda.current_device()].split(","))))
    except (OSError, IndexError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name()}


def tile_order(tbl, n, window):
    wsb = lib.pcb_conv_tile_order_ws_bytes(n)
    ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device="cuda")
    perm = torch.empty(n, dtype=torch.int32, device="cuda")
    check(lib.pcb_conv_tile_order(ptr(tbl), tbl.shape[1], tbl.shape[0], n, window, ptr(perm), ptr(ws), wsb, stream()))
    return perm


def tile_stats(mask, order):
    """(mean offsets per tile, share of MMA rows with a real pair) of the 128-row tiles in `order`."""
    m = np.concatenate([mask[order], np.zeros(-len(order) % BM, np.int64)]).reshape(-1, BM)
    nk = np.array([bin(int(v)).count("1") for v in np.bitwise_or.reduce(m, axis=1)])
    pairs = sum(bin(int(v)).count("1") for v in mask)
    return float(nk.mean()), float(pairs / (nk.sum() * BM))


def pool_stats(t):
    """Row-pool view of the identity order's 128-row tiles of table t [K, n] (-1: no neighbour)."""
    K, n = t.shape
    m = np.concatenate([t, np.full((K, -n % BM), -1, t.dtype)], axis=1).reshape(K, -1, BM).transpose(1, 0, 2).reshape(-1, K * BM)
    m = np.sort(m, axis=1)
    valid = m >= 0
    distinct = (valid & np.concatenate([np.ones((len(m), 1), bool), m[:, 1:] != m[:, :-1]], axis=1)).sum(1)
    span = np.where(valid.any(1), m.max(1) - np.where(valid, m, np.iinfo(m.dtype).max).min(1), 0)
    fallback = (span >= POOL_SPAN) | (distinct > POOL_ROWS)
    return {"distinct_rows_mean": round(float(distinct.mean()), 1), "distinct_rows_max": int(distinct.max()),
            "gathers_per_distinct_row": round(float(valid.sum() / max(int(distinct.sum()), 1)), 2), "span_max": int(span.max()),
            "fallback_share": round(float(fallback.mean()), 4)}


def time_launch(fn, seconds):
    """ms per call of fn, from CUDA events around enough back-to-back calls to fill `seconds`."""
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        fn()
    e1.record()
    e1.synchronize()
    reps = max(5, int(seconds * 1e3 / (e0.elapsed_time(e1) / 5)) + 1)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def wgrad_shapes(sched, geom, dev, seconds):
    """Per-shape time of every tensor-core weight-gradient call of one step (pcb_unit_backward and the final layer's me.wgrad)."""
    shapes = {}                                  # (plan, K, Cin, Cout) -> launches per step
    for u in list(sched.units) + [sched.final]:
        if u.tc:
            key = (u.plan, u.K, u.Cin, u.Cout)
            shapes[key] = shapes.get(key, 0) + 1
    rows, total = [], 0.0
    for (pi, K, Cin, Cout), count in shapes.items():
        plan = geom.plans[pi]
        if plan.wg_gather_x:                     # A = the input, gathered; B = the output gradient
            Ca, Cb, tr, n_a, rows_ = Cin, Cout, 0, plan.n_in, plan.n_out
        else:                                    # A = the output gradient, gathered; B = the input; dW written transposed
            Ca, Cb, tr, n_a, rows_ = Cout, Cin, 1, plan.n_out, plan.n_in
        planes = []
        for n, C in ((n_a, Ca), (rows_, Cb)):
            v = torch.randn(n, C, device=dev)
            hi = v.to(torch.bfloat16)
            planes += [hi, (v - hi.float()).to(torch.bfloat16)]
        ah, al, bh, bl = planes
        tbl = plan.wg_tbl
        dW = torch.zeros(K, Ca, Cb, device=dev)
        wsb = lib.pcb_conv_wgrad_split_ws_bytes(K, rows_, Ca, Cb)
        ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=dev)

        def call(flags=_lib.CONV_ACCUMULATE):
            check(lib.pcb_conv_wgrad_split(ptr(ah), ptr(al), Ca, ptr(bh), ptr(bl), Cb, ptr(tbl), tbl.shape[1], K, rows_, Ca, Cb, ptr(dW), tr,
                                           ptr(ws), wsb, flags, stream()))
        call(0)
        crc = zlib.crc32(dW.cpu().numpy().tobytes())
        ms = time_launch(call, seconds)
        total += count * ms
        rows.append({"K": K, "Ca": Ca, "Cb": Cb, "rows": rows_, "transposed_out": tr, "launches_per_step": count, "ms": round(ms, 4),
                     "ms_per_step": round(count * ms, 4), "dW_crc32": crc})
    return {"per_step_ms": round(total, 3), "launches_per_step": sum(shapes.values()), "shapes": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0, help="least timed window per (shape, order)")
    ap.add_argument("--windows", default=WINDOWS, help="tile-order windows to time besides the identity order (comma list, may be empty)")
    ap.add_argument("--parts", default="conv,wgrad", help="blocks to run: conv (forward / data-gradient launches), wgrad")
    args = ap.parse_args()
    parts = set(args.parts.split(","))
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    net = load_model("Res16UNet34C")(3, 32, default_config(), D=3).to(dev).train()
    sched = fused.schedule(net)
    b = to_torch(synth.synth_batch(0, 4, 0.9, 0.025, 300_000), False)
    sinput, n0 = fused.stack_views(b["sinput0_F"], b["sinput0_C"], b["sinput1_F"], b["sinput1_C"], dev)
    geom = fused.Geometry(net, sinput, n0)

    out = {"rows_per_level": geom.n, "seconds_per_measurement": args.seconds}
    if "wgrad" in parts:
        out["wgrad"] = wgrad_shapes(sched, geom, dev, args.seconds)
    shapes = {}                                  # (plan, role, K, contraction, columns) -> units of one step that issue it
    for u in sched.units if "conv" in parts else ():
        if u.tc and u.K > 1:
            for role in ("fwd", "dgrad"):
                key = (u.plan, role, u.K) + ((u.Cin, u.Cout) if role == "fwd" else (u.Cout, u.Cin))
                shapes[key] = shapes.get(key, 0) + 1
    rows = []
    totals = {}
    for (pi, role, K, Ck, N), count in shapes.items():
        plan = geom.plans[pi]
        tbl, kmap = (plan.fwd_tbl, plan.c_kmap("fwd_kmap")) if role == "fwd" else (plan.dg_tbl, plan.c_kmap("dg_kmap"))
        n_out, n_src = (plan.n_out, plan.n_in) if role == "fwd" else (plan.n_in, plan.n_out)
        if lib.pcb_conv_forward_split_ws_bytes(K, n_out, Ck, N):
            continue                             # offset-split: identity order
        fp16 = role == "fwd" and me.FWD_FP16     # as the executor runs them: fp16 planes forward, bf16 for the data gradient
        dt = torch.float16 if fp16 else torch.bfloat16
        x = torch.randn(n_src, Ck, device=dev)
        xh = x.to(dt)
        xl = (x - xh.float()).to(dt)
        W = torch.randn(K, Ck, N, device=dev) * (1.0 / (K * Ck) ** 0.5)
        tiles = torch.empty(lib.pcb_weight_tile_bytes(K, Ck, N, 0), dtype=torch.uint8, device=dev)
        spare = torch.empty(lib.pcb_weight_tile_bytes(K, Ck, N, 1), dtype=torch.uint8, device=dev)
        check(lib.pcb_weight_tile(ptr(W), K, Ck, N, ptr(tiles), ptr(spare), _lib.PLANES_B_FP16 if fp16 else 0, stream()))
        flags = (_lib.PLANES_A_FP16 | _lib.PLANES_B_FP16) if fp16 else 0
        Y = torch.empty(n_out, N, device=dev)
        t = tbl[:, :n_out].cpu().numpy()
        mask = ((t >= 0).astype(np.int64) << np.arange(K)[:, None]).sum(0)
        orders = {"identity": None}
        for w in (int(v) for v in args.windows.split(",") if v.strip()):
            orders[str(w) if w else "level"] = tile_order(tbl, n_out, w if w else -(-n_out // BM) * BM)
        rec = {"role": role, "K": K, "Cin": Ck, "Cout": N, "rows": n_out, "units_per_step": count, "ms": {}, "offsets_per_tile": {},
               "useful_rows": {}, "pool": pool_stats(t)}
        ref = None
        for name, perm in orders.items():
            def call(perm=perm):
                check(lib.pcb_conv_forward_split_ordered(ptr(xh), ptr(xl), Ck, ptr(tbl), tbl.shape[1], kmap, K, ptr(perm), n_out, Ck, N,
                                                         ptr(tiles), None, ptr(Y), N, None, 0, flags, stream()))
            call()
            if ref is None:
                ref = Y.clone()
            rec["same_bits_as_identity" if name == "identity" else f"same_bits_{name}"] = bool(torch.equal(Y.view(torch.int32),
                                                                                                             ref.view(torch.int32)))
            rec["ms"][name] = round(time_launch(call, args.seconds), 4)
            order = np.arange(n_out) if perm is None else perm.cpu().numpy()
            nk, useful = tile_stats(mask, order)
            rec["offsets_per_tile"][name] = round(nk, 2)
            rec["useful_rows"][name] = round(useful, 3)
            totals[name] = totals.get(name, 0.0) + count * rec["ms"][name]
        rec.pop("same_bits_as_identity")
        rows.append(rec)
    if "conv" in parts:
        out.update(per_step_ms={k: round(v, 3) for k, v in totals.items()}, shapes=rows)
    print(json.dumps({"gpu": gpu_info(), **out}), flush=True)


if __name__ == "__main__":
    main()
