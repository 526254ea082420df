"""Sweep the window of the table-driven verify's fixed-base table (AFC_VERIFY_BASE_WINDOW, DESIGN.md section 4) on one GPU.

For each window w it creates a fresh context and measures, on bench.py's headline workload (1 M x 512 B credentials, 1024
issuers): the first call on an empty cache (which also builds the w table), the headline step (cache emptied before every step),
k_ed_verify_cached_dyn through the library's per-kernel events, the warm step (tables kept) and the key-set step, plus the table's
bytes and build time.  Windows alternate and every one is measured `--reps` times, so that drift on a shared machine lands on
every window alike.  Prints one JSON line per run, then a summary line with the card's name and power limit.

    python tools/base_window_sweep.py --windows 16,18,20,21,22 --reps 3 --steps 30
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def run_one(w, steps, dev):
    import torch
    import agentfield_b200 as afb
    import bench
    os.environ["AFC_VERIFY_BASE_WINDOW"] = str(w)
    ctx = afb.Context(0)
    try:
        d_pks, d_sigs, d_msgs, d_off, expect = bench.make_workload(ctx, dev, 0)
        n = bench.N_ITEMS
        d_ok = torch.empty(n, dtype=torch.uint8, device=dev)
        c0, c1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        c0.record()
        ctx.verify_dev(d_pks, d_sigs, d_msgs, d_off, n, d_ok)
        c1.record(); torch.cuda.synchronize()
        first_ms = c0.elapsed_time(c1)
        st = ctx.keycache_stats()

        def cold():
            ctx.keycache_clear()
            ctx.verify_dev(d_pks, d_sigs, d_msgs, d_off, n, d_ok)

        def warm():
            ctx.verify_dev(d_pks, d_sigs, d_msgs, d_off, n, d_ok)

        def timed(fn, k):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(k):
                fn()
            b.record(); torch.cuda.synchronize()
            return a.elapsed_time(b) / k

        cold_ms = timed(cold, steps)
        assert torch.equal(d_ok, expect)
        ctx.profile_begin(64 + 32 * 10)
        for _ in range(10):
            cold()
        prof = ctx.profile_end()
        warm_ms = timed(warm, steps)
        assert torch.equal(d_ok, expect)
        ks = afb.KeySet([bytes(r) for r in d_pks[:bench.N_KEYS].cpu().numpy()], ctx)
        d_ki = (torch.arange(n, device=dev) % bench.N_KEYS).to(torch.int32)
        keyed_ms = timed(lambda: ks.verify_dev(d_ki, d_sigs, d_msgs, d_off, n, d_ok), steps)
        assert torch.equal(d_ok, expect)
        ks.close()
        kv = prof.get("k_ed_verify_cached_dyn", {"avg_ms": float("nan")})
        return {"w": w, "base_window_in_use": st["base_window"], "table_bytes": st["base_table_bytes"], "build_ms": st["base_build_us"] / 1e3,
                "first_call_ms": first_ms, "cold_step_ms": cold_ms, "k_ed_verify_cached_dyn_ms": kv["avg_ms"], "warm_ms": warm_ms,
                "keyed_ms": keyed_ms}
    finally:
        ctx.close()
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", default="16,18,20,21,22")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    args = ap.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    ws = [int(x) for x in args.windows.split(",")]
    runs = []
    for rep in range(args.reps):
        for w in ws:
            r = run_one(w, args.steps, dev)
            r["rep"] = rep
            runs.append(r)
            print(json.dumps(r), flush=True)
    summary = {"card": card(), "steps": args.steps, "reps": args.reps, "by_window": {}}
    for w in ws:
        rs = [r for r in runs if r["w"] == w]
        summary["by_window"][w] = {k: [round(r[k], 3) for r in rs] for k in ("cold_step_ms", "k_ed_verify_cached_dyn_ms", "warm_ms", "keyed_ms",
                                                                           "first_call_ms", "build_ms")}
        summary["by_window"][w]["table_bytes"] = rs[0]["table_bytes"]
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
