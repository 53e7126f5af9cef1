"""Event-timed aggregation of the output layer's backward pass (`backward2` of the 3-layer GCN) with and without
skipping its all-zero gradient rows, at the ogbn-products shape.

    python tools/bench_spmm_live.py [--scale 1.0] [--F 256] [--reps 10] [--json out.json]

The loss only sees the train rows, so the gradient the top layer aggregates is exactly zero on every other row.  The
input here is that matrix: random rows on the synthetic partition's train mask, zero rows elsewhere.  Configurations,
alternated launch by launch (median of `--reps` launches each):
  today      the aggregation as it runs without liveness (`spmm(..., live=None)`);
  skip       the row-liveness kernel over the gradient + the aggregation that skips dead source rows;
  all_live   the same two launches on a dense matrix (every row live): the cost where nothing is skipped;
  live_only  the row-liveness kernel alone.
Also prints the share of all-zero rows and of non-zeros whose source row is all-zero, the card and its power limit,
and whether each skipping output is bitwise equal to the matching `today` output.  On a build without the liveness
path only `today` and the shares are reported."""
import argparse, json, os, subprocess, sys
import numpy as np, torch, yaml
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return {"query": q, "value": r.stdout.strip().splitlines()[0] if r.stdout.strip() else r.stderr.strip()}
    except (OSError, subprocess.SubprocessError) as e:
        return {"query": q, "value": f"nvidia-smi unavailable: {e}"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--F", type=int, default=256)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", type=str, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_spmm_live needs a GPU")
    from adaqp_b200 import build
    build.build()
    from adaqp_b200.manager import graph as G
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import spec_from_config
    cfg = yaml.safe_load(open(os.path.join(ROOT, "adaqp_b200", "config", "ogbn-products.yaml")))
    L = prepare_all_in_process(spec_from_config(cfg, 1, a.scale))[0]
    dev = torch.device("cuda:0")
    g = G.LocalGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo, dev)
    n, nnz, F = L.n_inner, int(L.indptr[-1]), a.F
    train = torch.from_numpy(np.asarray(L.train_mask, dtype=bool)).to(dev)
    has_live = hasattr(G, "row_live")
    # the backward norms of the GCN aggregation (ops.GCN_aggregation, ProprogationMode.Backward)
    pre, post = g.norm["in_-0.5"], g.norm["out_-0.5"]
    gen = torch.Generator(device=dev).manual_seed(0)
    dense = torch.randn(n, F, device=dev, generator=gen)
    grad = dense * train.unsqueeze(1)
    dead = ~train
    idx = torch.from_numpy(L.indices.astype(np.int64)).to(dev)
    info = {"card": card(), "device": torch.cuda.get_device_name(dev), "scale": a.scale, "rows": n, "nnz": nnz, "F": F,
            "reps": a.reps, "zero_row_share": float(dead.float().mean()),
            "zero_source_nnz_share": float(dead[idx].float().mean()), "liveness_path": has_live}
    del idx
    print(json.dumps(info), flush=True)

    outs = {}
    live_buf = torch.empty(n, dtype=torch.uint8, device=dev)

    def today(x, key):
        outs[key] = G.spmm(g, x, None, pre, post, out=outs.get(key))

    def skip(x, key):
        G.row_live(x, out=live_buf)
        outs[key] = G.spmm(g, x, None, pre, post, out=outs.get(key), live=live_buf)

    configs = {"today": lambda: today(grad, "today"), "today_dense": lambda: today(dense, "today_dense")}
    if has_live:
        configs.update({"skip": lambda: skip(grad, "skip"), "all_live": lambda: skip(dense, "all_live"),
                        "live_only": lambda: G.row_live(grad, out=live_buf)})
    for fn in configs.values():             # warm-up of every shape
        fn()
    torch.cuda.synchronize()
    ts = {k: [] for k in configs}
    for _ in range(a.reps):
        for k, fn in configs.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(); fn(); e.record()
            torch.cuda.synchronize()
            ts[k].append(s.elapsed_time(e))
    res = {k: {"ms_median": float(np.median(v)), "ms_min": float(min(v)), "ms_max": float(max(v))} for k, v in ts.items()}
    if has_live:
        res["skip"]["bitwise_equal_today"] = bool(torch.equal(outs["skip"], outs["today"]))
        res["all_live"]["bitwise_equal_today"] = bool(torch.equal(outs["all_live"], outs["today_dense"]))
        want = (grad != 0).any(1)
        res["live_only"]["equal_any_nonzero"] = bool(torch.equal(live_buf.bool(), want))
    print(json.dumps(res), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"info": info, "results": res}, f, indent=1)


if __name__ == "__main__":
    main()
