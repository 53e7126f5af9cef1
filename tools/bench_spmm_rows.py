"""Event-timed aggregation of the output layer's forward pass (`forward2` of the 3-layer GCN) over every row against
over the train rows only, at the ogbn-products shape.

    python tools/bench_spmm_rows.py [--scale 1.0] [--F 256] [--reps 10] [--json out.json]

The loss only reads the train rows, and the output layer is aggregate -> linear, so its forward aggregation only has
to compute those rows.  The input is a random [n, F] matrix on the synthetic partition with its real train mask;
the aggregation uses the forward GCN norms.  Configurations, alternated launch by launch (median of `--reps` each):
  today       the aggregation of every row, as the output layer ran it before (`spmm(..., rows=None)`);
  restricted  zero-fill of the output + the aggregation of the listed train rows (`spmm(..., rows=row_list(train))`);
  zero_only   the zero-fill alone.
Also prints the share of rows and of non-zeros that are listed, the card and its power limit, and whether the listed
rows of `restricted` are bitwise equal to those of `today` (and the other rows zero)."""
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
        raise SystemExit("bench_spmm_rows needs a GPU")
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
    train = torch.from_numpy(np.asarray(L.train_mask, dtype=bool))
    rows = G.row_list(train, n, dev)
    deg = np.diff(np.asarray(L.indptr, dtype=np.int64))
    listed_nnz = int(deg[rows.ids.cpu().numpy()].sum())
    # the forward norms of the GCN aggregation (ops.GCN_aggregation, ProprogationMode.Forward)
    pre, post = g.norm["out_-0.5"], g.norm["in_-0.5"]
    gen = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(n, F, device=dev, generator=gen)
    info = {"card": card(), "device": torch.cuda.get_device_name(dev), "scale": a.scale, "rows": n, "nnz": nnz, "F": F,
            "reps": a.reps, "listed_rows": rows.n, "listed_row_share": rows.n / n, "listed_nnz_share": listed_nnz / nnz}
    print(json.dumps(info), flush=True)

    out_today = torch.empty(n, F, device=dev)
    out_rows = torch.empty(n, F, device=dev)

    def today():
        G.spmm(g, x, None, pre, post, out=out_today)

    def restricted():
        out_rows.zero_()
        G.spmm(g, x, None, pre, post, out=out_rows, rows=rows)

    configs = {"today": today, "restricted": restricted, "zero_only": lambda: out_rows.zero_()}
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
    restricted()
    torch.cuda.synchronize()
    keep = train.to(dev)
    res["restricted"]["listed_rows_bitwise_equal_today"] = bool(torch.equal(out_rows[keep].view(torch.int32),
                                                                           out_today[keep].view(torch.int32)))
    res["restricted"]["other_rows_zero"] = bool((out_rows[~keep].view(torch.int32) == 0).all())
    res["saved_ms"] = res["today"]["ms_median"] - res["restricted"]["ms_median"]
    print(json.dumps(res), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"info": info, "results": res}, f, indent=1)


if __name__ == "__main__":
    main()
