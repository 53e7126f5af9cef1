"""Event-timed sweep of the aggregation kernel variants on an ogbn-products-shaped partition.

    python tools/bench_spmm.py [--scale 1.0] [--world 1] [--reps 10] [--json out.json]
    python tools/bench_spmm.py --slices 1,2,4 [--dims 256,100]      # column-slice sweep (slice_sweep)

Variants (library option `spmm_impl`, adaqp_b200/_lib.py): 1 = register-staged gather (default),
2 = cp.async lane-private ring, 3 = TMA tensor-map ring (one row copy per neighbour, four-row groups),
4 = one TMA bulk copy per neighbour row; plus the streaming hints of v1 (bit 0: st.global.cs for
the output rows, bit 1: ld.global.cs for the index stream) and rows per grab.  Every variant's
output is compared with v1's (max abs difference relative to the largest magnitude)."""
import argparse, json, os, sys
import numpy as np, torch, yaml
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--world", type=int, default=1)
    ap.add_argument("--dims", type=str, default="256,100")
    ap.add_argument("--json", type=str, default=None)
    ap.add_argument("--variants", type=str, default="1:0:0,1:1:0,1:2:0,1:3:0,3:0:1,3:0:2,3:0:4,3:0:8,4:0:4,2:0:0",
                    help="impl:hints:rows_per_grab (0 = default), comma separated")
    ap.add_argument("--slices", type=str, default=None,
                    help="column-slice sweep instead of the variant sweep: slice counts, comma separated (e.g. 1,2,4)")
    ap.add_argument("--hints", type=int, default=0, help="spmm_hints for the slice sweep")
    a = ap.parse_args()
    from adaqp_b200 import build
    build.build()
    from adaqp_b200 import _lib
    from adaqp_b200.manager.graph import LocalGraph, spmm
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import spec_from_config
    cfg = yaml.safe_load(open(os.path.join(ROOT, "adaqp_b200", "config", "ogbn-products.yaml")))
    spec = spec_from_config(cfg, a.world, a.scale)
    L = prepare_all_in_process(spec)[0]
    dev = torch.device("cuda:0")
    g = LocalGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo, dev)
    nnz = int(L.indptr[-1])
    if a.slices:
        slice_sweep(a, g, L, nnz, dev, _lib, spmm)
        return
    results = []
    for F in [int(x) for x in a.dims.split(",")]:
        xl = torch.randn(L.n_inner, F, device=dev)
        xh = torch.randn(max(L.n_halo, 1), F, device=dev) if L.n_halo else None
        out = torch.empty(L.n_inner, F, device=dev)
        ref = None
        for var in a.variants.split(","):
            impl, hints, grab = (int(x) for x in var.split(":"))
            _lib.set_option("spmm_impl", impl)
            _lib.set_option("spmm_hints", hints)
            _lib.set_option("spmm_rows_per_grab", grab)
            for _ in range(3):
                spmm(g, xl, xh, g.norm["out_-0.5"], g.norm["in_-0.5"], out=out)
            ts = []
            for _ in range(a.reps):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record(); spmm(g, xl, xh, g.norm["out_-0.5"], g.norm["in_-0.5"], out=out); e.record()
                torch.cuda.synchronize(); ts.append(s.elapsed_time(e))
            if ref is None:
                ref = out.clone()
            diff = float((out - ref).abs().max() / ref.abs().max())
            ms = float(np.median(ts))
            comp = 4 * nnz + 8 * (L.n_inner + 1) + 4 * F * (2 * L.n_inner + L.n_halo) + 4 * (2 * L.n_inner + L.n_halo)
            results.append({"impl": impl, "hints": hints, "rows_per_grab": grab, "F": F, "rows": L.n_inner, "nnz": nnz,
                            "ms": ms, "ms_min": float(min(ts)), "no_reuse_GBps": 4 * F * nnz / ms / 1e6,
                            "compulsory_GBps": comp / ms / 1e6, "max_rel_diff_vs_v1": diff})
            print(json.dumps(results[-1]), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"scale": a.scale, "world": a.world, "results": results}, f, indent=1)


def slice_widths(F: int, n: int):
    """n column slices of F: widths rounded up to a multiple of 4 (16-byte slice starts), the last one takes the rest."""
    w = -(-F // n)
    w = -(-w // 4) * 4
    out, c = [], 0
    while c < F:
        out.append(min(w, F - c))
        c += out[-1]
    return out


def card():
    import subprocess
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return {"query": q, "value": r.stdout.strip().splitlines()[0] if r.stdout.strip() else r.stderr.strip()}
    except (OSError, subprocess.SubprocessError) as e:
        return {"query": q, "value": f"nvidia-smi unavailable: {e}"}


def slice_sweep(a, g, L, nnz, dev, _lib, spmm):
    """Time the aggregation of F columns as 1, 2, 4 ... column slices (GCN forward norms), repetitions alternated
    across the configurations.  Two ways to slice: `launches` runs one launch per slice on column views of the
    same tensors; `fused` is the library's own slice-major kernel (option `spmm_slice_cols`, one launch).  Every
    output is compared bit for bit with the unsliced launch (`spmm_slice_cols` = F)."""
    info = {"card": card(), "device": torch.cuda.get_device_name(dev), "scale": a.scale, "world": a.world,
            "rows": L.n_inner, "nnz": nnz, "reps": a.reps}
    print(json.dumps(info), flush=True)
    try:
        _lib.get_option("spmm_slice_cols")
        has_opt = True
    except ValueError:
        has_opt = False
    pre, post = g.norm["out_-0.5"], g.norm["in_-0.5"]
    _lib.set_option("spmm_hints", a.hints)
    results = []
    for F in [int(x) for x in a.dims.split(",")]:
        xl = torch.randn(L.n_inner, F, device=dev)
        xh = torch.randn(max(L.n_halo, 1), F, device=dev) if L.n_halo else None
        ref = torch.empty(L.n_inner, F, device=dev)
        if has_opt:
            _lib.set_option("spmm_slice_cols", F)
        spmm(g, xl, xh, pre, post, out=ref)
        torch.cuda.synchronize()
        configs = []
        for n in [int(x) for x in a.slices.split(",")]:
            widths = slice_widths(F, n)
            if n > 1 and len(widths) != n:
                continue
            configs.append({"F": F, "slices": widths, "mode": "launches", "out": torch.empty_like(ref)})
            if has_opt and n > 1 and widths[0] <= 128:
                configs.append({"F": F, "slices": widths, "mode": "fused", "out": torch.empty_like(ref)})
        if has_opt:
            configs.append({"F": F, "slices": None, "mode": "auto", "out": torch.empty_like(ref)})

        def run(cf):
            out = cf["out"]
            if cf["mode"] == "launches":
                if has_opt:
                    _lib.set_option("spmm_slice_cols", F)
                c = 0
                for w in cf["slices"]:
                    spmm(g, xl[:, c:c + w], xh[:, c:c + w] if xh is not None else None, pre, post, out=out[:, c:c + w])
                    c += w
            else:
                _lib.set_option("spmm_slice_cols", cf["slices"][0] if cf["mode"] == "fused" else 0)
                spmm(g, xl, xh, pre, post, out=out)

        for cf in configs:
            for _ in range(2):
                run(cf)
            cf["ts"] = []
        for _ in range(a.reps):
            for cf in configs:
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record(); run(cf); e.record()
                torch.cuda.synchronize(); cf["ts"].append(s.elapsed_time(e))
        for cf in configs:
            ts = cf["ts"]
            ms = float(np.median(ts))
            results.append({"F": F, "mode": cf["mode"], "slices": cf["slices"], "ms": ms, "ms_min": float(min(ts)),
                            "ms_max": float(max(ts)), "no_reuse_GBps": 4 * F * nnz / ms / 1e6,
                            "bitwise_equal_unsliced": bool(torch.equal(cf["out"], ref))})
            print(json.dumps(results[-1]), flush=True)
        if has_opt:
            _lib.set_option("spmm_slice_cols", 0)
        del xl, xh, ref, configs
    if a.json:
        with open(a.json, "w") as f:
            json.dump({**info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
