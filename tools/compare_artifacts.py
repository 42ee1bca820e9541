"""Check that two trees of this repository write the same Categorify artefact files.

    python tools/compare_artifacts.py fit OUT [--root TREE] [--rows N]
        fits bench.py's Criteo workflow once, at bench size by default, with the package and
        bench.py of TREE (default: this repository), then reads every op.categories path so
        that the lazily written large vocabularies exist too; the files land in OUT/categories
    python tools/compare_artifacts.py compare A B
        pd.read_parquet of every file under A/categories and B/categories: the same file names,
        frame-equal (values, dtypes, RangeIndex)

Needs a CUDA device for `fit`; `compare` is host only."""
import argparse
import os
import sys


def fit(out, root, rows):
    root = os.path.abspath(root)
    sys.path.insert(0, root)
    import torch
    import bench
    import nvtabular_b200 as nvt
    assert os.path.dirname(os.path.abspath(nvt.__file__)) == os.path.join(root, "nvtabular_b200"), nvt.__file__
    os.environ["NVTB_ARTIFACTS"] = "eager"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    table = bench.make_table("criteo", rows, dev, 0, 4_370_000_000)
    wf = bench.build_workflow(nvt, "criteo", os.path.abspath(out))
    wf.fit(nvt.Dataset(list(bench.cut(table, 4))))
    for node in wf.output_node.topo_order():
        cats = getattr(getattr(node, "op", None), "categories", None)
        for name in list(cats or []):
            cats[name]                      # writes a vocabulary above the eager limit
    torch.cuda.synchronize()
    print(f"fit {rows} rows with {root}: {len(os.listdir(os.path.join(out, 'categories')))} files")


def compare(a, b):
    import pandas as pd
    da, db = os.path.join(a, "categories"), os.path.join(b, "categories")
    fa, fb = sorted(os.listdir(da)), sorted(os.listdir(db))
    if fa != fb:
        raise SystemExit(f"different files: {sorted(set(fa) ^ set(fb))}")
    for f in fa:
        x, y = pd.read_parquet(os.path.join(da, f)), pd.read_parquet(os.path.join(db, f))
        pd.testing.assert_frame_equal(x, y, check_exact=True)
        assert type(x.index) is type(y.index) and list(x.index[:1]) == list(y.index[:1]), f
    print(f"{len(fa)} files frame-equal")


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    f = sub.add_parser("fit")
    f.add_argument("out")
    f.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    f.add_argument("--rows", type=int, default=100_000_000)
    c = sub.add_parser("compare")
    c.add_argument("a")
    c.add_argument("b")
    args = ap.parse_args()
    if args.cmd == "fit":
        fit(args.out, args.root, args.rows)
    else:
        compare(args.a, args.b)


if __name__ == "__main__":
    main()
