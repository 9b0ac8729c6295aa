"""Manual multi-GPU check (not collected by pytest): ``python -m fadtk_b200.prdc`` under torchrun, where every rank takes
its share of the radii and ball-count tiles, must write the same ``precision`` / ``recall`` / ``density`` /
``coverage`` row as a single process.  Usage on a box with >= 2 GPUs (and with 4 and 8 where available):

    python tests/multi_gpu_prdc_check.py prepare /tmp/mp
    python -m fadtk_b200.prdc vggish /tmp/mp/base /tmp/mp/ev /tmp/mp/one.csv -k 5
    torchrun --nproc-per-node 2 --master-addr 127.0.0.1 -m fadtk_b200.prdc vggish /tmp/mp/base /tmp/mp/ev /tmp/mp/two.csv -k 5
    python tests/multi_gpu_prdc_check.py compare /tmp/mp two
"""
import csv
import sys
from pathlib import Path

from multi_gpu_kad_check import prepare


def compare(root: Path, tag: str):
    rows = {t: list(csv.DictReader((root / f"{t}.csv").open())) for t in ("one", tag)}
    for a, b in zip(rows["one"], rows[tag], strict=True):
        for k in ("k", "precision", "recall", "density", "coverage", "n_baseline", "n_eval"):
            assert a[k] == b[k], (k, a[k], b[k])
    print(f"multi-GPU PRDC identical: {len(rows['one'])} rows ({tag})")


if __name__ == "__main__":
    if sys.argv[1] == "prepare":
        prepare(Path(sys.argv[2]))
    else:
        compare(Path(sys.argv[2]), sys.argv[3])
