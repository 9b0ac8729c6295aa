"""Manual multi-GPU check (not collected by pytest): ``python -m fadtk_b200.kad`` under torchrun, where every rank takes
its share of the pair tiles, must print the same ``kad`` / ``bandwidth`` and write the same ``--indiv`` table as a
single process.  Usage on a box with >= 2 GPUs (and with 4 and 8 where available):

    python tests/multi_gpu_kad_check.py prepare /tmp/mk
    python -m fadtk_b200.kad vggish /tmp/mk/base /tmp/mk/ev /tmp/mk/one.csv
    python -m fadtk_b200.kad vggish /tmp/mk/base /tmp/mk/ev /tmp/mk/one_indiv.csv --indiv
    torchrun --nproc-per-node 2 --master-addr 127.0.0.1 -m fadtk_b200.kad vggish /tmp/mk/base /tmp/mk/ev /tmp/mk/two.csv
    torchrun --nproc-per-node 2 --master-addr 127.0.0.1 -m fadtk_b200.kad vggish /tmp/mk/base /tmp/mk/ev /tmp/mk/two_indiv.csv --indiv
    python tests/multi_gpu_kad_check.py compare /tmp/mk two
"""
import csv
import sys
from pathlib import Path

import numpy as np


def prepare(root: Path):
    rng = np.random.default_rng(5)
    d = 128
    mix = rng.standard_normal((d, d)) / np.sqrt(d)
    for name, files, scale in (("base", 40, 1.0), ("ev", 37, 0.8)):
        (root / name / "embeddings" / "vggish").mkdir(parents=True, exist_ok=True)
        for i in range(files):
            rows = ((rng.standard_normal((200 + 37 * i, d)) @ mix) * (scale + 0.01 * i)).astype(np.float16)
            (root / name / f"s{i:03d}.wav").write_bytes(b"")
            np.save(root / name / "embeddings" / "vggish" / f"s{i:03d}.npy", rows)


def compare(root: Path, tag: str):
    rows = {t: list(csv.DictReader((root / f"{t}.csv").open())) for t in ("one", tag)}
    for a, b in zip(rows["one"], rows[tag], strict=True):
        for k in ("kad", "bandwidth", "n_baseline", "n_eval"):
            assert a[k] == b[k], (k, a[k], b[k])
    a = (root / "one_indiv.csv").read_text()
    b = (root / f"{tag}_indiv.csv").read_text()
    assert a == b, "the --indiv tables differ"
    print(f"multi-GPU KAD identical: {len(rows['one'])} rows, {len(a.splitlines())} --indiv rows ({tag})")


if __name__ == "__main__":
    if sys.argv[1] == "prepare":
        prepare(Path(sys.argv[2]))
    else:
        compare(Path(sys.argv[2]), sys.argv[3])
