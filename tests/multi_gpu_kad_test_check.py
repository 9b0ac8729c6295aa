"""Manual multi-GPU check (not collected by pytest): ``python -m fadtk_b200.kad_test`` under torchrun, where every rank
takes its share of the pair tiles of the permutation pass (fad_kad_perm_sums_sharded over the library's NCCL
communicator, with a, the labellings, the seed and sigma compared across ranks first), must write the same kad,
p_value and bandwidth as a single process, for the test against the baseline, the comparison and a prepared baseline.
Usage on a box with >= 2 GPUs (and with 4 and 8 where available):

    python tests/multi_gpu_kad_test_check.py prepare /tmp/mt
    python -m fadtk_b200.kad_test vggish /tmp/mt/base /tmp/mt/ev /tmp/mt/one.csv --permutations 1500
    python -m fadtk_b200.kad_test vggish /tmp/mt/base /tmp/mt/ev /tmp/mt/one.csv --versus /tmp/mt/vs
    python -m fadtk_b200.kad_test vggish /tmp/mt/base /tmp/mt/ev /tmp/mt/one.csv --prepared
    torchrun --nproc-per-node 2 --master-addr 127.0.0.1 -m fadtk_b200.kad_test vggish /tmp/mt/base /tmp/mt/ev /tmp/mt/two.csv --permutations 1500
    torchrun --nproc-per-node 2 --master-addr 127.0.0.1 -m fadtk_b200.kad_test vggish /tmp/mt/base /tmp/mt/ev /tmp/mt/two.csv --versus /tmp/mt/vs
    torchrun --nproc-per-node 2 --master-addr 127.0.0.1 -m fadtk_b200.kad_test vggish /tmp/mt/base /tmp/mt/ev /tmp/mt/two.csv --prepared
    python tests/multi_gpu_kad_test_check.py compare /tmp/mt two
"""
import csv
import sys
from pathlib import Path

from multi_gpu_kad_check import prepare as prepare_kad

FIELDS = ("versus", "kad", "kad_versus", "difference", "p_value", "permutations", "seed", "bandwidth", "n_baseline",
          "n_eval", "n_versus")


def prepare(root: Path):
    prepare_kad(root)
    # a third directory: the eval files' rows, scaled, as system B
    import numpy as np
    (root / "vs" / "embeddings" / "vggish").mkdir(parents=True, exist_ok=True)
    for f in sorted((root / "ev" / "embeddings" / "vggish").glob("*.npy"))[:20]:
        np.save(root / "vs" / "embeddings" / "vggish" / f.name, (np.load(f).astype(np.float32) * 1.05).astype(np.float16))
        (root / "vs" / f"{f.stem}.wav").write_bytes(b"")


def compare(root: Path, tag: str):
    rows = {t: list(csv.DictReader((root / f"{t}.csv").open())) for t in ("one", tag)}
    for a, b in zip(rows["one"], rows[tag], strict=True):
        for k in FIELDS:
            assert a[k].replace("/one", "") == b[k].replace(f"/{tag}", ""), (k, a[k], b[k])
    print(f"multi-GPU KAD permutation tests identical: {len(rows['one'])} rows ({tag})")


if __name__ == "__main__":
    if sys.argv[1] == "prepare":
        prepare(Path(sys.argv[2]))
    else:
        compare(Path(sys.argv[2]), sys.argv[3])
