"""Manual multi-GPU check (not collected by pytest): a baseline prepared under torchrun, where every rank takes its share
of the bandwidth, S_xx and radius-list tiles, must score an eval directory with ``--prepared`` exactly as a single
process without a preparation does, byte for byte.
Usage on a box with >= 2 GPUs (and with 4 and 8 where available):

    python tests/multi_gpu_pairwise_baseline_check.py prepare /tmp/mp
    python -m fadtk_b200.prdc vggish /tmp/mp/base /tmp/mp/ev /tmp/mp/one.csv --indiv
    torchrun --nproc-per-node 2 --master-addr 127.0.0.1 -m fadtk_b200.prepare vggish /tmp/mp/base
    torchrun --nproc-per-node 2 --master-addr 127.0.0.1 -m fadtk_b200.prdc vggish /tmp/mp/base /tmp/mp/ev /tmp/mp/two.csv --indiv --prepared
    python tests/multi_gpu_pairwise_baseline_check.py compare /tmp/mp two
"""
import sys
from pathlib import Path

from multi_gpu_kad_check import prepare


def compare(root: Path, tag: str):
    a, b = (root / "one.csv").read_text(), (root / f"{tag}.csv").read_text()
    assert a == b, "the per-file PRDC tables differ"
    print(f"multi-GPU prepared baseline identical: {len(a.splitlines()) - 1} files ({tag})")


if __name__ == "__main__":
    if sys.argv[1] == "prepare":
        prepare(Path(sys.argv[2]))
    else:
        compare(Path(sys.argv[2]), sys.argv[3])
