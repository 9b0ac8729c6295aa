"""Manual multi-GPU check (not collected by pytest): ``python -m fadtk_b200.nearest`` under torchrun, where every rank
takes its share of the nearest tiles, must write the same per-file table as a single process, byte for byte.
Usage on a box with >= 2 GPUs (and with 4 and 8 where available):

    python tests/multi_gpu_nearest_check.py prepare /tmp/mn
    python -m fadtk_b200.nearest vggish /tmp/mn/base /tmp/mn/ev /tmp/mn/one.csv
    torchrun --nproc-per-node 2 --master-addr 127.0.0.1 -m fadtk_b200.nearest vggish /tmp/mn/base /tmp/mn/ev /tmp/mn/two.csv
    python tests/multi_gpu_nearest_check.py compare /tmp/mn two
"""
import sys
from pathlib import Path

from multi_gpu_kad_check import prepare


def compare(root: Path, tag: str):
    a, b = (root / "one.csv").read_text(), (root / f"{tag}.csv").read_text()
    assert a == b, "the per-file nearest tables differ"
    print(f"multi-GPU nearest identical: {len(a.splitlines()) - 1} lines ({tag})")


if __name__ == "__main__":
    if sys.argv[1] == "prepare":
        prepare(Path(sys.argv[2]))
    else:
        compare(Path(sys.argv[2]), sys.argv[3])
