"""Manual multi-GPU check (not collected by pytest): ``python -m fadtk_b200.prdc --indiv`` under torchrun, where every
rank takes its share of the per-song radii and ball-count tiles, must write the same per-file table as a single
process.  Usage on a box with >= 2 GPUs (and with 4 and 8 where available):

    python tests/multi_gpu_prdc_songs_check.py prepare /tmp/mp
    python -m fadtk_b200.prdc vggish /tmp/mp/base /tmp/mp/ev /tmp/mp/one.csv -k 3 --indiv
    torchrun --nproc-per-node 2 --master-addr 127.0.0.1 -m fadtk_b200.prdc vggish /tmp/mp/base /tmp/mp/ev /tmp/mp/two.csv -k 3 --indiv
    python tests/multi_gpu_prdc_songs_check.py compare /tmp/mp two
"""
import sys
from pathlib import Path

from multi_gpu_kad_check import prepare


def compare(root: Path, tag: str):
    one, other = ((root / f"{t}.csv").read_text() for t in ("one", tag))
    assert one == other, f"the {tag} table differs from the single-process one"
    print(f"multi-GPU per-song PRDC identical: {len(one.splitlines()) - 1} files ({tag})")


if __name__ == "__main__":
    if sys.argv[1] == "prepare":
        prepare(Path(sys.argv[2]))
    else:
        compare(Path(sys.argv[2]), sys.argv[3])
