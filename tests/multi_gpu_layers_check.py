"""Manual multi-GPU check (not collected by pytest): the per-layer sweep under torchrun must write the same caches, byte
for byte, and the same scores as a single process.  Usage on a box with >= 2 GPUs:

    FADTK_SYNTHETIC=1 python tests/multi_gpu_layers_check.py prepare /tmp/ml
    FADTK_SYNTHETIC=1 python -m fadtk_b200.layers MERT-v1-95M /tmp/ml/one/base /tmp/ml/one/eval /tmp/ml/one.csv
    FADTK_SYNTHETIC=1 torchrun --nproc-per-node 2 --master-addr 127.0.0.1 -m fadtk_b200.layers MERT-v1-95M \
        /tmp/ml/two/base /tmp/ml/two/eval /tmp/ml/two.csv
    python tests/multi_gpu_layers_check.py compare /tmp/ml
"""
import shutil
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def prepare(root: Path):
    from fadtk_b200 import synth
    for kind, n in (("base", 9), ("eval", 7)):
        d = root / "one" / kind
        d.mkdir(parents=True, exist_ok=True)
        for i in range(n):
            secs = (2.0, 5.0, 7.5, 10.0, 31.0)[i % 5] if kind == "eval" else 3.0 + 0.75 * i
            synth.write_wav(d / f"f{i:02d}.wav", synth.musiclike_clip(i, secs, 24000, baseline=(kind == "base")), 24000)
    shutil.copytree(root / "one", root / "two")


def compare(root: Path):
    one = {p.relative_to(root / "one"): p for p in sorted((root / "one").rglob("embeddings/*/*.npy"))}
    two = {p.relative_to(root / "two"): p for p in sorted((root / "two").rglob("embeddings/*/*.npy"))}
    assert sorted(one) == sorted(two) and len(one) == 16 * 12, (len(one), len(two))
    for rel in one:
        assert one[rel].read_bytes() == two[rel].read_bytes(), rel
    a = [ln.split(",")[:4] for ln in (root / "one.csv").read_text().splitlines()[1:]]
    b = [ln.split(",")[:4] for ln in (root / "two.csv").read_text().splitlines()[1:]]
    assert [r[0] for r in a] == [r[0] for r in b] and [r[3] for r in a] == [r[3] for r in b], (a, b)
    print(f"multi-GPU layer sweep identical: {len(one)} caches, {len(a)} scores")


if __name__ == "__main__":
    {"prepare": prepare, "compare": compare}[sys.argv[1]](Path(sys.argv[2]))
