"""CPU oracle for the embedding -> statistics -> Frechet-distance hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``fadtk_b200/`` imports this package.
The only callers are ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py``, and they use it as
the checker (or as the timed CPU baseline), never as the thing that ships.

Contents
--------
``fad_oracle``      numpy restatement of the reference's statistics + Frechet code
                    (reference: fadtk/fad.py:42-120, :304-395, fadtk/utils.py:13-46).
                    PINNED: checked against the reference's own functions imported
                    from the reference checkout (see ``ref_shims`` / ``make_golden``); the
                    outputs are committed under ``tests/golden/``.
``vggish_oracle``   numpy (fp64) log-mel front-end + torch-CPU fp32 VGG stack that
                    the reference reaches through ``torch.hub.load('harritaylor/
                    torchvggish', 'vggish')`` (fadtk/model_loader.py:99-108).
                    PARITY UNPINNED for the network: torchvggish is an un-vendored,
                    un-pinned hub dependency with no source, weights or golden
                    embeddings in the reference checkout, so this is a restatement of the
                    published algorithm anchored on the reference's call site.
``ref_shims``       import the real ``fadtk`` package from the reference checkout with
                    no-arithmetic stub modules (only usable in the build container).
``make_golden``     regenerates ``tests/golden/*.npz`` from the real reference.
"""
