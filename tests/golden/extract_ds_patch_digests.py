#!/usr/bin/env python
"""Record tests/golden/ds_patch_digests.json: one SHA-256 per seed over every patch segment the DS encoder
emits on the seeded DsWorld streams of tests/test_ds_informer.py (60 flushes, one to five events each).

    python tests/golden/extract_ds_patch_digests.py

The recorded digests are those of the DS encoder before it had a link table; tests/test_ds_links.py
checks that an encoder without a link resolver still emits exactly these bytes.
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from ds_world import DsWorld  # noqa: E402
from lws_b200 import ds_informer  # noqa: E402

SEEDS = (1, 2, 3, 4)


def digest(seed: int) -> str:
    world = DsWorld(seed)
    enc = ds_informer.DsIncrementalEncoder(world.initial_items(), spare=1.0)
    h = hashlib.sha256()
    for t in enc.tables():
        h.update(t.tobytes())
    for _ in range(60):
        for _ in range(int(world.rng.integers(1, 6))):
            world.step(enc)
        patches = enc.flush()
        for table, rows, values in patches.segments:
            h.update(int(table).to_bytes(4, "little"))
            h.update(rows.tobytes())
            h.update(values.tobytes())
        h.update(b"|reload" if enc.needs_reload else b"|")
        if enc.needs_reload:
            enc = ds_informer.DsIncrementalEncoder([world.item(k) for k in world.items], spare=1.0)
            for t in enc.tables():
                h.update(t.tobytes())
    return h.hexdigest()


def main():
    out = {str(s): digest(s) for s in SEEDS}
    with open(os.path.join(HERE, "ds_patch_digests.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(out)


if __name__ == "__main__":
    main()
