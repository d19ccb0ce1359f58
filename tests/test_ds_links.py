"""The DS encoder's link table (LWSE_TABLE_DS_LINKS): after every DS flush each revision-role row links to
what a fresh resolution by child name gives (LWS row and uid_hash from the LWS encoder, or NONE), with
LWS objects created and deleted (rows reused) and both encoders flushed in random order; an encoder
without a resolver emits exactly the bytes it emitted before links existed; the header layout."""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

from ds_link_world import LinkWorld, fresh_links, linked_revroles, none_links
from lws_b200 import records as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))


def _check_links(w: LinkWorld, mirror, where):
    enc = w.ds_enc
    assert mirror.tobytes() == enc.links.tobytes(), f"{where}: patched mirror vs encoder"
    owned = np.zeros(len(enc.links), bool)
    for key in sorted(enc.items):
        sl = enc.slots[key]
        got = enc.links[sl.rev_base: sl.rev_base + sl.rev_cap]
        assert got.tobytes() == fresh_links(enc, w.lws_enc, key).tobytes(), f"{where}: {key}"
        owned[sl.rev_base: sl.rev_base + sl.rev_cap] = True
    assert mirror[~owned].tobytes() == none_links(int((~owned).sum())).tobytes(), f"{where}: rows no DS owns"


@pytest.mark.parametrize("seed", [1, 2, 3, 4, 5, 6])
def test_links_follow_lws_rows(seed):
    w = LinkWorld(seed)
    mirror = w.ds_enc.links.copy()  # what the first DS tick after a load sends as one range
    _check_links(w, mirror, "initial")
    relinked = 0
    for step in range(80):
        for _ in range(int(w.rng.integers(1, 5))):
            w.step()
        order = ["lws", "ds"] if w.rng.random() < 0.5 else ["ds", "lws"]
        for which in order:
            if which == "lws":
                w.lws_enc.flush()
                assert not w.lws_enc.needs_reload
                relinked += len(w.lws_enc.moved_keys)
                w.ds_enc.relink(w.lws_enc.moved_keys)
                continue
            p = w.ds_enc.flush()
            if w.ds_enc.needs_reload:  # (a caller re-encodes, reloads and sends the link table whole)
                from lws_b200 import ds_informer

                w.ds_enc = ds_informer.DsIncrementalEncoder([w.ds.item(k) for k in w.ds.items], spare=1.0,
                                                            links=w.lws_enc)
                mirror = w.ds_enc.links.copy()
            else:
                for table, rows, values in p.segments:
                    if table == R.TABLE_DS_LINKS:
                        mirror[rows] = values
            _check_links(w, mirror, f"seed {seed} step {step}")
    assert relinked > 0


def test_moved_keys_are_the_rows_taken_and_given_back():
    w = LinkWorld(9)
    enc = w.lws_enc
    key = sorted(w.lws)[0]
    row, uid = enc.lws_link(*key)
    enc.lws_event("DELETED", w.lws.pop(key))
    assert enc.lws_link(*key) == (row, uid)  # still resident until the flush
    enc.flush()
    assert enc.moved_keys == {key} and enc.lws_link(*key) is None
    w.lws[key] = w._item(*key)
    enc.lws_event("ADDED", w.lws[key])
    enc.flush()
    assert enc.moved_keys == {key}
    row2, uid2 = enc.lws_link(*key)
    assert row2 == row and uid2 != uid  # the freed row, another object
    enc.lws_event("MODIFIED", w.lws[key])
    enc.flush()
    assert enc.moved_keys == set()
    w.lws[key] = w._item(*key)  # replaced under its name: a new uid in the same row
    enc.lws_event("MODIFIED", w.lws[key])
    enc.flush()
    assert enc.moved_keys == {key}
    row3, uid3 = enc.lws_link(*key)
    assert row3 == row2 and uid3 != uid2


def test_replaced_child_is_relinked():
    """A child replaced under its name (new uid, same LWS row) is re-linked by the next DS flush."""
    w = LinkWorld(11)
    linked = [(k, s) for k, s in w.ds_enc.slots.items()
              if (w.ds_enc.links[s.rev_base: s.rev_base + s.rev_cap]["lws_row"] != R.NONE).any()]
    key, sl = linked[0]
    rows = w.ds_enc.links[sl.rev_base: sl.rev_base + sl.rev_cap]
    i = int(np.flatnonzero(rows["lws_row"] != R.NONE)[0])
    lws_key = w.lws_enc.object_of_lws_row(int(rows["lws_row"][i]))
    w.lws[lws_key] = w._item(*lws_key)
    w.lws_enc.lws_event("MODIFIED", w.lws[lws_key])
    w.lws_enc.flush()
    w.ds_enc.relink(w.lws_enc.moved_keys)
    p = w.ds_enc.flush()
    segs = [sg for sg in p.segments if sg[0] == R.TABLE_DS_LINKS]
    assert len(segs) == 1 and sl.rev_base + i in segs[0][1].tolist()
    assert w.ds_enc.links[sl.rev_base + i]["lws_uid_hash"] == w.lws_enc.lws_link(*lws_key)[1]


def test_without_resolver_patches_match_recorded_digests():
    """The DsWorld streams of test_ds_informer, hashed as tests/golden/extract_ds_patch_digests.py
    recorded them before the link table existed."""
    import sys

    sys.path.insert(0, os.path.join(HERE, "golden"))
    import extract_ds_patch_digests as X

    want = json.load(open(os.path.join(HERE, "golden", "ds_patch_digests.json")))
    for seed in X.SEEDS:
        assert X.digest(seed) == want[str(seed)], seed


def test_linked_revroles_rule():
    """The test-side statement of the rule, on one row per condition."""
    rr = R.aligned_empty(8, R.DS_REVROLE_REC)
    rr["ready_replicas"] = 1
    rr["flags"] = R.RR_EXISTS
    rr["flags"][6] = 0  # a row without RR_EXISTS
    lws = R.aligned_empty(4, R.LWS_REC)
    lws["uid_hash"] = [11, 12, 13, 14]
    lo = R.aligned_empty(4, R.LWS_OUT)
    lo["ready_replicas"] = [5, 6, 7, 8]
    lo["flags"][2] = R.LOUT_STATUS_ERROR
    links = none_links(8)
    #                row 0: ok   1: uid   2: flags  3: L>=n  4: none  5: ok   6: !exists 7: none
    links["lws_row"][:7] = [0, 1, 2, 4, R.NONE, 3, 0]
    links["lws_uid_hash"][:7] = [11, 99, 13, 0, 0, 14, 11]
    got, took, fell = linked_revroles(rr, links, lws, lo)
    assert got["ready_replicas"].tolist() == [5, 1, 1, 1, 1, 8, 1, 1] and (took, fell) == (2, 4)
    got, took, fell = linked_revroles(rr, links)  # no LWS results
    assert got["ready_replicas"].tolist() == [1] * 8 and (took, fell) == (0, 6)


def test_link_layout_matches_header():
    """sizeof / offsetof of lwse_ds_link and lwse_ds_tick_info via a gcc-compiled probe, and the table id."""
    info = [f for f, _ in R.DsTickInfo._fields_]
    link = list(R.DS_LINK.names)
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{ROOT}/include/lwse.h"', "int main(){",
             'printf("link_size %zu\\n", sizeof(lwse_ds_link));', 'printf("info_size %zu\\n", sizeof(lwse_ds_tick_info));',
             'printf("id %d\\n", (int)LWSE_TABLE_DS_LINKS);']
    lines += [f'printf("link.{f} %zu\\n", offsetof(lwse_ds_link, {f}));' for f in link]
    lines += [f'printf("info.{f} %zu\\n", offsetof(lwse_ds_tick_info, {f}));' for f in info]
    lines += ["return 0;}"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(src, "w").write("\n".join(lines))
        subprocess.run(["gcc", "-o", exe, src], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    got = dict(l.split(" ", 1) for l in out.strip().splitlines())
    assert int(got["link_size"]) == R.DS_LINK.itemsize == 16
    assert int(got["info_size"]) == C.sizeof(R.DsTickInfo) == 24
    assert int(got["id"]) == R.TABLE_DS_LINKS == 9
    for f in link:
        assert int(got[f"link.{f}"]) == R.DS_LINK.fields[f][1], f
    for f in info:
        assert int(got[f"info.{f}"]) == getattr(R.DsTickInfo, f).offset, f
