"""DisaggregatedSet and child-LeaderWorkerSet events through the DS encoder: after every flush the
resident tables with the patches applied mean, DS by DS, what a fresh ``encode_ds`` of the same
objects means, and give the oracle the same results; a reload is asked for exactly when spare rows
run out.  Also the layout of ``lwse_ds_changes`` against the header."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from ds_world import DsWorld, apply_patches, check_against_fresh
from lws_b200 import api, ds_informer, encoder
from lws_b200 import records as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_event_streams_match_fresh_encode(seed):
    world = DsWorld(seed)
    enc = ds_informer.DsIncrementalEncoder(world.initial_items(), spare=1.0)
    mirror = [t.copy() for t in enc.tables()]
    check_against_fresh(world, enc, mirror, "initial")
    for step in range(60):
        for _ in range(int(world.rng.integers(1, 6))):
            world.step(enc)
        patches = enc.flush()
        if enc.needs_reload:  # (spare rows ran out: re-encode everything, as a caller reloads)
            enc = ds_informer.DsIncrementalEncoder([world.item(k) for k in world.items], spare=1.0)
            mirror = [t.copy() for t in enc.tables()]
        else:
            apply_patches(mirror, patches)
        for t, m in zip(enc.tables(), mirror):
            assert t.tobytes() == m.tobytes(), f"seed {seed} step {step}: encoder tables vs patched mirror"
        check_against_fresh(world, enc, mirror, f"seed {seed} step {step}")


def test_status_update_is_one_revrole_row():
    """The common event — a child's readyReplicas changes — patches exactly one revision-role row."""
    world = DsWorld(7, n_ds=3)
    enc = ds_informer.DsIncrementalEncoder(world.initial_items())
    key = sorted(world.items)[1]
    role, rev = next(iter(world.children[key]))
    c = world.children[key][(role, rev)]
    c2 = api.ChildLWS(c.role, c.revision, c.replicas, c.readyReplicas + 1, c.creationTimestamp, dict(c.annotations))
    enc.child_event("MODIFIED", key[0], key[1], c2)
    p = enc.flush()
    assert [(t, len(r)) for t, r, _ in p.segments] == [(R.TABLE_DS_REVROLES, 1)]
    row = int(p.segments[0][1][0])
    sl = enc.slots[key]
    assert sl.rev_base <= row < sl.rev_base + sl.rev_cap
    assert int(p.segments[0][2]["ready_replicas"][0]) == c.readyReplicas + 1
    assert enc.flush().n_rows() == 0  # nothing dirty: nothing emitted


def _two_role_ds(i):
    return api.DisaggregatedSet(f"n{i}", "x", roles=[api.DisaggregatedRoleSpec("p", 1), api.DisaggregatedRoleSpec("d", 1)])


def test_reload_exactly_when_ds_rows_run_out():
    enc = ds_informer.DsIncrementalEncoder([], spare=0.0)  # 4 spare DS rows, 16 role rows, 32 revision-role rows
    assert (len(enc.ds), len(enc.roles), len(enc.revroles)) == (4, 16, 32)
    for i in range(4):  # each takes 1 DS row, 4 role rows (_slack(2)) and 4 revision-role rows
        enc.ds_event("ADDED", _two_role_ds(i), "r")
    p = enc.flush()
    assert not enc.needs_reload and p.n_rows() > 0
    enc.ds_event("DELETED", _two_role_ds(0), "r")
    enc.ds_event("ADDED", _two_role_ds(4), "r")  # the freed rows are not free before the next flush
    enc.flush()
    assert enc.needs_reload and ("x", "n4") not in enc.slots
    enc.needs_reload = False
    enc.ds_event("ADDED", _two_role_ds(4), "r")
    enc.flush()
    assert not enc.needs_reload and enc.ds_row("x", "n4") == 0  # the row n0 had


def test_reload_exactly_when_revision_rows_run_out():
    """A DS that gains revisions moves its revision-role range to first-fit free rows; the reload is
    asked for on the first growth that no free range and no tail rows can hold."""
    ds = _two_role_ds(0)
    enc = ds_informer.DsIncrementalEncoder([encoder.DsItem(ds, "r0", [])], spare=0.0)
    t = 10.0
    for k in range(1, 40):
        sl = enc.slots[("x", "n0")]
        n_old = k  # revisions r0 .. r{k-1} become old ones once r{k} is the target
        need = (n_old + 1) * 2
        fits = need <= sl.rev_cap
        cap = need + max(2, need // 4)
        free_ok = fits or any(n >= cap for _, n in enc._free_revroles) or enc.rev_end + cap <= len(enc.revroles)
        t += 1
        enc.child_event("ADDED", "x", "n0", api.ChildLWS("p", f"r{k - 1}", 1, 1, t))
        enc.ds_event("MODIFIED", ds, f"r{k}")
        enc.flush()
        assert enc.needs_reload == (not free_ok), k
        if enc.needs_reload:
            break
    assert enc.needs_reload


def test_ds_changes_layout_matches_header():
    """sizeof / offsetof of lwse_ds_changes via a gcc-compiled probe against records.DsChanges, and the
    new table ids."""
    fields = [f for f, _ in R.DsChanges._fields_]
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{ROOT}/include/lwse.h"', "int main(){",
             'printf("size %zu\\n", sizeof(lwse_ds_changes));']
    lines += [f'printf("{f} %zu\\n", offsetof(lwse_ds_changes, {f}));' for f in fields]
    lines += ['printf("ids %d %d %d\\n", (int)LWSE_TABLE_DS, (int)LWSE_TABLE_DS_ROLES, (int)LWSE_TABLE_DS_REVROLES);',
              "return 0;}"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(src, "w").write("\n".join(lines))
        subprocess.run(["gcc", "-o", exe, src], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    got = dict(l.split(" ", 1) for l in out.strip().splitlines())
    assert int(got["size"]) == C.sizeof(R.DsChanges) == 40
    for f in fields:
        assert int(got[f]) == getattr(R.DsChanges, f).offset, f
    assert got["ids"].split() == [str(R.TABLE_DS), str(R.TABLE_DS_ROLES), str(R.TABLE_DS_REVROLES)]
