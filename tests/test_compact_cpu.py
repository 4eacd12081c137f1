"""CPU checks of the compact receive format: the numpy dtypes match the C structs of include/swarmdb_b200.h, and
expand_compact rebuilds receive_batch's (headers, payload) from synthetic compact results."""
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]

LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "swarmdb_b200.h"
#define F(S, m) printf(#S " " #m " %zu %zu\n", offsetof(S, m), sizeof(((S*)0)->m))
int main(void) {
  printf("sdb_recv_entry size %zu\n", sizeof(sdb_recv_entry));
  F(sdb_recv_entry, seq); F(sdb_recv_entry, send); F(sdb_recv_entry, receiver);
  printf("sdb_recv_send size %zu\n", sizeof(sdb_recv_send));
  F(sdb_recv_send, timestamp); F(sdb_recv_send, payload_off); F(sdb_recv_send, sender); F(sdb_recv_send, group);
  F(sdb_recv_send, len); F(sdb_recv_send, prio); F(sdb_recv_send, type); F(sdb_recv_send, reserved);
  return 0;
}
"""


def test_dtypes_match_the_c_structs(tmp_path):
    from swarmdb_b200._native import ENTRY_DTYPE, SEND_DTYPE
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text(LAYOUT_C)
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{ROOT / 'include'}",
                           str(src), "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    for struct, dt in (("sdb_recv_entry", ENTRY_DTYPE), ("sdb_recv_send", SEND_DTYPE)):
        lines = [ln.split() for ln in out if ln.startswith(struct + " ")]
        assert lines[0][1] == "size" and int(lines[0][2]) == dt.itemsize
        fields = {ln[1]: (int(ln[2]), int(ln[3])) for ln in lines[1:]}
        assert list(fields) == list(dt.names)
        for name, (off, size) in fields.items():
            assert dt.fields[name][1] == off and dt.fields[name][0].itemsize == size, (struct, name)


def _pad32(n):
    return (np.asarray(n, np.int64) + 31) & ~31


def _compact_from_records(rng, hdr, payloads, image):
    """Build a compact result from full records: `image[r]` names record r's payload image (records with the same
    image share header fields and bytes); rows in first-appearance order."""
    from swarmdb_b200._native import ENTRY_DTYPE, SEND_DTYPE
    _, first, inv = np.unique(image, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")
    rank = np.empty(len(order), np.int64); rank[order] = np.arange(len(order))
    heads = first[order]
    ent = np.zeros(len(hdr), ENTRY_DTYPE)
    ent["seq"], ent["receiver"], ent["send"] = hdr["seq"], hdr["receiver"], rank[inv]
    snd = np.zeros(len(heads), SEND_DTYPE)
    for f in ("timestamp", "sender", "group", "len", "prio", "type"):
        snd[f] = hdr[f][heads]
    plen = _pad32(snd["len"])
    off = np.zeros(len(heads), np.int64)
    if len(heads) > 1:
        np.cumsum(plen[:-1], out=off[1:])
    snd["payload_off"] = off
    pay = np.concatenate([payloads[h] for h in heads]) if len(heads) else np.zeros(0, np.uint8)
    return ent, snd, pay


def _records(rng, n_images, members, max_len, zero_len=False):
    from swarmdb_b200._native import HDR_DTYPE
    image = rng.integers(0, n_images, int(n_images * members)) if n_images else np.zeros(0, np.int64)
    n = len(image)
    lens = np.zeros(n_images, np.int64) if zero_len else rng.integers(0, max_len + 1, n_images)
    img_pay = [rng.integers(0, 256, _pad32(L)).astype(np.uint8) for L in lens]
    hdr = np.zeros(n, HDR_DTYPE)
    hdr["seq"] = rng.permutation(n) + 1
    hdr["receiver"] = rng.integers(0, 1 << 20, n)
    for f, hi in (("sender", 1 << 20), ("group", 1 << 14), ("prio", 4), ("type", 7)):
        per = rng.integers(0, hi, n_images)
        hdr[f] = per[image]
    hdr["timestamp"] = rng.random(n_images)[image]
    hdr["len"] = lens[image]
    payloads = [img_pay[i] for i in image]
    return hdr, payloads, image


@pytest.mark.parametrize("case", ["mixed", "one_row_many_entries", "zero_length", "all_distinct", "empty"])
def test_expand_compact_round_trips(case):
    from swarmdb_b200._native import expand_compact
    rng = np.random.default_rng(["mixed", "one_row_many_entries", "zero_length", "all_distinct", "empty"].index(case))
    if case == "mixed":
        hdr, payloads, image = _records(rng, 300, 5.5, 256)
    elif case == "one_row_many_entries":
        hdr, payloads, image = _records(rng, 1, 4096, 200)
    elif case == "zero_length":
        hdr, payloads, image = _records(rng, 50, 3, 0, zero_len=True)
    elif case == "all_distinct":
        hdr, payloads, _ = _records(rng, 700, 1, 65504 // 64)
        image = np.arange(len(hdr))
    else:
        hdr, payloads, image = _records(rng, 0, 1, 0)
    ent, snd, pay = _compact_from_records(rng, hdr, payloads, image)
    h2, p2 = expand_compact(ent, snd, pay)
    assert h2.tobytes() == hdr.tobytes()
    want = np.concatenate(payloads) if payloads else np.zeros(0, np.uint8)
    assert p2.tobytes() == want.tobytes()
    if case == "one_row_many_entries":
        assert len(snd) == 1 and len(pay) == _pad32(snd["len"][0])
    if case == "zero_length":
        assert len(pay) == 0 and len(p2) == 0 and len(snd) == len(np.unique(image))


def test_expand_compact_takes_views_of_larger_buffers():
    """Results are views into reusable buffers; a payload buffer longer than the returned bytes is fine."""
    from swarmdb_b200._native import expand_compact
    rng = np.random.default_rng(9)
    hdr, payloads, image = _records(rng, 40, 4, 100)
    ent, snd, pay = _compact_from_records(rng, hdr, payloads, image)
    big = np.zeros(len(pay) + 4096, np.uint8); big[: len(pay)] = pay
    h2, p2 = expand_compact(ent, snd, big[: len(pay)])
    assert h2.tobytes() == hdr.tobytes() and p2.tobytes() == np.concatenate(payloads).tobytes()
