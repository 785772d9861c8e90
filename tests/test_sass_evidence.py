"""The built library really contains the Hopper instructions DESIGN.md claims (cuobjdump needs no GPU).
SASS mnemonics: UBLKCP = 1-D TMA bulk copy (cp.async.bulk), SYNCS = mbarrier transaction arrive/wait,
LDGSTS = cp.async, REDG = global reduction."""
import collections
import re
import shutil
import subprocess
from pathlib import Path

import pytest

LIB = Path(__file__).resolve().parents[1] / "gaussian_splatting_b200" / "libgsr_b200.so"


def sass_counts():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(exe).exists() or not LIB.exists():
        pytest.skip("cuobjdump or the built library is missing")
    text = subprocess.run([exe, "-sass", str(LIB)], check=True, capture_output=True, text=True).stdout
    cur, counts = None, collections.defaultdict(collections.Counter)
    for line in text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
        if m and cur:
            counts[cur][m.group(1)] += 1
    assert "sm_90a" in text or counts, "no SASS found"
    return counts


def find(counts, fragment):
    hits = [c for name, c in counts.items() if fragment in name]
    assert hits, f"kernel {fragment} not in the library"
    return hits[0]


def test_tile_kernels_pair_pixels_without_cta_barriers():
    counts = sass_counts()
    for masks in ("ILb1EE", "ILb0EE"):
        for k in ("k_render_fwd", "k_render_bwd"):
            c = find(counts, f"gsr{len(k)}{k}{masks}")  # N3gsr<len><name>I<template args>E
            assert c["FFMA"] >= 20 and c["FMUL"] >= 20, (k, masks, dict(c))  # two pixels per lane: every op issued twice
            assert c["BAR"] <= 4, (k, masks, dict(c))                        # no CTA barrier in the batch loops


def test_gather_variants_fetch_records_with_cp_async_on_the_stage_barrier():
    """The tile kernels read no tile-ordered copy of the records: the warp that recycles a stage gathers the batch's
    records with 16-byte cp.async (SASS LDGSTS) and signals the stage's mbarrier (SYNCS / ARRIVES)."""
    counts = sass_counts()
    for k in ("k_render_fwd", "k_render_bwd"):
        c = find(counts, f"gsr{len(k)}{k}ILb1EE")
        assert c["LDGSTS"] >= 3 and c["SYNCS"] >= 1, (k, dict(c))
        assert c["FFMA"] >= 20 and c["BAR"] <= 4, (k, dict(c))


def test_per_gaussian_kernels_stage_through_tma():
    counts = sass_counts()
    fwd = find(counts, "k_preprocess_fwdILi16ELb1")
    bwd = find(counts, "k_preprocess_bwdILi16ELb1")
    assert fwd["UBLKCP"] >= 2 and bwd["UBLKCP"] >= 6   # SH slice in + records out; six gradient slices out


def _tool_output(*args):
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(exe).exists() or not LIB.exists():
        pytest.skip("cuobjdump or the built library is missing")
    return subprocess.run([exe, *args, str(LIB)], check=True, capture_output=True, text=True).stdout


def test_render_backward_flushes_gradient_rows_with_vector_reductions():
    """DESIGN.md 3.7: a (gaussian, tile) pair's nine sums leave as two 16-byte vector reductions
    (red.global.add.v4.f32 -> SASS REDG.E.ADD.F32x4) + one scalar, not as nine scalar atomics."""
    text = _tool_output("-sass")
    body = text.split("Function : _ZN3gsr12k_render_bwdILb1EE", 1)[1].split("Function :", 1)[0]
    assert len(re.findall(r"REDG\.E\.ADD\.F32x4", body)) >= 2, "no 16-byte vector reductions in the render backward"


def test_render_kernels_keep_the_occupancy_design_md_states():
    """DESIGN.md 3.8 / 6: the backward runs 8 CTAs per SM (<= 64 registers, <= 28 KB of shared memory per CTA), the
    forward 9 (<= 56 registers); neither keeps arrays in local memory."""
    text = _tool_output("--dump-resource-usage")
    usage = {}
    for name, line in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", text):
        usage[name] = {k: int(v) for k, v in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", line)}
    bwd = next(v for k, v in usage.items() if "12k_render_bwdILb1EE" in k)
    fwd = next(v for k, v in usage.items() if "12k_render_fwdILb1EE" in k)
    assert bwd["REG"] <= 64 and bwd["SHARED"] <= 28 * 1024 and bwd["STACK"] <= 16, bwd
    assert fwd["REG"] <= 56 and fwd["SHARED"] <= 24 * 1024, fwd
    assert 8 * (bwd["SHARED"] + 1024) <= 227 * 1024  # eight resident CTAs fit the SM's shared memory
