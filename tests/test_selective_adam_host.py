"""Visibility-masked Adam without a GPU: the C ABI's argument checks (libgsr_selective_adam.so), the Python layer's
mask checks, the OR of masks over ranks under gloo, and the kernels in the built libraries."""
import ctypes as C
import json
import os
import re
import shutil
import socket
import subprocess
from pathlib import Path

import pytest
import torch

from gaussian_splatting_b200.flat_adam import FlatAdam, section_ends, sh_rest_of_layout

ROOT = Path(__file__).resolve().parents[1]
SEL_LIB = ROOT / "gaussian_splatting_b200" / "libgsr_selective_adam.so"
MAIN_LIB = ROOT / "gaussian_splatting_b200" / "libgsr_b200.so"
GSR_ERR_BAD_ARG = -1
P = C.c_void_p


def _lib():
    so = C.CDLL(str(SEL_LIB))
    so.gsr_adam_step_selective.argtypes = [C.c_int64, C.c_int, P, P, P, P, P, C.c_int, P, P, C.c_double, C.c_double,
                                           C.c_double, C.c_int, P]
    so.gsr_adam_step_selective_sharded.argtypes = [C.c_int64, C.c_int64, C.c_int, P, P, P, C.c_int, P, P, C.c_int64,
                                                   C.c_int, C.c_int, P, P, C.c_double, C.c_double, C.c_double, C.c_int,
                                                   P]
    return so


def _arrays(n_rows, n_rest, ends=None):
    ends = section_ends(n_rows, n_rest) if ends is None else ends
    e = (C.c_int64 * len(ends))(*ends)
    lr = (C.c_double * len(ends))(*([1e-3] * len(ends)))
    return len(ends), e, lr


def test_header_declares_and_library_exports_the_entry_points():
    text = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "gsr_selective_adam.h").read_text(), flags=re.S)
    declared = sorted(set(re.findall(r"\b(gsr_[a-z0-9_]+)\s*\(", text)))
    assert declared == ["gsr_adam_step_selective", "gsr_adam_step_selective_sharded"]
    so = C.CDLL(str(SEL_LIB))
    assert all(hasattr(so, s) for s in declared)
    main = C.CDLL(str(MAIN_LIB))
    assert not any(hasattr(main, s) for s in declared), "the selective step must stay out of libgsr_b200.so"


def test_selective_argument_errors():
    """Every check fires before any launch: fake (never dereferenced) device pointers for the buffers."""
    so = _lib()
    p, g, m, v, vis = (P(0x1000000 * k) for k in range(1, 6))

    def call(n_rows=1001, n_rest=15, ends=None, vis_=vis, step=1, bufs=(p, g, m, v)):
        ns, e, lr = _arrays(max(n_rows, 0), n_rest, ends)
        return so.gsr_adam_step_selective(n_rows, n_rest, *bufs, vis_, ns, e, lr, 0.9, 0.999, 1e-8, step, None)

    assert call(n_rows=-1) == GSR_ERR_BAD_ARG
    assert call(n_rest=-1, ends=section_ends(1001, 0)) == GSR_ERR_BAD_ARG
    assert call(vis_=None) == GSR_ERR_BAD_ARG                                       # no mask
    assert call(step=0) == GSR_ERR_BAD_ARG
    assert call(bufs=(p, None, m, v)) == GSR_ERR_BAD_ARG
    assert call(ends=section_ends(1000, 15)) == GSR_ERR_BAD_ARG                     # layout of another N
    assert call(ends=section_ends(1001, 8)) == GSR_ERR_BAD_ARG                      # layout of another SH width
    assert call(ends=section_ends(1001, 15)[:5]) == GSR_ERR_BAD_ARG                 # a section missing
    assert call(ends=section_ends(1001, 15)[:5] + [section_ends(1001, 15)[5] + 4]) == GSR_ERR_BAD_ARG
    assert call(n_rows=100_000_000, ends=section_ends(100_000_000, 15)) == GSR_ERR_BAD_ARG  # past 32-bit offsets
    assert call(n_rows=0, ends=section_ends(0, 15), vis_=None, bufs=(None,) * 4) == 0  # empty: ok, nothing launched


def test_sharded_argument_errors():
    so = _lib()
    n_rows, n_rest = 1001, 15
    total = section_ends(n_rows, n_rest)[-1]
    world = 2
    grads = (P * world)(*[0x1000000 * (k + 1) for k in range(world)])
    params = (P * world)(*[0x3000000 * (k + 1) for k in range(world)])
    vis = (P * world)(*[0x9000000 * (k + 1) for k in range(world)])
    vis_hole = (P * world)(0x9000000, None)
    m, v = P(0x20000000), P(0x30000000)

    def call(lo=0, hi=total // 2 // 4 * 4, world_=world, rank=0, peers_vis=vis, rows=n_rows, rest=n_rest, ends=None):
        ns, e, lr = _arrays(max(rows, 0), max(rest, 0), ends)
        return so.gsr_adam_step_selective_sharded(lo, hi, world_, grads, params, peers_vis, rank, m, v, rows, rest, ns,
                                                  e, lr, 0.9, 0.999, 1e-8, 1, None)

    assert call(rows=-1, ends=section_ends(0, n_rest)) == GSR_ERR_BAD_ARG
    assert call(ends=section_ends(1002, n_rest)) == GSR_ERR_BAD_ARG                  # inconsistent sections
    assert call(peers_vis=None) == GSR_ERR_BAD_ARG                                  # no masks
    assert call(peers_vis=vis_hole) == GSR_ERR_BAD_ARG                              # one rank's mask missing
    assert call(rank=2) == GSR_ERR_BAD_ARG                                          # rank outside the world
    assert call(rank=-1) == GSR_ERR_BAD_ARG
    assert call(world_=0, rank=0) == GSR_ERR_BAD_ARG
    assert call(world_=17) == GSR_ERR_BAD_ARG
    assert call(lo=2) == GSR_ERR_BAD_ARG                                            # shard not 16-byte aligned
    assert call(lo=8, hi=4) == GSR_ERR_BAD_ARG
    assert call(hi=total + 4) == GSR_ERR_BAD_ARG                                    # shard past the buffer
    assert call(lo=0, hi=0) == 0                                                    # empty shard: ok


def test_binding_rejects_cpu_tensors_and_wrong_masks():
    from gaussian_splatting_b200 import native

    n, rest = 10, 3
    ends = section_ends(n, rest)
    p, g, m, v = (torch.zeros(ends[-1]) for _ in range(4))
    lrs = [1e-3] * len(ends)
    with pytest.raises(RuntimeError, match="not a CUDA tensor"):
        native().adam_step_selective(p, g, m, v, torch.ones(n, dtype=torch.bool), rest, ends, lrs, 0.9, 0.999, 1e-8, 1)
    opt = FlatAdam(p, ends, lrs)
    with pytest.raises(RuntimeError, match="not a CUDA tensor"):
        opt.step(g, visible=torch.ones(n, dtype=torch.bool))
    with pytest.raises(ValueError, match="stale mask"):
        opt.step(g, visible=torch.ones(n + 1, dtype=torch.bool))
    with pytest.raises(TypeError, match="bool or uint8"):
        opt.step(g, visible=torch.ones(n, dtype=torch.int32))
    assert opt.t == 0  # a rejected mask does not count as a step
    with pytest.raises(RuntimeError):
        native().adam_step_selective_sharded(0, 4, [0], [0], [0], 0, torch.zeros(4), torch.zeros(4), n, rest, ends, lrs,
                                             0.9, 0.999, 1e-8, 1)


@pytest.mark.parametrize("rest", [0, 3, 8, 15])
def test_sh_width_is_recovered_from_the_layout(rest):
    for n in (2, 3, 1001):
        assert sh_rest_of_layout(section_ends(n, rest), n) == rest
    # one row: the padding can hold a whole coefficient, so the width is only known up to the same layout
    assert section_ends(1, sh_rest_of_layout(section_ends(1, rest), 1)) == section_ends(1, rest)
    for n in (1, 2, 3, 1001):
        with pytest.raises(ValueError):
            sh_rest_of_layout(section_ends(n, rest), n + 7)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _vis_worker(rank, world, port, out):
    import torch.distributed as dist

    from gaussian_splatting_b200.view_parallel import all_reduce_visibility

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        n = 1001
        u8 = torch.zeros(n, dtype=torch.uint8)
        u8[rank::3] = 1 + rank                       # any nonzero byte means "seen"
        b = torch.zeros(n, dtype=torch.bool)
        b[rank * 7::5] = True
        ptr = b.data_ptr()
        assert all_reduce_visibility(u8) is u8 and all_reduce_visibility(b) is b
        assert b.data_ptr() == ptr and b.dtype == torch.bool
        out.put((rank, u8.tolist(), b.tolist()))
    finally:
        dist.destroy_process_group()


def test_all_reduce_visibility_two_ranks_gloo():
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    world, port = 2, _free_port()
    procs = [ctx.Process(target=_vis_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict((r, (u, b)) for r, u, b in (q.get(timeout=120) for _ in range(world)))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    n = 1001
    want_u = [max(1 + r if i % 3 == r else 0 for r in range(world)) for i in range(n)]
    want_b = [any(i >= r * 7 and (i - r * 7) % 5 == 0 for r in range(world)) for i in range(n)]
    for r in range(world):
        assert got[r][0] == want_u and got[r][1] == want_b


def test_all_reduce_visibility_without_process_group_is_a_no_op():
    from gaussian_splatting_b200.view_parallel import all_reduce_visibility

    x = torch.tensor([0, 1, 0], dtype=torch.uint8)
    assert all_reduce_visibility(x) is x and x.tolist() == [0, 1, 0]


# the kernels in the built libraries ------------------------------------------------------------------------------
def _tool(name):
    exe = shutil.which(name) or f"/usr/local/cuda/bin/{name}"
    if not Path(exe).exists():
        pytest.skip(f"{name} is missing")
    return exe


def _kernel_names(lib):
    sass = subprocess.run([_tool("cuobjdump"), "-sass", str(lib)], check=True, capture_output=True, text=True).stdout
    return sass, re.findall(r"Function : (\S+)", sass)


def test_selective_library_is_sm90a_only_without_local_memory():
    elfs = subprocess.run([_tool("cuobjdump"), "-lelf", str(SEL_LIB)], capture_output=True, text=True).stdout
    assert set(re.findall(r"sm_(\d+a?)", elfs)) == {"90a"}
    sass, names = _kernel_names(SEL_LIB)
    assert sorted(names) == sorted(n for n in names if "16k_adam_selective" in n) and len(names) == 2, names
    usage = subprocess.run([_tool("cuobjdump"), "--dump-resource-usage", str(SEL_LIB)], check=True,
                           capture_output=True, text=True).stdout
    found = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", usage))
    assert sorted(found) == sorted(names)
    for name, line in found.items():
        u = {k: int(v) for k, v in re.findall(r"([A-Z]+(?:\[0\])?):(\d+)", line)}
        assert u["LOCAL"] == 0 and u["STACK"] == 0, (name, u)
    assert not re.search(r"\b(?:STL|LDL)\b", sass)


def test_main_library_has_the_kernels_of_the_parent():
    """libgsr_b200.so keeps exactly its kernel set: those recorded before MCMC plus the three MCMC kernels."""
    rec = json.loads((ROOT / "tests" / "golden" / "sass_digests_before_mcmc.json").read_text())["kernels"]
    _, names = _kernel_names(MAIN_LIB)
    extra = sorted(set(names) - set(rec))
    assert set(rec) <= set(names)
    assert len(extra) == 3 and all(any(k in n for n in extra) for k in ("k_mcmc_relocation", "k_mcmc_apply",
                                                                        "k_mcmc_noise")), extra
    assert not any("selective" in n for n in names)
