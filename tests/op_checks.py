"""Checks shared by the GPU tests of the kernel-backed operators: the guarded C-ABI run, the error-code driver, CGLS
graph replay against the step loop, and the multi-rank launch under torchrun."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
TORCH_DT = {np.float32: "float32", np.float64: "float64"}


def host(t):
    """a device tensor (or an array-like) as a NumPy array"""
    return t.cpu().numpy() if hasattr(t, "cpu") else np.asarray(t)


def device_input(x_np, dt, misalign=False):
    """x_np as a contiguous device vector of dtype dt, one element past an allocation's start when ``misalign``"""
    import torch
    s = 1 if misalign else 0
    xb = torch.zeros(x_np.size + s, dtype=getattr(torch, TORCH_DT[dt]), device="cuda")
    xb[s:] = torch.as_tensor(np.ascontiguousarray(x_np, dtype=dt).ravel())
    return xb[s:]


def guarded_twice(call, n, dt, guard=5, offset=0):
    """``call(y)`` twice, y the n elements that start ``offset`` elements past ``guard`` cells of 7.25 and end
    ``guard`` cells before the end of one buffer; returns (the first result on the host, guards intact, second call
    bit-equal)"""
    import torch
    yb = torch.full((n + 2 * guard + offset,), 7.25, dtype=getattr(torch, TORCH_DT[dt]), device="cuda")
    lo = guard + offset
    y = yb[lo:lo + n]
    rc = call(y.data_ptr())
    assert rc == 0, rc
    first = y.clone()
    assert call(y.data_ptr()) == 0
    torch.cuda.synchronize()
    g = host(yb)
    guards_ok = bool(np.all(g[:lo] == 7.25) and np.all(g[lo + n:] == 7.25))
    return host(first), guards_ok, bool(torch.equal(first, y))


def assert_rejected(call, base, cases, y):
    """``call(args)`` with ``base`` updated by each ``kwargs`` of ``cases`` returns its ``rc`` (``y="x"``: y is x),
    and none of the calls touches the device array y"""
    import torch
    before = y.clone()
    for kw, want in cases:
        a = dict(base)
        a.update(kw)
        if a.get("y") == "x":
            a["y"] = a["x"]
        rc = call(a)
        assert rc == want, (kw, rc)
    torch.cuda.synchronize()
    assert torch.equal(y, before)


def assert_cgls_replay_matches_steps(pm, Op, y, x0, niter, min_replays):
    """CGLS over ``Op`` is graph safe, its graph-replayed run replays at least ``min_replays`` iterations, and it
    gives the bits of ``niter`` step() calls: the solution and every cost"""
    from pylops_mpi_b200.optimization.cls_basic import CGLS, _graph_safe
    assert _graph_safe(Op)
    a = CGLS(Op)
    xa = a.setup(y=y, x0=x0, niter=niter, damp=0.0, tol=0.0)
    xa = a.run(xa, niter)
    a.finalize()
    assert a.graph_error is None, a.graph_error
    assert a.graph_replays >= min_replays
    b = CGLS(Op)
    xb = b.setup(y=y, x0=x0, niter=niter, damp=0.0, tol=0.0)
    for _ in range(niter):
        xb = b.step(xb)
    b.finalize()
    np.testing.assert_array_equal(host(xa.asarray()), host(xb.asarray()))
    np.testing.assert_array_equal(np.asarray(a.cost), np.asarray(b.cost))


def needs_gpus(n):
    import torch
    if torch.cuda.device_count() < n:
        pytest.skip(f"needs {n} GPUs, box has {torch.cuda.device_count()}")


def run_on_ranks(script_or_module, nproc, args=(), env=None, timeout=900):
    """``nproc`` processes of a script (a path ending in .py) or of ``on_ranks`` in a test module (a module name, run
    by rank_worker.py, each rank printing its OK line) under torchrun with ``args`` after it, on a rendezvous port it
    picks itself; returns the standard output"""
    module = not script_or_module.endswith(".py")
    script = os.path.join(HERE, "rank_worker.py") if module else script_or_module
    argv = ([script_or_module] if module else []) + list(args)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc-per-node={nproc}",
                        script, *argv], capture_output=True, text=True, timeout=timeout,
                       env=None if env is None else dict(os.environ, **env))
    assert r.returncode == 0, (r.stdout[-4000:] + r.stderr[-8000:])
    if module:
        assert r.stdout.count(f"RANK_WORKER_OK {script_or_module} ") == nproc, r.stdout[-4000:]
    return r.stdout
