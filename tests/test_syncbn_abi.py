"""CPU: the synchronised BatchNorm entry points (ffb6d_bn_sync_moments / _fwd / _bwd_sums / _bwd) check their
arguments before any launch -- sizes, W, null and misaligned pointers, short workspaces -- and report them through
ffb6d_last_error; and a layer of ffb6d_b200.modules picks the synchronised path exactly when nn.SyncBatchNorm would:
a converted BatchNorm, training mode, an initialised process group of more than one rank."""
import ctypes as C

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from ffb6d_b200 import _lib, modules as M
from conftest import ROOT

BIG = 1 << 40                                   # a byte count that passes every workspace check


@pytest.fixture
def buf():
    b = (C.c_int64 * 64)()
    return (C.addressof(b) + 15) & ~15, b       # 16-byte aligned address (the array keeps it alive)


BAD_SIZES = (dict(B=0), dict(C_=0), dict(P=0), dict(B=-1), dict(B=65536), dict(C_=65536), dict(P=1 << 31),
             dict(B=40000, C_=60000))


def test_bn_sync_moments_rejects_bad_arguments(buf):
    lib = _lib.lib
    p, _keep = buf

    def call(z=p, B=2, C_=3, P=5, mom=p, ws=p, nbytes=BIG):
        return lib.ffb6d_bn_sync_moments(z, B, C_, P, mom, ws, nbytes, None)

    for size in BAD_SIZES:
        assert call(**size) == _lib.ERR_INVALID, size
        assert "bn_sync_moments: bad size" in _lib.last_error()
    for ptr in ("z", "mom", "ws"):
        assert call(**{ptr: None}) == _lib.ERR_INVALID, ptr
        assert "bn_sync_moments: null pointer" in _lib.last_error()
    assert call(mom=p + 4) == _lib.ERR_INVALID
    assert "8-byte aligned" in _lib.last_error()
    assert call(nbytes=lib.ffb6d_bn_workspace_bytes(3, 5) - 1) == _lib.ERR_INVALID
    assert "bn_sync_moments: workspace too small" in _lib.last_error()


def test_bn_sync_fwd_rejects_bad_arguments(buf):
    lib = _lib.lib
    p, _keep = buf

    def call(z=p, B=2, C_=3, P=5, rows=p, W=2, gamma=p, beta=p, rm=p, rv=p, act=1, stats=p, count=p, y=p):
        return lib.ffb6d_bn_sync_fwd(z, B, C_, P, rows, W, gamma, beta, 1e-5, 0.1, rm, rv, act, 0.0, stats, count, y, None)

    for size in BAD_SIZES:
        assert call(**size) == _lib.ERR_INVALID, size
        assert "bn_sync_fwd: bad size" in _lib.last_error()
    for w in (0, -1, 65537):
        assert call(W=w) == _lib.ERR_INVALID, w
        assert "bn_sync_fwd: W=%d" % w in _lib.last_error()
    for ptr in ("z", "rows", "stats", "count", "y"):
        assert call(**{ptr: None}) == _lib.ERR_INVALID, ptr
        assert "bn_sync_fwd: null pointer" in _lib.last_error()
    for a in (-1, 3):
        assert call(act=a) == _lib.ERR_INVALID
        assert "act=%d" % a in _lib.last_error()
    assert call(stats=p + 8) == _lib.ERR_INVALID
    assert "stats must be 16-byte aligned" in _lib.last_error()
    for ptr in ("rows", "count"):
        assert call(**{ptr: p + 4}) == _lib.ERR_INVALID, ptr
        assert "8-byte aligned" in _lib.last_error()


def test_bn_sync_bwd_sums_rejects_bad_arguments(buf):
    lib = _lib.lib
    p, _keep = buf

    def call(z=p, g=p, stats=p, B=2, C_=3, P=5, act=2, sums=p, gg=p, gb=p, ws=p, nbytes=BIG):
        return lib.ffb6d_bn_sync_bwd_sums(z, g, stats, B, C_, P, act, 0.2, sums, gg, gb, ws, nbytes, None)

    for size in BAD_SIZES:
        assert call(**size) == _lib.ERR_INVALID, size
        assert "bn_sync_bwd_sums: bad size" in _lib.last_error()
    for ptr in ("z", "g", "stats", "sums", "ws"):
        assert call(**{ptr: None}) == _lib.ERR_INVALID, ptr
        assert "bn_sync_bwd_sums: null pointer" in _lib.last_error()
    assert call(act=3) == _lib.ERR_INVALID
    assert "act=3" in _lib.last_error()
    assert call(stats=p + 4) == _lib.ERR_INVALID
    assert "stats must be 16-byte aligned" in _lib.last_error()
    assert call(sums=p + 4) == _lib.ERR_INVALID
    assert "8-byte aligned" in _lib.last_error()
    assert call(nbytes=lib.ffb6d_bn_workspace_bytes(3, 5) - 1) == _lib.ERR_INVALID
    assert "bn_sync_bwd_sums: workspace too small" in _lib.last_error()


def test_bn_sync_bwd_rejects_bad_arguments(buf):
    lib = _lib.lib
    p, _keep = buf

    def call(z=p, g=p, stats=p, B=2, C_=3, P=5, rows=p, W=3, count=p, act=0, dz=p, ws=p, nbytes=BIG):
        return lib.ffb6d_bn_sync_bwd(z, g, stats, B, C_, P, rows, W, count, act, 0.0, dz, ws, nbytes, None)

    for size in BAD_SIZES:
        assert call(**size) == _lib.ERR_INVALID, size
        assert "bn_sync_bwd: bad size" in _lib.last_error()
    for w in (0, -3, 1 << 20):
        assert call(W=w) == _lib.ERR_INVALID, w
        assert "bn_sync_bwd: W=%d" % w in _lib.last_error()
    for ptr in ("z", "g", "stats", "rows", "count", "dz", "ws"):
        assert call(**{ptr: None}) == _lib.ERR_INVALID, ptr
        assert "bn_sync_bwd: null pointer" in _lib.last_error()
    assert call(act=-1) == _lib.ERR_INVALID
    assert "act=-1" in _lib.last_error()
    assert call(stats=p + 8) == _lib.ERR_INVALID
    assert "stats must be 16-byte aligned" in _lib.last_error()
    for ptr in ("rows", "count"):
        assert call(**{ptr: p + 4}) == _lib.ERR_INVALID, ptr
        assert "8-byte aligned" in _lib.last_error()
    assert call(nbytes=lib.ffb6d_bn_workspace_bytes(3, 5) - 1) == _lib.ERR_INVALID
    assert "bn_sync_bwd: workspace too small" in _lib.last_error()


def _layers():
    """One layer of each flavour with BatchNorm, and one converted copy of each."""
    def make():
        return [M.Conv2d(8, 4, bn=True), M.RandLAConv2d(8, 4, bn=True), M.Conv1d(8, 4, bn=True),
                M.RandLAConv1d(8, 4, bn=True)]
    return make(), [nn.SyncBatchNorm.convert_sync_batchnorm(m) for m in make()]


def test_conversion_keeps_state_dict_keys():
    plain, conv = _layers()
    for a, b in zip(plain, conv):
        assert isinstance(b._bn, nn.SyncBatchNorm) and not isinstance(a._bn, nn.SyncBatchNorm)
        assert list(a.state_dict()) == list(b.state_dict())
        b.load_state_dict(a.state_dict())


def test_no_process_group_never_syncs():
    assert not dist.is_initialized()
    plain, conv = _layers()
    for m in plain + conv:
        m.train()
        assert m._bn_sync() is None
        m.eval()
        assert m._bn_sync() is None


def test_one_value_per_channel_is_rejected_only_without_sync():
    m = nn.SyncBatchNorm.convert_sync_batchnorm(M.Conv2d(8, 4, bn=True)).train()
    with pytest.raises(ValueError, match="Expected more than 1 value per channel"):
        m._train_momentum(torch.zeros(1, 8, 1, 1))
    n0 = int(m._bn.num_batches_tracked)
    assert m._train_momentum(torch.zeros(1, 8, 1, 1), sync=(None, 2)) == pytest.approx(0.1)   # a synchronised group
    assert int(m._bn.num_batches_tracked) == n0 + 1


def _selection_worker(rank, world, init_file, q):
    import sys
    sys.path.insert(0, ROOT)
    import torch.distributed as dist_
    import torch.nn as nn_
    from ffb6d_b200 import modules as M_
    try:
        dist_.init_process_group("gloo", init_method="file://" + init_file, rank=rank, world_size=world)
        plain = M_.Conv2d(8, 4, bn=True).train()
        conv = nn_.SyncBatchNorm.convert_sync_batchnorm(M_.Conv1d(8, 4, bn=True)).train()
        solos = [dist_.new_group([r]) for r in range(world)] if world > 1 else None    # every rank creates every group
        solo = solos[rank] if solos else None
        own = nn_.SyncBatchNorm.convert_sync_batchnorm(M_.RandLAConv2d(8, 4, bn=True), process_group=solo).train()
        got = {"plain": plain._bn_sync(), "conv": conv._bn_sync(), "own": own._bn_sync() if solo is not None else None}
        got = {k: (v[1] if v is not None else None) for k, v in got.items()}
        got["conv_is_world"] = conv._bn_sync() is not None and conv._bn_sync()[0] is dist_.group.WORLD
        conv.eval()
        got["eval"] = conv._bn_sync()
        dist_.barrier()
        dist_.destroy_process_group()
        q.put((rank, got))
    except BaseException as e:       # reported by the parent
        q.put((rank, repr(e)))


def _run_selection(world, tmp_path):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    init_file = str(tmp_path / "pg_init")
    procs = [ctx.Process(target=_selection_worker, args=(r, world, init_file, q)) for r in range(world)]
    try:
        for p in procs:
            p.start()
        res = dict(q.get(timeout=120) for _ in procs)
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()
    return [res[r] for r in range(world)]


def test_gloo_world_of_one_selects_the_local_path(tmp_path):
    (got,) = _run_selection(1, tmp_path)
    assert got == {"plain": None, "conv": None, "own": None, "conv_is_world": False, "eval": None}, got


def test_gloo_world_of_two_syncs_converted_training_layers_only(tmp_path):
    for got in _run_selection(2, tmp_path):
        # plain BN never syncs; a converted one syncs over WORLD (2 ranks); one scoped to a one-rank group does not
        assert got == {"plain": None, "conv": 2, "own": None, "conv_is_world": True, "eval": None}, got
