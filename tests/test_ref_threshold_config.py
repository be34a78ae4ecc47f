"""pcdn_config.ref_min_bytes (delivery by reference above a size threshold): what pcdn_create refuses, on
host-only engines (device = -1), so it runs without a GPU.  The deliveries themselves are checked in
test_gpu_ref_threshold.py."""
import ctypes as C

import pytest

from gpu_world import PCDN_EINVAL

BASE = dict(device=-1, max_conns=1024, max_keys=1024)


def refused(pcdn, **kw):
    with pytest.raises(pcdn.PcdnError) as ei:
        pcdn.Engine(**BASE, **kw)
    assert ei.value.code == PCDN_EINVAL
    return str(ei.value)


def test_refused_thresholds(pcdn):
    assert "ref_min_bytes" in refused(pcdn, ref_min_bytes=2048, flags=pcdn.FLAG_SHARED_PAYLOAD)
    assert "ref_min_bytes" in refused(pcdn, ref_min_bytes=0x20000000, ring_bytes_per_conn=1 << 31)
    # the largest copied record, round_up(4 + T - 1, 32), must fit an empty ring / the pool
    assert "ring_bytes_per_conn" in refused(pcdn, ref_min_bytes=4094, ring_bytes_per_conn=4096)    # 4128 > 4096
    assert "pool_bytes" in refused(pcdn, ref_min_bytes=8190, flags=pcdn.FLAG_OUTPUT_POOL, pool_bytes=8192)
    # (the pool's default size is max_conns x ring_bytes_per_conn)
    assert "pool_bytes" in refused(pcdn, ref_min_bytes=1024 * 4096, flags=pcdn.FLAG_OUTPUT_POOL, ring_bytes_per_conn=4096)


@pytest.mark.parametrize("kw", [dict(ring_bytes_per_conn=4096, ref_min_bytes=4093),
                                dict(flags=16, pool_bytes=8192, ref_min_bytes=8189),
                                dict(flags=16, ring_bytes_per_conn=4096, ref_min_bytes=1024 * 4096 - 3),
                                dict(ring_bytes_per_conn=4096, ref_min_bytes=1),
                                dict(ref_min_bytes=0x1FFFFFFF, ring_bytes_per_conn=1 << 31),
                                dict(flags=32, ref_min_bytes=0)],
                         ids=["ring-edge", "pool-edge", "default-pool-edge", "one", "max", "shared-zero"])
def test_admitted_thresholds(pcdn, kw):
    pcdn.Engine(**BASE, **kw).close()


def test_old_config_size(pcdn):
    """a config of the size before ref_min_bytes is accepted (the field reads as 0); any other size is not"""
    old = pcdn.Config.ref_min_bytes.offset
    pcdn.Engine(**BASE, struct_size=old).close()
    # the bytes behind the old size are never read: a threshold there does not meet the shared-payload check
    pcdn.Engine(**BASE, struct_size=old, flags=pcdn.FLAG_SHARED_PAYLOAD, ref_min_bytes=2048).close()
    for size in (old - 8, old + 4, C.sizeof(pcdn.Config) + 8):
        refused(pcdn, struct_size=size)

