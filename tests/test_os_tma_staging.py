"""The 16384-point Float32 overlap-save kernels load an interior block's input in one of two ways: TMA bulk copies into
shared memory (16-byte aligned input whose copy, rounded up to 16 bytes, stays inside the signal) or predicated global
loads in the first pass (any other block).  Both must feed the same values into the same butterflies, so the outputs are
bit-equal whichever way the blocks were loaded.

The signals are long enough that every CTA of the persistent grid (one per SM) runs several units in turn, so the
copies issued during one unit for the next (the head-region copy after the first pass, the copy in the last pass, the
mbarrier phase flip) and CTAs that mix staged and directly loaded units are all exercised."""
import numpy as np
import pytest

from conftest import relerr

pytestmark = pytest.mark.gpu

dsp = pytest.importorskip("dspb200")
from oracle import dspbase as od          # noqa: E402

RNG = np.random.default_rng(4097)
N = 16384
SMS_H100 = 132                            # H100 SXM: one resident CTA of this kernel per SM


def _conv_dev(plan, u, offset):
    """conv(u, v) through the device-pointer entry, with u stored `offset` samples into a 16-byte aligned buffer."""
    from dspb200 import device
    nu = u.size
    nout = nu + plan.nv - 1
    buf = device.DeviceArray((nu + offset,), u.dtype)
    assert buf.ptr % 16 == 0
    du = buf[offset:offset + nu].copy_from_host(u)
    out = device.DeviceArray((nout,), u.dtype)
    plan.exec_dev(du.ptr, nu, 1, out.ptr, nout, 0)
    device.sync()
    return out.to_host()


def _units(nu, nv, cplx):
    """Per unit of a one-column conv: (first sample index i0, interior, stored samples from i0 on) -- the kernel's
    geometry with out_begin = u_begin = 0 and out_count = nu + nv - 1."""
    L = N - nv + 1
    span = N if cplx else N + L
    nout = nu + nv - 1
    nblk = -(-nout // L)
    upc = nblk if cplx else (nblk + 1) // 2
    res = []
    for u in range(upc):
        i0 = (u if cplx else 2 * u) * L - (nv - 1)
        interior = i0 >= 0 and nu - i0 >= span and nout - i0 >= span
        res.append((i0, interior, nu - i0))
    return res, span


def _check(dt, nu, nv, staged_offset, direct_offset):
    cplx = np.dtype(dt).kind == "c"
    if cplx:
        u = (RNG.standard_normal(nu) + 1j * RNG.standard_normal(nu)).astype(dt)
        v = (RNG.standard_normal(nv) + 1j * RNG.standard_normal(nv)).astype(dt)
    else:
        u = RNG.standard_normal(nu).astype(dt)
        v = RNG.standard_normal(nv).astype(dt)
    plan = _lib_plan(v)
    try:
        staged = _conv_dev(plan, u, staged_offset)
        direct = _conv_dev(plan, u, direct_offset)
    finally:
        plan.close()
    assert np.array_equal(staged, direct), dt
    assert relerr(staged, od.conv(u, v, f64=True)) < 1e-6


def _lib_plan(v):
    from dspb200 import _lib
    plan = _lib.OsPlan(v, N)
    assert plan.nfft == N and plan.fused
    return plan


@pytest.mark.parametrize("dt,nu", [(np.complex64, 1 << 23), (np.float32, 1 << 24)])
def test_os_16384_tma_staged_equals_direct_loads(dt, nu):
    # nv = 4097: slot 0 of every unit sits (nv - 1) * itemsize = 16 KB (complex: 32 KB) before a multiple of 2 L samples,
    # so at offset 0 every interior unit is 16-byte aligned and staged, at offset 1 (8 or 4 bytes) none is: every unit
    # takes the direct loads
    nv = 4097
    units, span = _units(nu, nv, np.dtype(dt).kind == "c")
    assert len(units) >= 4 * SMS_H100                # several units per CTA
    itemsize = np.dtype(dt).itemsize
    assert all(i0 * itemsize % 16 == 0 for i0, interior, _ in units if interior)
    assert span * itemsize % 16 == 0
    _check(dt, nu, nv, 0, 1)


def test_os_16384_tma_round_up_past_the_signal_falls_back():
    # Real signal, nv = 4095: L = 12290 is even and nv - 1 = 4094 = 2 (mod 4), so slot 0 of every unit is 2 floats past a
    # 16-byte boundary -- at offset 2 every interior unit is aligned, at offset 1 none is.  The span, 2 N - nv + 1 = 28674
    # floats, is no multiple of 4: the copy is rounded up to 28676 floats.  With nu = 24580 K the unit K - 1 is interior and
    # aligned but ends exactly at the last stored sample (jhi == span), so its rounded-up copy would read past the signal;
    # it must take the direct loads while its neighbours are staged.
    nv, K = 4095, 683
    nu = 24580 * K
    units, span = _units(nu, nv, False)
    rounded = -(-span // 4) * 4
    assert span % 4 != 0
    assert len(units) >= 4 * SMS_H100
    edge = [k for k, (i0, interior, jhi) in enumerate(units) if interior and (i0 + 2) % 4 == 0 and span <= jhi < rounded]
    assert edge == [K - 1] and K - 1 >= SMS_H100      # reached as some CTA's next unit, not as its first
    assert all((i0 + 2) % 4 == 0 for i0, interior, _ in units if interior)
    _check(np.float32, nu, nv, 2, 1)
