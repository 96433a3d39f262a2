"""evab_rotate_wsum weights the q rows of the rotations' key-switch accumulators where they are computed (k_rot_wsum_ip): they are
never stored, so the workspace holds only the P rows, their inverse transforms and the two weighted halves A and D of every sum, and
P * c0 is formed from c0 itself instead of the diagonal of the extended digits."""
import pytest

import parity_cases as pc
from test_rotation_wsum import WsumEmuBackend, case_rotation_wsum


@pytest.mark.parametrize("ell,n,nout", [(1, 1, 1), (2, 8, 2), (3, 16, 4), (3, 7, 2)])
def test_rotation_wsum_work_bytes(ell, n, nout):
    N = 1024
    orc = pc.get_oracle(N, [60, 60, 60, 60])
    be = WsumEmuBackend(N, orc.primes)
    prow_and_tmp = 2 * n * 2 * N       # [n][2][N] each
    a_and_d = 2 * nout * 2 * ell * N   # [nout][2][ell][N] each
    assert be.lib.emu_rotate_wsum_work_bytes(be.h, ell, n, nout) == 8 * (prow_and_tmp + a_and_d)


def test_rotation_wsum_needs_no_scaled_c0():
    """the same bits as the oracle with the diagonal of the extended digits left empty (no evab_rotate_modup_scale_c0 call)"""
    orc = pc.get_oracle(1024, [60, 40, 40, 60])
    be = WsumEmuBackend(1024, orc.primes)
    be.lib.emu_rotate_modup_scale_c0 = lambda *args: 0
    case_rotation_wsum(be, orc, 2, 8, 2, seed=3)
