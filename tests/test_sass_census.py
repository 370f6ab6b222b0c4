"""The built library is Hopper-native: its SASS holds warpgroup MMAs (HGMMA), bulk-TMA copies (UBLKCP), mbarrier ops (SYNCS),
cluster barriers (UCGABAR_*) and the programmatic-dependent-launch pair (PREEXIT / ACQBULK), and no warp-level mma.sync
fallback (HMMA).  Runs without a GPU (cuobjdump reads the cubin inside the .so)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'pyprob_b200', 'lib', 'libpyprob_b200.so')


@pytest.mark.skipif(shutil.which('cuobjdump') is None, reason='cuobjdump not on PATH')
@pytest.mark.skipif(not os.path.exists(LIB), reason='library not built')
def test_library_sass_is_wgmma_tma_and_pdl():
    sass = subprocess.run(['cuobjdump', '-sass', LIB], capture_output=True, text=True, timeout=600).stdout
    assert 'sm_90a' in sass or 'SM90A' in sass.upper()

    def count(mnemonic):
        return len(re.findall(r'[^A-Z]' + mnemonic + r'[. ]', sass))
    for m in ('HGMMA', 'UBLKCP', 'SYNCS', 'UCGABAR_ARV', 'UCGABAR_WAIT', 'PREEXIT', 'ACQBULK'):
        assert count(m) > 0, m
    assert count('HMMA') == 0
    # the persistent and the cluster GEMM kernels are in the build
    assert 'k_grouped_persistent' in sass and 'k_lstm_cluster' in sass and 'k_cluster' in sass
