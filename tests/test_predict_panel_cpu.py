"""The L^-1 panel's layout (predict_streamk.cuh: psk_panel_chunk, panel_pack_kernel), restated on the CPU.

A host program compiled from the product's own header prints psk_kstart, psk_ksteps and psk_panel_chunk for a set of
Npad; the test restates them from the definition of the lower-mode k-step list (tile jt covers k < min(256 (jt + 1),
Npad)) and of the stage layout the product's warps read (128-byte rows, 16-byte chunk c of row r at c ^ (r & 7), the
fragment loads' k-permutation).  It checks that block g = a T + psk_kstart(jt) + s enumerates the list in order, so a
CTA's range of the list is one contiguous stretch of the panel, and that every element lands where the consumer
expects the column it multiplies."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'gp-mpc_b200', 'csrc')
BN, BK = 256, 16
BLOCK = BN * BK                      # doubles per k-step block
NPADS = (128, 256, 384, 512, 1152, 4096, 16384)

PROG = r'''
#include <cstdio>
#include <cstdlib>
#include "predict_streamk.cuh"
int main(int argc, char** argv)
{
    for (int i = 1; i < argc; ++i) {
        const int np = atoi(argv[i]), ntb = (np + PSK_BN - 1) / PSK_BN, nk = np / GEMM_BK;
        printf("N %d %d %d %lld\n", np, ntb, nk, psk_steps_per_output(ntb, nk, 0));
        for (int jt = 0; jt < ntb; ++jt) {
            printf("T %d %lld %d\n", jt, psk_kstart(ntb, nk, 0, jt), psk_ksteps(ntb, nk, 0, jt));
            const int ks = psk_ksteps(ntb, nk, 0, jt);
            for (int s : {0, ks / 2, ks - 1}) {
                printf("C %d %d", jt, s);
                for (int r = 0; r < PSK_BN; ++r)
                    for (int c = 0; c < 8; ++c) printf(" %lld", psk_panel_chunk(ntb, nk, jt, s, r, c));
                printf("\n");
            }
        }
    }
    return 0;
}
'''


@pytest.fixture(scope='module')
def printed(tmp_path_factory):
    nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    if not os.path.exists(nvcc):
        pytest.skip('nvcc not found')
    d = tmp_path_factory.mktemp('panel')
    src, exe = d / 'panel_layout.cu', d / 'panel_layout'
    src.write_text(PROG)
    subprocess.check_call([nvcc, '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a', '-I', CSRC, str(src),
                           '-o', str(exe), '-ldl'])
    out = subprocess.check_output([str(exe)] + [str(n) for n in NPADS], text=True)
    res, cur = {}, None
    for line in out.splitlines():
        f = line.split()
        if f[0] == 'N':
            cur = res.setdefault(int(f[1]), dict(ntb=int(f[2]), nk=int(f[3]), T=int(f[4]), tiles={}, chunks={}))
        elif f[0] == 'T':
            cur['tiles'][int(f[1])] = (int(f[2]), int(f[3]))
        else:
            cur['chunks'][(int(f[1]), int(f[2]))] = np.array(f[3:], dtype=np.int64).reshape(BN, 8)
    return res


@pytest.mark.parametrize('npad', NPADS)
def test_block_index_enumerates_the_lower_k_step_list(printed, npad):
    p = printed[npad]
    ntb, nk = -(-npad // BN), npad // BK
    assert (p['ntb'], p['nk']) == (ntb, nk)
    steps = [min(BN * (jt + 1), npad) // BK for jt in range(ntb)]      # tile jt: k < min(256 (jt + 1), Npad)
    start = np.concatenate([[0], np.cumsum(steps)])
    assert p['T'] == start[-1]
    for jt in range(ntb):
        assert p['tiles'][jt] == (start[jt], steps[jt]), jt
    # g = a T + kstart(jt) + s walks the list (a, jt, s) in order with no gap: a CTA's range is one stretch
    nloc = 3
    g = [a * p['T'] + p['tiles'][jt][0] + s for a in range(nloc) for jt in range(ntb) for s in range(p['tiles'][jt][1])]
    assert g == list(range(nloc * p['T']))


@pytest.mark.parametrize('npad', NPADS)
def test_chunks_sit_where_the_consumer_reads_them(printed, npad):
    p = printed[npad]
    r = np.arange(BN)[:, None]
    c = np.arange(8)[None, :]
    for (jt, s), off in p['chunks'].items():
        base = (p['tiles'][jt][0] + s) * BLOCK
        assert np.array_equal(off, base + r * BK + 2 * (c ^ (r & 7))), (jt, s)
        assert sorted((off - base).ravel().tolist()) == list(range(0, BLOCK, 2))     # one 32 KB block, no overlap
    # the warps' fragment loads: lane (g, t) reads slot j of L-row r (r & 7 == g) at ((j + 4 (t >> 1)) ^ g) << 1 | (t & 1)
    # of the row and multiplies it as column k = 2 j + (t & 1) + 8 (t >> 1); the pack stores column 2 c + e of row r at
    # chunk position c ^ (r & 7), half e
    for row in range(BN):
        g = row & 7
        for t in range(4):
            for j in range(4):
                pos = (((j + 4 * (t >> 1)) ^ g) << 1) + (t & 1)
                k = 2 * j + (t & 1) + 8 * (t >> 1)
                assert pos == 2 * ((k >> 1) ^ (row & 7)) + (k & 1)
