"""The predict product's paired schedule (predict_streamk.cuh: psk_pair_units, psk_pair_first, psk_pair_next,
psk_pair_cta_steps), checked on the CPU.

A host program compiled from the product's own header walks every CTA's tile sequence the way the kernel's iterator does
(from the long tile of unit c, psk_pair_next after each whole tile, psk_pair_cta_steps k-steps in all) and prints it.  The
test checks that the CTAs together visit every (output, tile, k-step) of the lower-mode list exactly once, that a unit is a
long tile followed by its short partner with 16 (ntb + 1) steps (8 fewer with the half tile of an odd Npad / 128, the middle
tile of an odd ntb alone), that the per-CTA step counts differ by at most one unit, and that the schedule is selected for the
benchmark's workloads as intended: C5 on one H100 (132 SMs) pairs, on 128 CTAs of two units each (psk_pair_grid), C2, C3
and C5 sharded over 2, 4 or 8 GPUs stay on stream-K, and so does a shape whose units would fill two rounds half."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'gp-mpc_b200', 'csrc')
BN, BK, SB = 256, 16, 16
SMS = 132                                  # H100 SXM: the automatic grid is one CTA per SM
# (Npad, nloc, grid): C5 at 132 and 128 CTAs, the half tile (8320 = 65 x 128) and an odd tile count (8448 = 33 x 256),
# each with 136 units on 68 CTAs, and uneven unit counts (85 units on 43 CTAs, 153 on 153)
CASES = ((16384, 8, 132), (16384, 8, 128), (8320, 8, 68), (8448, 8, 68), (8320, 5, 43), (8448, 9, 153))

PROG = r'''
#include <cstdio>
#include <cstdlib>
#include "predict_streamk.cuh"
int main(int argc, char** argv)
{
    if (argv[1][0] == 'S') {              // S nloc ntb grid: the selection and the paired schedule's automatic grid
        const int nloc = atoi(argv[2]), upo = psk_pair_units(nloc, atoi(argv[3]), atoi(argv[4]));
        printf("%d %d\n", upo, upo ? psk_pair_grid((long long)nloc * upo, atoi(argv[4])) : 0);
        return 0;
    }
    const int np = atoi(argv[1]), nloc = atoi(argv[2]), C = atoi(argv[3]);
    const int ntb = (np + PSK_BN - 1) / PSK_BN, nk = np / GEMM_BK, upo = psk_pair_units(nloc, ntb, C);
    printf("N %d %d %d\n", ntb, nk, upo);
    for (int p = 0; p < (ntb + 1) / 2; ++p) printf("U %d %d\n", p, psk_unit_steps(ntb, nk, p));
    for (int c = 0; c < C; ++c) {
        const long long n = psk_pair_cta_steps(nloc, ntb, nk, upo, c, C);
        printf("C %d %lld", c, n);
        int a, jt;
        psk_pair_first(ntb, upo, c, a, jt);
        for (long long i = 0; i < n; ) {
            const int ks = psk_ksteps(ntb, nk, 0, jt);
            printf(" %d:%d:%d", a, jt, ks);
            i += ks;
            psk_pair_next(ntb, upo, C, a, jt);
        }
        printf("\n");
    }
    return 0;
}
'''


@pytest.fixture(scope='module')
def exe(tmp_path_factory):
    nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    if not os.path.exists(nvcc):
        pytest.skip('nvcc not found')
    d = tmp_path_factory.mktemp('pairs')
    src, out = d / 'pairs.cu', d / 'pairs'
    src.write_text(PROG)
    subprocess.check_call([nvcc, '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a', '-I', CSRC, str(src),
                           '-o', str(out), '-ldl'])
    return str(out)


def walk(exe, npad, nloc, grid):
    out = subprocess.check_output([exe, str(npad), str(nloc), str(grid)], text=True)
    res = dict(units={}, ctas={})
    for line in out.splitlines():
        f = line.split()
        if f[0] == 'N':
            res['ntb'], res['nk'], res['upo'] = map(int, f[1:])
        elif f[0] == 'U':
            res['units'][int(f[1])] = int(f[2])
        else:
            res['ctas'][int(f[1])] = (int(f[2]), [tuple(map(int, x.split(':'))) for x in f[3:]])
    return res


def ksteps(npad, jt):                      # lower mode: tile jt covers k < min(256 (jt + 1), Npad)
    return min(BN * (jt + 1), npad) // BK


@pytest.mark.parametrize('npad,nloc,grid', CASES)
def test_every_k_step_is_visited_once(exe, npad, nloc, grid):
    r = walk(exe, npad, nloc, grid)
    ntb = -(-npad // BN)
    assert (r['ntb'], r['nk'], r['upo']) == (ntb, npad // BK, (ntb + 1) // 2)
    seen = []
    for c, (n, tiles) in r['ctas'].items():
        assert n == sum(ks for _, _, ks in tiles), c             # a CTA's steps are whole tiles: none is cut
        for a, jt, ks in tiles:
            assert ks == ksteps(npad, jt)
            seen += [(a, jt, s) for s in range(ks)]
    want = [(a, jt, s) for a in range(nloc) for jt in range(ntb) for s in range(ksteps(npad, jt))]
    assert len(seen) == len(want) and set(seen) == set(want)


@pytest.mark.parametrize('npad,nloc,grid', CASES)
def test_units_pair_long_with_short_and_are_dealt_round_robin(exe, npad, nloc, grid):
    r = walk(exe, npad, nloc, grid)
    ntb, upo = r['ntb'], r['upo']
    half = 8 if (npad // 128) % 2 else 0
    for p, steps in r['units'].items():
        if p == ntb - 1 - p:                                     # the middle tile of an odd ntb is a unit alone
            assert steps == ksteps(npad, p)
        else:
            assert steps == SB * (ntb + 1) - (half if p == 0 else 0)
    for c, (n, tiles) in r['ctas'].items():
        units = list(range(c, nloc * upo, grid))
        want = []
        for u in units:                                          # unit u = a upo + p: long tile ntb-1-p, then p
            a, p = divmod(u, upo)
            want += [(a, ntb - 1 - p)] + ([(a, p)] if p != ntb - 1 - p else [])
        assert [(a, jt) for a, jt, _ in tiles] == want, c
        assert n == sum(r['units'][u % upo] for u in units)
    # the CTAs' unit counts differ by at most one, so their step counts by at most one unit plus the units' own spread
    # (the half-tile pair and the middle tile of an odd ntb are shorter)
    nunits = [len(range(c, nloc * upo, grid)) for c in range(grid)]
    assert min(nunits) >= 1 and max(nunits) - min(nunits) <= 1
    counts = [n for n, _ in r['ctas'].values()]
    lo, hi = min(r['units'].values()), max(r['units'].values())
    assert max(counts) - min(counts) <= hi + (hi - lo)
    if lo == hi:
        assert max(counts) - min(counts) in (0, hi)


def test_c5_at_128_ctas_is_two_units_each(exe):
    r = walk(exe, 16384, 8, 128)
    assert {n for n, _ in r['ctas'].values()} == {2 * SB * 65}


def auto_grid(npad, nloc):                 # gpmpc.cu psk_grid: one CTA per SM, at least 4 k-steps each
    ntb = -(-npad // BN)
    G = nloc * sum(ksteps(npad, jt) for jt in range(ntb))
    return min(SMS, max(1, G // 4))


@pytest.mark.parametrize('name,N,Ny,ranks,paired', [
    ('c5', 16384, 8, 1, True), ('c5', 16384, 8, 2, False), ('c5', 16384, 8, 4, False), ('c5', 16384, 8, 8, False),
    ('c3', 4096, 6, 1, False), ('c2', 1000, 6, 1, False), ('136 units', 8320, 8, 1, False)])
def test_selection_by_shape(exe, name, N, Ny, ranks, paired):
    npad = -(-N // 128) * 128
    nloc, ntb = Ny // ranks, -(-npad // BN)
    grid = auto_grid(npad, nloc)
    upo, pgrid = map(int, subprocess.check_output([exe, 'S', str(nloc), str(ntb), str(grid)], text=True).split())
    assert upo == ((ntb + 1) // 2 if paired else 0), (name, ranks, nloc, ntb, grid)
    if paired:                             # C5: 256 units on 128 CTAs of 2 each instead of 132 of 2 or 1
        assert (grid, pgrid) == (132, 128)


@pytest.mark.parametrize('units,grid', [(256, 132), (264, 132), (132, 132), (136, 68), (1000, 7), (136, 132), (265, 132),
                                        (153, 150), (100, 132)])
def test_paired_grid_keeps_the_rounds_and_evens_the_units(exe, units, grid):
    nloc, ntb = units, 2                   # one unit per output
    upo, pgrid = map(int, subprocess.check_output([exe, 'S', str(nloc), str(ntb), str(grid)], text=True).split())
    rounds = -(-units // grid)
    # paired when every CTA owns a unit and the rounds fill 7/8 of the grid's unit slots
    assert upo == (1 if units >= grid and units >= 0.875 * rounds * grid else 0), (units, grid)
    if upo:
        assert pgrid <= grid and -(-units // pgrid) == rounds and -(-units // (pgrid - 1)) > rounds
        per = [len(range(c, units, pgrid)) for c in range(pgrid)]
        assert min(per) >= rounds - 1 and max(per) == rounds
