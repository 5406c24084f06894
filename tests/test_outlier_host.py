"""Outlier removal without a GPU: the float64 oracle (tests/outlier_oracle.py) against scipy's kd-tree and a plain-Python
restatement of Open3D's sequential statistics, hand-built edge cases, `eval.remove_outliers`' call layout with fakes,
the command lines' flags and usage errors, and the compiler's report on outlier.cu."""
import math
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import outlier_oracle as O
from regtr_b200 import eval as E
from regtr_b200 import multiway as MW
from regtr_b200 import register as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REAL = os.path.join(ROOT, 'tests', 'golden', 'real')
FIXTURES = ['real_3dmatch_redkitchen_0_5', 'real_3dmatch_sun3d_home_38_41', 'real_3dmatch_sun3d_hotel3_8_15']


def open3d_sequential(xyz, k, std_ratio):
    """RemoveStatisticalOutliers as Open3D writes it, in plain Python: per point the sqrt of its kNN d2 summed with
    std::accumulate, then the cloud sums over every point in index order."""
    idx, d2 = O.knn(xyz, k, brute=True)
    avg = []
    for row in d2:
        s = 0.0
        for d in row:
            s += math.sqrt(d)
        avg.append(s / len(row) if len(row) else -1.0)
    valid = sum(1 for a in avg if a != -1.0)
    mean = 0.0
    for a in avg:
        mean = mean + a if a > 0 else mean
    mean /= valid
    sq = 0.0
    for a in avg:
        sq += (a - mean) * (a - mean) if a > 0 else 0.0
    sd = math.sqrt(sq / (valid - 1)) if valid > 1 else float('nan')
    thr = mean + std_ratio * sd
    return np.array(avg), (mean, sd, thr)


def test_knn_against_kdtree_on_tie_free_data():
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(5)
    xyz = rng.random((3000, 3)) * [2.0, 1.0, 0.5]
    for k in (1, 7, 20, 64):
        idx, d2 = O.knn(xyz, k)
        dist, want = cKDTree(xyz).query(xyz, k=k)
        assert np.array_equal(idx, np.asarray(want).reshape(idx.shape))
        assert np.allclose(np.sqrt(d2), np.asarray(dist).reshape(d2.shape), rtol=1e-12, atol=0)
        assert np.array_equal(idx[:, 0], np.arange(3000))                       # the point itself comes first


def test_knn_tree_path_equals_brute_force_with_ties():
    """Above 4096 points the oracle ranks kd-tree candidates; with duplicates and lattice ties it still equals the
    brute-force rule."""
    g = np.stack(np.meshgrid(np.arange(17), np.arange(17), np.arange(17), indexing='ij'), -1).reshape(-1, 3) * 0.01
    xyz = np.concatenate([g, g[::7]])                                           # exact duplicates
    assert xyz.shape[0] > 4096
    for k in (6, 27, 40):
        a = O.knn(xyz, k)
        b = O.knn(xyz, k, brute=True)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_radius_counts_against_kdtree():
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(6)
    xyz = rng.random((5000, 3))
    for r in (0.02, 0.05, 0.1):
        want = cKDTree(xyz).query_ball_point(xyz, r, return_length=True)
        assert np.array_equal(O.radius_counts(xyz, r), want)
        assert np.array_equal(O.radius_counts(xyz, r, brute=True), want)


def test_points_at_exactly_the_radius_are_excluded():
    xyz = np.array([[0.0, 0.0, 0.0], [0.5, 0.0, 0.0], [0.0, 0.25, 0.0], [10.0, 0.0, 0.0]])
    counts, keep = O.radius_outlier(xyz, 2, 0.5)
    assert counts.tolist() == [2, 1, 2, 1]                                      # 0 - 1 is exactly 0.5 apart
    assert keep.tolist() == [1, 0, 1, 0]


@pytest.mark.parametrize('name', FIXTURES)
def test_statistics_against_open3d_sequential(name):
    xyz = np.load(os.path.join(REAL, name + '_input.npz'))['src_xyz'].astype(np.float64)[::4]
    k, s = 20, 2.0
    avg, keep, st = O.statistical_outlier(xyz, k, s)
    want_avg, want_st = open3d_sequential(xyz, k, s)
    assert np.array_equal(avg, want_avg)                                        # the same sequential per-point sum
    for a, b in zip(st, want_st):
        assert abs(a - b) <= 1e-12 * abs(b)
    far = np.abs(avg - want_st[2]) > 1e-9 * want_st[2]
    assert np.array_equal(keep[far], ((want_avg > 0) & (want_avg < want_st[2]))[far])
    assert 0 < keep.sum() < xyz.shape[0]


def test_chunk_sum_is_the_documented_tree():
    rng = np.random.default_rng(7)
    for n in (0, 1, 255, 256, 257, 1000, 4097):
        v = rng.random(n)
        parts = []
        for a in range(0, n, 256):
            e = list(v[a:a + 256]) + [0.0] * (256 - len(v[a:a + 256]))
            h = 128
            while h >= 1:
                e = [e[i] + e[i + h] for i in range(h)]
                h //= 2
            parts.append(e[0])
        s = 0.0
        for p in parts:
            s += p
        assert O.chunk_sum(v) == s


def test_duplicates_and_identical_clouds():
    same = np.tile([[1.0, 2.0, 3.0]], (50, 1))
    avg, keep, st = O.statistical_outlier(same, 10, 2.0)
    assert (avg == 0).all() and keep.sum() == 0 and st[0] == 0.0                # all-identical: nothing kept
    rng = np.random.default_rng(8)
    pts = rng.random((200, 3))
    dup = np.concatenate([pts, np.tile(pts[:1], (4, 1))])                       # 5 copies of point 0
    avg, keep, _ = O.statistical_outlier(dup, 5, 2.0)
    assert avg[0] == 0.0 and (avg[200:] == 0).all() and keep[[0, 200, 201, 202, 203]].sum() == 0
    avg6, _, _ = O.statistical_outlier(dup, 6, 2.0)
    assert avg6[0] > 0.0                                                        # k above the copies: kept again


def test_small_clouds():
    one = np.array([[0.5, 0.5, 0.5]])
    avg, keep, st = O.statistical_outlier(one, 20, 2.0)
    assert avg.tolist() == [0.0] and keep.tolist() == [0] and math.isnan(st[2])
    avg, keep, st = O.statistical_outlier(np.zeros((0, 3)), 20, 2.0)
    assert avg.shape == (0,) and keep.shape == (0,) and math.isnan(st[0])
    rng = np.random.default_rng(9)
    few = rng.random((7, 3))
    avg, _, _ = O.statistical_outlier(few, 20, 2.0)                             # k > n: all 7 points
    want = [sum(math.sqrt(((p - q) ** 2).sum()) for q in few) for p in few]
    assert np.allclose(avg, np.array(want) / 7, rtol=1e-14)


def test_planar_cloud_and_far_clusters():
    g = np.stack(np.meshgrid(np.arange(40), np.arange(40), indexing='ij'), -1).reshape(-1, 2) * 0.01
    plane = np.concatenate([g, np.zeros((g.shape[0], 1))], 1)
    avg, keep, _ = O.statistical_outlier(plane, 9, 1.0)
    assert keep.sum() > 0 and avg.min() > 0
    rng = np.random.default_rng(10)
    a = rng.random((30, 3)) * 0.1
    b = rng.random((40, 3)) * 0.1 + 100.0
    both = np.concatenate([a, b])
    idx, d2 = O.knn(both, 35, brute=True)                                       # k above the first cluster's size
    assert set(idx[0, :30]) == set(range(30)) and (idx[0, 30:] >= 30).all()
    avg, keep, st = O.statistical_outlier(both, 35, 1.0)
    assert keep[:30].sum() == 0 and keep[30:].sum() == 40                       # the small cluster's means jump


def test_select_points_is_stable():
    xyz = np.arange(30.0).reshape(10, 3)
    keep = np.array([0, 1, 1, 0, 0, 1, 0, 0, 0, 1])
    out, col, idx = O.select_points(xyz, keep, xyz + 0.5)
    assert idx.tolist() == [1, 2, 5, 9] and np.array_equal(out, xyz[idx]) and np.array_equal(col, xyz[idx] + 0.5)


def test_outlier_scan_is_seeded():
    a, ma = O.outlier_scan(3, 20000)
    b, mb = O.outlier_scan(3, 20000)
    assert np.array_equal(a, b) and np.array_equal(ma, mb) and ma.sum() == 200


def test_remove_outliers_call_layout():
    """Statistical first, the radius filter on what it kept, colours alike, indices into the files' rows."""
    calls = []

    def fake(name, drop):
        def fn(clouds, a, b, colors=None):
            calls.append((name, a, b, [c.shape[0] for c in clouds], colors is not None))
            idx = [np.array([i for i in range(c.shape[0]) if i % drop]) for c in clouds]
            return ([c[i] for c, i in zip(clouds, idx)], None if colors is None else
                    [c[i] for c, i in zip(colors, idx)], idx)
        return fn
    clouds = [np.arange(30.0).reshape(10, 3), np.arange(18.0).reshape(6, 3)]
    cols = [c + 0.5 for c in clouds]
    out, oc, ix = E.remove_outliers(clouds, cols, (20, 2.0), (16, 0.05), fake('stat', 2), fake('rad', 3))
    assert calls == [('stat', 20, 2.0, [10, 6], True), ('rad', 16, 0.05, [5, 3], True)]
    assert ix[0].tolist() == [3, 5, 9] and ix[1].tolist() == [3, 5]
    assert np.array_equal(out[0], clouds[0][ix[0]]) and np.array_equal(oc[1], cols[1][ix[1]])
    calls.clear()
    out, oc, ix = E.remove_outliers(clouds, None, None, (4, 0.1), fake('stat', 2), fake('rad', 2))
    assert calls == [('rad', 4, 0.1, [10, 6], False)] and oc is None


REG = ['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth']


def test_flags_parse():
    opt = R.parse_args(REG + ['--remove_statistical_outlier', '20', '2.0', '--remove_radius_outlier', '16', '0.05'])
    assert opt.remove_statistical_outlier == (20, 2.0) and opt.remove_radius_outlier == (16, 0.05)
    opt = R.parse_args(['a.ply', 'b.ply', '--fpfh', '0.05', '--remove_radius_outlier', '3', '0.1'])
    assert opt.remove_statistical_outlier is None and opt.remove_radius_outlier == (3, 0.1)
    opt = R.parse_args(REG)
    assert opt.remove_statistical_outlier is None and opt.remove_radius_outlier is None
    ap = MW.parser()
    opt = ap.parse_args(['a.ply', 'b.ply', '--ckpt', 'x', '--out', 'o', '--remove_statistical_outlier', '8', '1.5'])
    E.check_outlier_arguments(ap, opt)
    assert opt.remove_statistical_outlier == (8, 1.5)


BAD = [(['--remove_statistical_outlier', '0', '2.0'], 'K must be in 1..64'),
       (['--remove_statistical_outlier', '65', '2.0'], 'K must be in 1..64'),
       (['--remove_statistical_outlier', '20', '0'], 'S finite and > 0'),
       (['--remove_statistical_outlier', '20', 'nan'], 'S finite and > 0'),
       (['--remove_statistical_outlier', '2.5', '2.0'], 'expected an integer K'),
       (['--remove_radius_outlier', '0', '0.05'], 'N must be >= 1'),
       (['--remove_radius_outlier', '16', '-0.05'], 'R finite and > 0'),
       (['--remove_radius_outlier', '16', 'inf'], 'R finite and > 0'),
       (['--remove_radius_outlier', 'x', '0.05'], 'expected an integer N')]


@pytest.mark.parametrize('extra,msg', BAD)
def test_usage_errors_before_the_checkpoint(extra, msg, capsys, tmp_path):
    """The checkpoint does not exist: the usage error comes first, on both command lines and the --fpfh path."""
    ckpt = str(tmp_path / 'none' / 'ckpt' / 'm.pth')
    runs = [lambda: R.main(['a.ply', 'b.ply', '--ckpt', ckpt] + extra),
            lambda: R.main(['a.ply', 'b.ply', '--fpfh', '0.05'] + extra),
            lambda: MW.main(['a.ply', 'b.ply', 'c.ply', '--ckpt', ckpt, '--out', str(tmp_path / 'o')] + extra)]
    for run in runs:
        with pytest.raises(SystemExit) as e:
            run()
        err = capsys.readouterr().err
        assert e.value.code == 2 and msg in err, err


def test_outlier_kernels_do_not_spill():
    """outlier.cu's kernels (the kNN walk, the radius counts, the statistics, the compaction and the shared scan): no
    spills and no stack frame."""
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    from regtr_b200 import build
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + build.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(build.CSRC, 'outlier.cu'),
                                                        '-o', os.path.join(tmp, 'outlier.o')],
                           capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    text = r.stdout + r.stderr
    entries = re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*Function properties for \w+\n\s*(\d+) "
                         r"bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n[^\n]*Used (\d+) "
                         r"registers", text)
    names = ('k_outlier_init', 'k_knn_avg', 'k_chunk_offsets', 'k_chunk_sum', 'k_cloud_stats', 'k_stat_keep',
             'k_radius_count', 'k_select_flags', 'k_select_scatter', 'k_scan_lookback')
    assert sorted(n for n in names if any(n in e[0] for e in entries)) == sorted(names), entries
    for name, frame, st, ld, regs in entries:
        assert (frame, st, ld) == ('0', '0', '0'), (name, frame, st, ld)
    assert set(re.findall(r'(\d+) bytes spill (?:stores|loads)', text)) == {'0'}
