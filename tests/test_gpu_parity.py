"""GPU parity tests (run on an H100): the CUDA product, called through the C ABI, against
(a) the golden fixtures produced by the unmodified reference and (b) the CPU oracle on the same
seeded inputs.  Integer / index results must be bit-exact; float tolerances are stated per test
(SURVEY.md 8c: features <= 1e-4 * max|ref|, correspondences <= 1e-5 m ... pose <= 1e-4)."""
import numpy as np
import pytest
import torch

from conftest import (FORWARD_CASES, REAL_CASES, VARIANT_CASES, check_forward_against_golden,
                      check_real_forward_against_golden, load_golden, make_case, make_real_case)

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'


def G(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return t.to(DEV) if dtype is None else t.to(DEV, dtype)


def N(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope='module', autouse=True)
def _native_loaded():
    from regtr_b200 import lib
    lib.load()
    assert torch.cuda.is_available()


# ------------------------------------------------------------------ op-level goldens

def test_kpconv_vs_reference_golden(ops_golden):
    from regtr_b200 import ops
    g = ops_golden
    y = ops.kpconv(G(g['kp_q']), G(g['kp_s']), G(g['kp_inds'], torch.int32), G(g['kp_x']), G(g['kp_W']),
                   G(g['kp_kp']), float(g['kp_extent']))
    assert np.abs(N(y) - g['kp_out']).max() <= 2e-5 * np.abs(g['kp_out']).max()
    assert np.all(N(y)[3] == 0)


@pytest.mark.parametrize('impl', ['pipe', 'mma', 'ffma'])
@pytest.mark.parametrize('cin,cout', [(1, 64), (4, 16), (32, 32), (64, 64), (128, 128), (256, 256)])
def test_kpconv_all_channel_paths_vs_oracle(cin, cout, impl, monkeypatch):
    """The aggregation implementations (software-pipelined persistent tensor-core kernel = the default; the
    one-query-per-warp tensor-core kernel and the CUDA-core kernels kept for A/B and as the large-K fallback)
    on every channel-width path, incl. the fused Cin=1 block."""
    from oracle import regtr_oracle as O
    from regtr_b200 import ops
    if impl == 'pipe':
        monkeypatch.delenv('REGTR_AGG_IMPL', raising=False)
    else:
        monkeypatch.setenv('REGTR_AGG_IMPL', impl)
    rng = np.random.default_rng(cin)
    Nq, Ns, K = 301, 457, 40
    q = rng.normal(size=(Nq, 3)).astype(np.float32) * 0.05
    s = rng.normal(size=(Ns, 3)).astype(np.float32) * 0.05
    idx = rng.integers(0, Ns + 1, size=(Nq, K))
    idx[:, 30:] = np.where(rng.random((Nq, 10)) < 0.7, Ns, idx[:, 30:])     # shadow tails
    idx[7] = Ns
    x = rng.normal(size=(Ns, cin)).astype(np.float32) + (1.0 if cin == 1 else 0.0)
    W = (rng.normal(size=(15, cin, cout)) / np.sqrt(15 * cin)).astype(np.float32)
    kp = (rng.normal(size=(15, 3)) * 0.03).astype(np.float32)
    want = O.kpconv(*(torch.from_numpy(a) for a in (q, s)), torch.from_numpy(idx), torch.from_numpy(x),
                    torch.from_numpy(W), torch.from_numpy(kp), 0.05).numpy()
    got = N(ops.kpconv(G(q), G(s), G(idx, torch.int32), G(x), G(W), G(kp), 0.05))
    # SURVEY 8c feature tolerance (1e-4 * max|ref|); the kernels measure ~2e-7 here.  Twice in ~20 suite runs the
    # Cin = 1 case came out 5e-5 off on a few entries (not reproduced in isolated processes, sanitizer-clean:
    # DESIGN.md 9), hence not the tighter 2e-5 the other paths would allow.
    assert np.abs(got - want).max() <= 1e-4 * np.abs(want).max(), np.abs(got - want).max() / np.abs(want).max()


def test_maxpool_instnorm_posemb_vs_reference_golden(ops_golden):
    from regtr_b200 import ops
    g = ops_golden
    assert np.array_equal(N(ops.max_pool(G(g['kp_x']), G(g['kp_inds'], torch.int32))), g['maxpool_out'])
    offs = ops.make_offsets(g['inorm_lens'].tolist(), DEV)
    np.testing.assert_allclose(N(ops.instnorm_act(G(g['kp_x']), offs, 2)), g['inorm_out'], rtol=0, atol=3e-6)
    np.testing.assert_allclose(N(ops.pos_embed_sine(G(g['pe_xyz']))), g['pe_out'], rtol=0, atol=2e-6)


def test_instnorm_residual_act_large():
    from oracle import regtr_oracle as O
    from regtr_b200 import ops
    rng = np.random.default_rng(3)
    lens = [2500, 1, 3000, 777]
    x = (rng.normal(size=(sum(lens), 96)) * 3 + 5).astype(np.float32)
    res = rng.normal(size=x.shape).astype(np.float32)
    want = torch.nn.functional.leaky_relu(O.instance_norm(torch.from_numpy(x), lens) + torch.from_numpy(res), 0.1)
    got = ops.instnorm_act(G(x), ops.make_offsets(lens, DEV), 4, res=G(res), slope=0.1)
    np.testing.assert_allclose(N(got), want.numpy(), rtol=0, atol=5e-6)


def test_kabsch_vs_reference_golden(ops_golden):
    from regtr_b200.se3 import compute_rigid_transform
    g = ops_golden
    T = N(compute_rigid_transform(G(g['kabsch_a']), G(g['kabsch_b']), G(g['kabsch_w'])))
    np.testing.assert_allclose(T, g['kabsch_T'], rtol=0, atol=2e-5)
    assert np.all(np.linalg.det(T[..., :3].astype(np.float64)) > 0.999)


def test_kabsch_well_conditioned_vs_fp64():
    """Kabsch kernel alone <= 1e-6 vs an fp64 solve on well-conditioned correspondences (SURVEY 8c)."""
    from oracle import regtr_oracle as O
    from regtr_b200.se3 import compute_rigid_transform
    rng = np.random.default_rng(11)
    a = rng.normal(size=(24, 900, 3))
    R = np.stack([np.linalg.qr(rng.normal(size=(3, 3)))[0] for _ in range(24)])
    R *= np.sign(np.linalg.det(R))[:, None, None]
    b = np.einsum('bij,bnj->bni', R, a) + rng.normal(size=(24, 1, 3)) + rng.normal(size=a.shape) * 0.01
    w = rng.uniform(0, 1, size=(24, 900))
    want = O.kabsch(torch.from_numpy(a), torch.from_numpy(b), torch.from_numpy(w)).numpy()
    got = N(compute_rigid_transform(G(a, torch.float32), G(b, torch.float32), G(w, torch.float32)))
    assert np.abs(got - want).max() <= 1e-6


def test_cross_encoder_padded_api_vs_reference_golden(ops_golden):
    """Reference-style padded interface of TransformerCrossEncoder, B=2, vs the reference's outputs."""
    from regtr_b200.config import get_config
    from regtr_b200.transformer import (PositionEmbeddingCoordsSine, TransformerCrossEncoder,
                                        TransformerCrossEncoderLayer)
    from regtr_b200.weights import random_state_dict
    g = ops_golden
    cfg = get_config('3dmatch')
    sd = random_state_dict(cfg, 21)
    layer = TransformerCrossEncoderLayer(256, 8, 1024, 0.0, activation='relu', normalize_before=True,
                                         sa_val_has_pos_emb=True, ca_val_has_pos_emb=True)
    enc = TransformerCrossEncoder(layer, 6, torch.nn.LayerNorm(256), return_intermediate=True)
    enc.load_state_dict({k[len('transformer_encoder.'):]: v for k, v in sd.items()
                         if k.startswith('transformer_encoder.')}, strict=True)
    enc = enc.to(DEV).eval()
    pe = PositionEmbeddingCoordsSine(3, 256, scale=1.0)
    pad = torch.nn.utils.rnn.pad_sequence
    src = [G(g[f'xenc_src_{b}']) for b in range(2)]
    tgt = [G(g[f'xenc_tgt_{b}']) for b in range(2)]
    spe = [pe(G(g[f'xenc_sxyz_{b}'])) for b in range(2)]
    tpe = [pe(G(g[f'xenc_txyz_{b}'])) for b in range(2)]

    def mask(ts):
        m = torch.zeros((len(ts), max(t.shape[0] for t in ts)), dtype=torch.bool, device=DEV)
        for i, t in enumerate(ts):
            m[i, t.shape[0]:] = True
        return m
    with torch.no_grad():
        so, to = enc(pad(src), pad(tgt), src_key_padding_mask=mask(src), tgt_key_padding_mask=mask(tgt),
                     src_pos=pad(spe), tgt_pos=pad(tpe))
    for b in range(2):
        np.testing.assert_allclose(N(so[:, :src[b].shape[0], b]), g[f'xenc_src_out_{b}'], rtol=0, atol=5e-5)
        np.testing.assert_allclose(N(to[:, :tgt[b].shape[0], b]), g[f'xenc_tgt_out_{b}'], rtol=0, atol=5e-5)


# ------------------------------------------------------------- pre-processing, bit-exact

def _pre_inputs(seed, lens, scale=0.5, snap=0.05):
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-scale, scale, size=(sum(lens), 3)).astype(np.float32)
    k = min(64, len(pts))
    pts[:k] = np.round(pts[:k] / snap) * snap          # points exactly on voxel / cell faces
    return pts


@pytest.mark.parametrize('lens', [[900, 1100], [1, 2000, 0, 37], [5000]])
def test_grid_subsample_and_ball_query_bit_exact(lens):
    from oracle import pre
    from regtr_b200 import ops
    pts = _pre_inputs(sum(lens), lens)
    dl, r, K = 0.05, 0.0625, 40
    n_clouds = len(lens)
    offs = ops.make_offsets(lens, DEV)
    status = ops.new_status(DEV)
    sub, sub_offs = ops.grid_subsample(G(pts), offs, n_clouds, dl, status)
    want_sub, want_len = pre.grid_subsample(pts, lens, dl)
    so = N(sub_offs)
    assert np.array_equal(np.diff(so), want_len)
    assert np.array_equal(N(sub)[:so[-1]], want_sub)            # bit-exact barycentres, canonical order
    grid = ops.CellGrid(G(pts), offs, n_clouds, r * 1.0001, status)
    i32, i64 = ops.ball_query(G(pts), offs, G(pts), offs, grid, K, r, q_order=grid.order)
    want = pre.ball_query(pts, lens, pts, lens, K, r)
    assert np.array_equal(N(i64), want) and np.array_equal(N(i32).astype(np.int64), want)
    # strided query: coarse queries against fine supports, capacity-padded query buffer
    p32, _ = ops.ball_query(sub, sub_offs, G(pts), offs, grid, K, r)
    want_p = pre.ball_query(want_sub, want_len, pts, lens, K, r)
    assert np.array_equal(N(p32)[:so[-1]].astype(np.int64), want_p)
    assert int(status.item()) == 0


def test_ball_query_dense_cluster_overflow_path():
    """More hits than the per-warp staging buffer (384): the keep-K-smallest compaction must still
    return the first K supports in index order."""
    from oracle import pre
    from regtr_b200 import ops
    rng = np.random.default_rng(2)
    pts = np.concatenate([rng.normal(size=(1500, 3)) * 0.01, rng.uniform(-1, 1, size=(500, 3))]).astype(np.float32)
    pts = pts[rng.permutation(len(pts))]
    lens = [len(pts)]
    offs = ops.make_offsets(lens, DEV)
    status = ops.new_status(DEV)
    grid = ops.CellGrid(G(pts), offs, 1, 0.0626, status)
    for K in (40, 50, 128):
        _, i64 = ops.ball_query(G(pts), offs, G(pts), offs, grid, K, 0.0625)
        assert np.array_equal(N(i64), pre.ball_query(pts, lens, pts, lens, K, 0.0625))


def test_key_range_status_flag():
    from regtr_b200 import ops
    pts = np.array([[0, 0, 0], [5000.0, 0, 0]], dtype=np.float32)     # 5000 / 0.05 = 100000 cells
    status = ops.new_status(DEV)
    ops.grid_subsample(G(pts), ops.make_offsets([2], DEV), 1, 0.05, status)
    assert int(status.item()) & 1


# ---------------------------------------------------------------------- full forward

def _run_model(cfg, sd, src, tgt):
    from regtr_b200.regtr import RegTR
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    batch = {'src_xyz': [G(s) for s in src], 'tgt_xyz': [G(t) for t in tgt]}
    out = model(batch)
    torch.cuda.synchronize()
    return out, batch['kpconv_meta']


@pytest.mark.parametrize('case', sorted(FORWARD_CASES))
def test_forward_vs_reference_golden(case):
    cfg, sd, src, tgt = make_case(case)
    out, meta = _run_model(cfg, sd, src, tgt)
    assert out['pose'].shape == (6, len(src), 3, 4)
    check_forward_against_golden(out, meta, load_golden(case), len(src), feat_rtol=1e-4, corr_atol=1e-4,
                                 logit_atol=2e-4, pose_atol=1e-4)


@pytest.mark.parametrize('case', sorted(VARIANT_CASES))
def test_variant_forward_vs_reference_golden(case):
    """SURVEY.md 8f N4 branches on the CUDA path: CorrespondenceDecoder (regtr_corr_decode_fwd), forward_post,
    PositionEmbeddingLearned -- against the unmodified reference run with the same config and weights."""
    cfg, sd, src, tgt = make_case(case)
    out, meta = _run_model(cfg, sd, src, tgt)
    check_forward_against_golden(out, meta, load_golden(case), len(src), feat_rtol=1e-4, corr_atol=1e-4,
                                 logit_atol=2e-4, pose_atol=1e-4)


def test_graph_executor_recaptures_after_load_state_dict():
    """The captured graphs hold pointers to the split TF32 weights: reloading the weights must not leave a graph
    replaying the old ones (ADVICE round 1)."""
    from regtr_b200.regtr import GraphedRegTR, RegTR
    from regtr_b200.weights import random_state_dict
    cfg, sd, src, tgt = make_case('fwd_modelnet_b1')
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    runner = GraphedRegTR(model, bucket=2048, ratio=1.0)
    batch = lambda: {'src_xyz': [G(a) for a in src], 'tgt_xyz': [G(a) for a in tgt]}
    p0 = N(runner(batch())['pose']).copy()
    model.load_state_dict(random_state_dict(cfg, 777), strict=True)
    p1 = N(runner(batch())['pose']).copy()
    want = N(model(batch())['pose'])
    assert np.abs(p1 - want).max() <= 1e-5 and np.abs(p1 - p0).max() > 1e-3


def test_variant_forward_through_graph_executor():
    """The attention decoder + learned embedding also run capacity-shaped inside a CUDA graph."""
    from regtr_b200.regtr import GraphedRegTR, RegTR
    case = 'var_modelnet_learnedpe_attndec_b2'
    cfg, sd, src, tgt = make_case(case)
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    # ModelNet's single subsampling step keeps ~85 % of the points: level capacities = level-0 capacity
    runner = GraphedRegTR(model, bucket=2048, ratio=1.0)
    batch = {'src_xyz': [G(a) for a in src], 'tgt_xyz': [G(a) for a in tgt]}
    out = runner(batch)
    check_forward_against_golden(out, batch['kpconv_meta'], load_golden(case), len(src), feat_rtol=1e-4,
                                 corr_atol=1e-4, logit_atol=2e-4, pose_atol=1e-4)
    assert runner.fallbacks == 0


def test_attention_cores_agree_and_match_float64(monkeypatch):
    """The fp32-accurate attention cores (mma.sync 3xTF32 default, CUDA-core REGTR_MHA_IMPL=ffma) on ragged
    self and cross problems, incl. a 1-token cloud and lengths around the 64-key chunk."""
    from regtr_b200 import ops
    from regtr_b200.transformer import AttentionPlan
    rng = np.random.default_rng(11)
    lens, E, H = [130, 1, 64, 65, 3, 200], 256, 8
    n = sum(lens)
    q, k, v = (G((rng.normal(size=(n, E)) * 0.7).astype(np.float32)) for _ in range(3))
    plan = AttentionPlan(lens, DEV)
    starts = np.concatenate([[0], np.cumsum(lens)])
    B = len(lens) // 2
    for cross in (False, True):
        ks, kl = (plan.xk_start, plan.xk_len) if cross else (plan.q_start, plan.q_len)
        ref = np.zeros((n, E))
        for c in range(len(lens)):
            o = (c + B if c < B else c - B) if cross else c
            qq = N(q)[starts[c]:starts[c + 1]].astype(np.float64).reshape(-1, H, 32).transpose(1, 0, 2)
            kk = N(k)[starts[o]:starts[o + 1]].astype(np.float64).reshape(-1, H, 32).transpose(1, 0, 2)
            vv = N(v)[starts[o]:starts[o + 1]].astype(np.float64).reshape(-1, H, 32).transpose(1, 0, 2)
            sc = qq @ kk.transpose(0, 2, 1) / np.sqrt(32)
            w = np.exp(sc - sc.max(-1, keepdims=True)); w /= w.sum(-1, keepdims=True)
            ref[starts[c]:starts[c + 1]] = (w @ vv).transpose(1, 0, 2).reshape(-1, E)
        for impl in ('mma', 'ffma'):
            monkeypatch.setenv('REGTR_MHA_IMPL', impl)
            got = N(ops.mha_varlen(q, k, v, plan.q_start, plan.q_len, ks, kl, plan.max_len, H))
            assert np.abs(got - ref).max() <= 1e-5, (impl, cross)
            if impl == 'mma':
                got_mma = got
        # linear tile table (capacity-shaped launches): host-built exact total, device-built with a capacity bound
        monkeypatch.setenv('REGTR_MHA_IMPL', 'mma')
        dplan = AttentionPlan.from_device(ops.make_offsets(lens, DEV), B, n + 500)
        assert np.array_equal(N(dplan.tiles64[0]), N(plan.tiles64[0])) and dplan.tiles64[1] >= plan.tiles64[1]
        assert np.array_equal(N(dplan.tiles128[0]), N(plan.tiles128[0]))
        for pl in (plan, dplan):
            ks2, kl2 = (pl.xk_start, pl.xk_len) if cross else (pl.q_start, pl.q_len)
            lin = N(ops.mha_varlen(q, k, v, pl.q_start, pl.q_len, ks2, kl2, pl.max_len, H, tiles=pl.tiles64))
            assert np.array_equal(lin, got_mma)


def test_corr_decode_vs_float64():
    """regtr_corr_decode_fwd alone: ragged problems, several layers, vs a float64 softmax-attention."""
    from regtr_b200 import ops
    from regtr_b200.transformer import AttentionPlan
    rng = np.random.default_rng(3)
    lens, L_, D = [37, 1, 50, 129], 3, 256
    n = sum(lens)
    qp = G(rng.normal(size=(L_ * n, D)).astype(np.float32))
    kp = G(rng.normal(size=(L_ * n, D)).astype(np.float32))
    xyz = G(rng.normal(size=(n, 3)).astype(np.float32))
    plan = AttentionPlan(lens, DEV)
    got = N(ops.corr_decode(qp, kp, xyz, plan.q_start, plan.q_len, plan.xk_start, plan.xk_len, plan.max_len, L_))
    starts = np.concatenate([[0], np.cumsum(lens)])
    B = len(lens) // 2
    q64, k64, x64 = N(qp).astype(np.float64).reshape(L_, n, D), N(kp).astype(np.float64).reshape(L_, n, D), N(xyz).astype(np.float64)
    for c in range(len(lens)):
        o = c + B if c < B else c - B
        qs, ks = slice(starts[c], starts[c + 1]), slice(starts[o], starts[o + 1])
        for l in range(L_):
            sc = q64[l, qs] @ k64[l, ks].T / np.sqrt(D)
            w = np.exp(sc - sc.max(1, keepdims=True)); w /= w.sum(1, keepdims=True)
            np.testing.assert_allclose(got.reshape(L_, n, 3)[l, qs], w @ x64[ks], rtol=0, atol=2e-5)


def test_forward_3dmatch_full_size_vs_oracle():
    """BASELINE config 2 (one ~20k-point pair): indices bit-exact vs the oracle pyramid, float stages
    vs the oracle run on the same pyramid, pose within 1e-4."""
    from oracle import pre, regtr_oracle as O
    from regtr_b200.config import get_config
    from regtr_b200.synthetic import make_3dmatch_pair
    from regtr_b200.weights import random_state_dict
    cfg = get_config('3dmatch')
    sd = random_state_dict(cfg, 5)
    p = make_3dmatch_pair(2000)
    out, meta = _run_model(cfg, sd, [p['src_xyz']], [p['tgt_xyz']])
    want = pre.preprocess(cfg, [p['src_xyz'], p['tgt_xyz']])
    for key in ('points', 'neighbors', 'pools', 'upsamples', 'stack_lengths'):
        for lvl, (a, b) in enumerate(zip(meta[key], want[key])):
            assert np.array_equal(N(a), b), f'{key}[{lvl}]'
    ref = O.forward(sd, cfg, [p['src_xyz']], [p['tgt_xyz']], meta=want)
    for k, rtol in (('src_feat_un', 1e-4), ('tgt_feat_un', 1e-4), ('src_feat', 1e-4), ('tgt_feat', 1e-4)):
        a, b = N(out[k][0]), ref[k][0].numpy()
        assert np.abs(a - b).max() <= rtol * np.abs(b).max(), k
    assert np.abs(N(out['src_kp_warped'][0]) - ref['src_kp_warped'][0].numpy()).max() <= 1e-4
    assert np.abs(N(out['pose']) - ref['pose'].numpy()).max() <= 1e-4
    # size-independent property: the pose is a proper rigid transform on every layer
    R = N(out['pose'])[..., :3].astype(np.float64)
    assert np.abs(R @ np.swapaxes(R, -1, -2) - np.eye(3)).max() <= 1e-5 and np.all(np.linalg.det(R) > 0)


def test_forward_is_deterministic_and_batch_invariant():
    """Same pair alone and inside a batch of 3 gives bit-identical indices and (near-)identical pose."""
    from regtr_b200.config import get_config
    from regtr_b200.synthetic import make_3dmatch_pair
    from regtr_b200.weights import random_state_dict
    cfg = get_config('3dmatch')
    sd = random_state_dict(cfg, 6)
    ps = [make_3dmatch_pair(2100 + i, 4000) for i in range(3)]
    o1, m1 = _run_model(cfg, sd, [ps[1]['src_xyz']], [ps[1]['tgt_xyz']])
    o1b, _ = _run_model(cfg, sd, [ps[1]['src_xyz']], [ps[1]['tgt_xyz']])
    o3, m3 = _run_model(cfg, sd, [p['src_xyz'] for p in ps], [p['tgt_xyz'] for p in ps])
    assert torch.equal(o1['pose'], o1b['pose'])
    assert torch.equal(o1['src_kp'][0], o3['src_kp'][1])
    assert float((o1['pose'][:, 0] - o3['pose'][:, 1]).abs().max()) <= 5e-5   # tile shapes differ with M


def test_graphed_executor_matches_eager_and_survives_overflow():
    """CUDA-graph executor (static capacities, device-side sizes) vs the eager forward: identical
    indices / key points, near-identical floats; several inputs through ONE captured graph; host
    (pinned) inputs; and the eager fallback when a level overflows its static capacity."""
    from regtr_b200.config import get_config
    from regtr_b200.regtr import GraphedRegTR, RegTR
    from regtr_b200.synthetic import make_3dmatch_pair
    from regtr_b200.weights import random_state_dict
    cfg = get_config('3dmatch')
    sd = random_state_dict(cfg, 8)
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    runner = GraphedRegTR(model, bucket=16384)
    for i, n in enumerate((5000, 6000, 5500)):
        p = make_3dmatch_pair(2200 + i, n)
        b_e = {'src_xyz': [G(p['src_xyz'])], 'tgt_xyz': [G(p['tgt_xyz'])]}
        b_g = {'src_xyz': [G(p['src_xyz'])], 'tgt_xyz': [G(p['tgt_xyz'])]} if i != 1 else \
            {'src_xyz': [torch.from_numpy(p['src_xyz']).pin_memory()], 'tgt_xyz': [torch.from_numpy(p['tgt_xyz']).pin_memory()]}
        want = model(b_e)
        got = runner(b_g)
        for key in ('neighbors', 'pools', 'upsamples', 'points', 'stack_lengths'):
            for a, b in zip(b_g['kpconv_meta'][key], b_e['kpconv_meta'][key]):
                assert torch.equal(a, b), key
        assert torch.equal(got['src_kp'][0], want['src_kp'][0])
        s = float(want['src_feat'][0].abs().max())
        assert float((got['src_feat'][0] - want['src_feat'][0]).abs().max()) <= 2e-5 * s
        assert float((got['pose'] - want['pose']).abs().max()) <= 5e-5     # two fp32-accurate evaluation orders
        assert torch.equal(got['host_pose'], got['pose'].cpu())
    assert len(runner.graphs) == 1 and runner.fallbacks == 0
    # volume-filling cloud: every point its own voxel -> level 1 does not fit 0.4 * cap0 -> eager fallback
    rng = np.random.default_rng(0)
    src = rng.uniform(-2, 2, size=(7000, 3)).astype(np.float32)
    tgt = rng.uniform(-2, 2, size=(7000, 3)).astype(np.float32)
    b_e = {'src_xyz': [G(src)], 'tgt_xyz': [G(tgt)]}
    b_g = {'src_xyz': [torch.from_numpy(src).pin_memory()], 'tgt_xyz': [torch.from_numpy(tgt).pin_memory()]}   # HOST clouds
    want, got = model(b_e), runner(b_g)
    assert runner.fallbacks == 1
    assert torch.equal(got['pose'], want['pose']) and torch.equal(got['host_pose'], want['pose'].cpu())
    assert torch.equal(b_g['kpconv_meta']['neighbors'][1], b_e['kpconv_meta']['neighbors'][1])
    # the bucket's graph (and its scratch namespace) was dropped for a re-capture with more head-room: the next
    # ordinary pair of that bucket is captured afresh and replayed without a fallback
    p = make_3dmatch_pair(2299, 6200)
    want3 = model({'src_xyz': [G(p['src_xyz'])], 'tgt_xyz': [G(p['tgt_xyz'])]})
    got3 = runner({'src_xyz': [G(p['src_xyz'])], 'tgt_xyz': [G(p['tgt_xyz'])]})
    assert runner.fallbacks == 1 and float((got3['pose'] - want3['pose']).abs().max()) <= 5e-5


def test_tcgen05_attention_core_vs_fp32_kernel():
    """bf16 wgmma attention (TMA-fed, register accumulators) vs the fp32 parity kernel on ragged self and
    cross problems (unaligned key ranges, partial tiles, a 7-token cloud).  Tolerance of the fast mode:
    3e-2 * max|ref| (bf16 operands, SURVEY 8c)."""
    from regtr_b200 import ops
    from regtr_b200.transformer import AttentionPlan
    torch.manual_seed(0)
    E, H = 256, 8
    for lens in ([410, 339], [130, 7, 300, 129], [64, 64]):
        N = sum(lens)
        x = torch.randn(N, E, device=DEV)
        W = torch.randn(3 * E, E, device=DEV) / E ** 0.5
        b = torch.randn(3 * E, device=DEV) * 0.1
        plan = AttentionPlan(lens, DEV)
        qkv = ops.linear(x, W, b)
        for ks, kl in ((plan.q_start, plan.q_len), (plan.xk_start, plan.xk_len)):
            want = ops.mha_varlen(qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:], plan.q_start, plan.q_len, ks, kl,
                                  plan.max_len, H)
            got = ops.mha_bf16_tc(x, W, b, plan.q_start, plan.q_len, ks, kl, plan.max_len, H)
            assert torch.isfinite(got).all()
            assert float((got - want).abs().max()) <= 3e-2 * float(want.abs().max())


def test_forward_fast_mode_bf16_attention():
    """Full forward with attention_impl='bf16_tc' vs the oracle: indices exact (same pyramid), features
    within 3e-2 * max|ref|, rotation still orthonormal; the parity mode keeps the 1e-4 pose bound."""
    from oracle import pre, regtr_oracle as O
    from regtr_b200.config import get_config
    from regtr_b200.regtr import RegTR
    from regtr_b200.synthetic import make_3dmatch_pair
    from regtr_b200.weights import random_state_dict
    cfg = get_config('3dmatch')
    cfg.attention_impl = 'bf16_tc'
    sd = random_state_dict(cfg, 5)
    p = make_3dmatch_pair(2300, 6000)
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    batch = {'src_xyz': [G(p['src_xyz'])], 'tgt_xyz': [G(p['tgt_xyz'])]}
    out = model(batch)
    want = pre.preprocess(cfg, [p['src_xyz'], p['tgt_xyz']])
    ref = O.forward(sd, cfg, [p['src_xyz']], [p['tgt_xyz']], meta=want)
    for k in ('src_feat', 'tgt_feat'):
        a, b = N(out[k][0]), ref[k][0].numpy()
        assert np.abs(a - b).max() <= 3e-2 * np.abs(b).max(), k
    assert np.abs(N(out['src_feat_un'][0]) - ref['src_feat_un'][0].numpy()).max() <= 1e-4 * float(ref['src_feat_un'][0].abs().max())
    R = N(out['pose'])[..., :3].astype(np.float64)
    assert np.abs(R @ np.swapaxes(R, -1, -2) - np.eye(3)).max() <= 1e-5
    assert np.abs(N(out['pose']) - ref['pose'].numpy()).max() <= 5e-2


def test_pipelined_executor_matches_serial():
    """Three forwards in flight on private streams give the same poses as the serial graph executor
    (private scratch namespaces: no aliasing between concurrently replayed graphs)."""
    from regtr_b200.config import get_config
    from regtr_b200.regtr import GraphedRegTR, PipelinedRegTR, RegTR
    from regtr_b200.synthetic import make_3dmatch_pair
    from regtr_b200.weights import random_state_dict
    cfg = get_config('3dmatch')
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(random_state_dict(cfg, 9), strict=True)
    pairs = [make_3dmatch_pair(2400 + i, 5000 + 300 * i) for i in range(7)]
    batches = lambda: [{'src_xyz': [G(p['src_xyz'])], 'tgt_xyz': [G(p['tgt_xyz'])]} for p in pairs]
    serial = GraphedRegTR(model, bucket=16384)
    want = [serial(b)['pose'].cpu().clone() for b in batches()]
    pipe = PipelinedRegTR(model, depth=3, bucket=16384)
    got = []
    for b in batches():
        done = pipe.submit(b)
        if done is not None:
            got.append(done['host_pose'].clone())
    got += [o['host_pose'].clone() for o in pipe.drain()]
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert torch.equal(a, b)


def test_graphed_executor_batch_of_two_pairs():
    """B=2 through the CUDA-graph executor: per-pair poses equal the eager forward's, lists have
    the reference's layout (B entries per key)."""
    from regtr_b200.config import get_config
    from regtr_b200.regtr import GraphedRegTR, RegTR
    from regtr_b200.synthetic import make_3dmatch_pair
    from regtr_b200.weights import random_state_dict
    cfg = get_config('3dmatch')
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(random_state_dict(cfg, 10), strict=True)
    ps = [make_3dmatch_pair(2500 + i, 4000 + 1500 * i) for i in range(2)]
    mk = lambda: {'src_xyz': [G(p['src_xyz']) for p in ps], 'tgt_xyz': [G(p['tgt_xyz']) for p in ps]}
    want, b_e = model(mk()), None
    runner = GraphedRegTR(model, bucket=16384)
    b_g = mk()
    got = runner(b_g)
    assert got['pose'].shape == (6, 2, 3, 4) and len(got['src_feat']) == 2 and len(got['tgt_kp_warped']) == 2
    assert float((got['pose'] - want['pose']).abs().max()) <= 5e-5
    for b in range(2):
        assert got['src_kp'][b].shape == want['src_kp'][b].shape and torch.equal(got['src_kp'][b], want['src_kp'][b])
        assert got['src_overlap'][b].shape == want['src_overlap'][b].shape
    assert [int(v) for v in b_g['kpconv_meta']['stack_lengths'][0]] == [len(p['src_xyz']) for p in ps] + [len(p['tgt_xyz']) for p in ps]


# ------------------------------------------------- the reference's own sample clouds (real data)

@pytest.mark.parametrize('case', sorted(REAL_CASES))
def test_forward_real_pairs_vs_reference_golden(case):
    """The inputs src/demo.py:154-192 runs -- real 3DMatch fragments (6 mm sensor lattice: voxel-boundary hits
    are common, SURVEY.md 7-H1) and the ModelNet demo plys -- through the CUDA path, against the unmodified
    reference: level sizes, coarse points and all neighbour indices bit-exact (SHA-256), features 1e-4, pose 1e-4."""
    cfg, sd, src, tgt = make_real_case(case)
    out, meta = _run_model(cfg, sd, [src], [tgt])
    check_real_forward_against_golden(out, meta, load_golden(case), feat_rtol=1e-4, corr_atol=1e-4,
                                      logit_atol=2e-4, pose_atol=1e-4)


def test_real_pair_through_graph_executor_host_inputs():
    """Same, through the CUDA-graph executor with pinned HOST clouds (the serving path of bench.py's e2e leg)."""
    from regtr_b200.regtr import GraphedRegTR, RegTR
    case = 'real_3dmatch_redkitchen_0_5'
    cfg, sd, src, tgt = make_real_case(case)
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    runner = GraphedRegTR(model)
    batch = {'src_xyz': [torch.from_numpy(src).pin_memory()], 'tgt_xyz': [torch.from_numpy(tgt).pin_memory()]}
    out = runner(batch)
    assert runner.fallbacks == 0
    check_real_forward_against_golden(out, batch['kpconv_meta'], load_golden(case), feat_rtol=1e-4, corr_atol=1e-4,
                                      logit_atol=2e-4, pose_atol=1e-4)
    assert torch.equal(out['host_pose'], out['pose'].cpu())


# ------------------------------------------------- BASELINE configs 3 / 4 (8 pairs per GPU per step) and 5

def _oracle_pose_and_meta(cfg, sd, p):
    from oracle import pre, regtr_oracle as O
    want = pre.preprocess(cfg, [p['src_xyz'], p['tgt_xyz']])
    return O.forward(sd, cfg, [p['src_xyz']], [p['tgt_xyz']], meta=want), want


def test_config3_batch8_full_size_vs_oracle():
    """BASELINE config 3 / the per-GPU share of config 4: 8 full-size (~20k-point) pairs in ONE forward through
    the CUDA-graph executor, fp32 parity mode.  Every pair is independent (SURVEY.md 8e), so each is checked
    against the oracle run on that pair alone: indices exact, features 1e-4, pose 1e-4."""
    from regtr_b200.config import get_config
    from regtr_b200.regtr import GraphedRegTR, RegTR
    from regtr_b200.synthetic import make_batch
    from regtr_b200.weights import random_state_dict
    cfg = get_config('3dmatch')
    sd = random_state_dict(cfg, 5)
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    B = 8
    b = make_batch(3, B)
    batch = {'src_xyz': [G(a) for a in b['src_xyz']], 'tgt_xyz': [G(a) for a in b['tgt_xyz']]}
    runner = GraphedRegTR(model)
    out = runner(batch)
    assert runner.fallbacks == 0 and out['pose'].shape == (6, B, 3, 4)
    meta = batch['kpconv_meta']
    n_lvl = len(meta['points'])
    lens = [[int(v) for v in meta['stack_lengths'][l]] for l in range(n_lvl)]
    starts = [np.concatenate([[0], np.cumsum(l)]) for l in lens]
    for i in (0, 3, 7):                                         # three of the eight pairs against the oracle
        p = {k: b[k][i] for k in ('src_xyz', 'tgt_xyz')}
        ref, want = _oracle_pose_and_meta(cfg, sd, p)
        for l in range(n_lvl):
            assert [lens[l][i], lens[l][B + i]] == [int(v) for v in want['stack_lengths'][l]], (i, l)
            # the pair's rows inside the stacked level: src block i, tgt block B + i; indices are stack-relative
            for blk, (lo_w, hi_w) in ((i, (0, lens[l][i])), (B + i, (lens[l][i], lens[l][i] + lens[l][B + i]))):
                rows = slice(starts[l][blk], starts[l][blk + 1])
                assert np.array_equal(N(meta['points'][l][rows]), want['points'][l][lo_w:hi_w]), (i, l, 'points')
                got = N(meta['neighbors'][l][rows])
                w = want['neighbors'][l][lo_w:hi_w]
                shadow_g, shadow_w = sum(lens[l]), want['points'][l].shape[0]
                # map stack-relative ids to cloud-relative ones on both sides (shadow -> -1)
                g_rel = np.where(got == shadow_g, -1, got - starts[l][blk])
                w_rel = np.where(w == shadow_w, -1, w - lo_w)
                assert np.array_equal(g_rel, w_rel), (i, l, 'neighbors')
        for side in ('src', 'tgt'):
            a, r = N(out[f'{side}_feat'][i]), ref[f'{side}_feat'][0].numpy()
            assert np.abs(a - r).max() <= 1e-4 * np.abs(r).max(), (i, side)
        assert np.abs(N(out['pose'][:, i]) - ref['pose'][:, 0].numpy()).max() <= 1e-4, i
    R = N(out['pose'])[..., :3].astype(np.float64)               # all 8: proper rotations on every layer
    assert np.abs(R @ np.swapaxes(R, -1, -2) - np.eye(3)).max() <= 1e-5 and np.all(np.linalg.det(R) > 0)


def test_config5_lomatch_30k_pair_vs_oracle():
    """BASELINE config 5: a ~30k-point low-overlap (10-30 %) pair -- a new level-0 capacity bucket and denser
    K-truncation -- eager and through the graph executor, against the oracle: indices exact, pose 1e-4."""
    from regtr_b200.config import get_config
    from regtr_b200.regtr import GraphedRegTR, RegTR
    from regtr_b200.synthetic import make_batch
    from regtr_b200.weights import random_state_dict
    cfg = get_config('3dmatch')
    sd = random_state_dict(cfg, 5)
    b = make_batch(5, 1)
    p = {k: b[k][0] for k in ('src_xyz', 'tgt_xyz')}
    assert 25000 <= len(p['src_xyz']) <= 36000
    ref, want = _oracle_pose_and_meta(cfg, sd, p)
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    runner = GraphedRegTR(model)
    for run in (model, runner):
        batch = {'src_xyz': [G(p['src_xyz'])], 'tgt_xyz': [G(p['tgt_xyz'])]}
        out = run(batch)
        meta = batch['kpconv_meta']
        for key in ('points', 'neighbors', 'pools', 'stack_lengths'):
            for lvl, (a, w) in enumerate(zip(meta[key], want[key])):
                assert np.array_equal(N(a), w), f'{key}[{lvl}]'
        for k in ('src_feat', 'tgt_feat'):
            a, r = N(out[k][0]), ref[k][0].numpy()
            assert np.abs(a - r).max() <= 1e-4 * np.abs(r).max(), k
        assert np.abs(N(out['pose']) - ref['pose'].numpy()).max() <= 1e-4
    assert runner.fallbacks == 0
    trunc = float((N(meta['neighbors'][0])[:, -1] < want['points'][0].shape[0]).mean())
    assert trunc > 0.02                                          # the K=40 truncation regime is exercised


def test_two_capacity_buckets_on_one_runner_keep_their_scratch():
    """One executor, two level-0 capacity buckets (8192-point and 16384-point graphs): capturing the larger
    graph must not free or alias the scratch the smaller graph's replay writes (every captured graph owns a
    private scratch namespace).  The small bucket is replayed AFTER the large one was captured and after
    unrelated allocations recycled the caching allocator's free blocks."""
    from regtr_b200.config import get_config
    from regtr_b200.regtr import GraphedRegTR, RegTR
    from regtr_b200.synthetic import make_3dmatch_pair
    from regtr_b200.weights import random_state_dict
    cfg = get_config('3dmatch')
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(random_state_dict(cfg, 12), strict=True)
    small = [make_3dmatch_pair(2600 + i, 3000 + 200 * i) for i in range(2)]
    large = make_3dmatch_pair(2610, 6500)
    mk = lambda p: {'src_xyz': [G(p['src_xyz'])], 'tgt_xyz': [G(p['tgt_xyz'])]}
    want_small = [model(mk(p))['pose'].clone() for p in small]
    want_large = model(mk(large))['pose'].clone()
    runner = GraphedRegTR(model, bucket=8192)
    got0 = runner(mk(small[0]))['pose'].clone()
    gotL = runner(mk(large))['pose'].clone()
    assert len(runner.graphs) == 2 and runner.fallbacks == 0
    junk = [torch.full((1 << 22,), float('nan'), device=DEV) for _ in range(8)]     # churn the allocator
    del junk
    torch.cuda.empty_cache()
    got1 = runner(mk(small[1]))['pose'].clone()
    got0b = runner(mk(small[0]))['pose'].clone()
    gotLb = runner(mk(large))['pose'].clone()
    assert torch.equal(got0, got0b) and torch.equal(gotL, gotLb)
    for g, w in ((got0, want_small[0]), (got1, want_small[1]), (gotL, want_large)):
        assert float((g - w).abs().max()) <= 5e-5


def test_staged_executor_matches_and_reports_stage_times():
    """stages=True: the four reference `_TIMEIT` stages as four graphs; same results, stage times add up."""
    from regtr_b200.config import get_config
    from regtr_b200.regtr import GraphedRegTR, RegTR
    from regtr_b200.synthetic import make_3dmatch_pair
    from regtr_b200.weights import random_state_dict
    cfg = get_config('3dmatch')
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(random_state_dict(cfg, 13), strict=True)
    p = make_3dmatch_pair(2700, 6000)
    mk = lambda: {'src_xyz': [G(p['src_xyz'])], 'tgt_xyz': [G(p['tgt_xyz'])]}
    one, four = GraphedRegTR(model, bucket=16384), GraphedRegTR(model, bucket=16384, stages=True)
    a = one(mk())
    b = four(mk())
    b = four(mk())
    assert torch.equal(a['pose'], b['pose'])
    ms = four.stage_ms()
    assert list(ms) == ['preprocess', 'encoder', 'attention_decoder', 'pose'] and all(v > 0 for v in ms.values())


# ------------------------------------------------- InstanceNorm statistics in the GEMM epilogue

@pytest.mark.parametrize('lens,N,K', [([700, 1, 0, 333, 90], 64, 96),        # cloud boundaries inside 32-row groups, empty + 1-row clouds
                                      ([4000, 4100], 128, 64),               # BN = 128 tiles, many m-tiles
                                      ([300, 260], 256, 3840),               # split-K path (k_splitk_reduce_stats)
                                      ([5000, 4000, 3000, 100], 32, 480)])   # BN = 32 contraction shape
def test_gemm_instats_matches_float64(lens, N, K):
    """regtr_gemm_tf32x3_instats: C and the per-cloud (mean, rstd) of C from the epilogue's 32-row partial sums
    (+ fixed-order finalisation, no atomics) vs float64; capacity padding rows (m_dev) excluded; bit-identical
    across repeated calls."""
    from regtr_b200 import ops
    rng = np.random.default_rng(N + K)
    M = sum(lens)
    cap = M + 200                                               # capacity-shaped launch with a device row count
    a = np.zeros((cap, K), dtype=np.float32)
    a[:M] = rng.normal(size=(M, K)) * 1.3 + 0.4
    a[M:] = 1e3                                                 # garbage in the padding rows must not leak into the statistics
    w = (rng.normal(size=(N, K)) / np.sqrt(K)).astype(np.float32)
    offs = ops.make_offsets(lens, DEV)
    m_dev = offs[len(lens):len(lens) + 1]
    hi, lo = ops.split_weight(G(w))
    out, stats = ops.gemm_instats(G(a), hi, lo, offs, len(lens), m_dev=m_dev)
    out2, stats2 = ops.gemm_instats(G(a), hi, lo, offs, len(lens), m_dev=m_dev)
    assert torch.equal(stats, stats2) and torch.equal(out[:M], out2[:M])           # deterministic
    c64 = a[:M].astype(np.float64) @ w.astype(np.float64).T
    assert np.abs(N_(out)[:M] - c64).max() <= 1e-5 * np.abs(c64).max() * max(1.0, (K / 256) ** 0.5)
    st = N_(stats)
    starts = np.concatenate([[0], np.cumsum(lens)])
    for c, n in enumerate(lens):
        if n == 0:
            continue
        blk = c64[starts[c]:starts[c + 1]]
        mean, var = blk.mean(0), blk.var(0)
        np.testing.assert_allclose(st[c, :, 0], mean, rtol=0, atol=2e-6 * max(1.0, np.abs(c64).max()))
        np.testing.assert_allclose(st[c, :, 1], 1.0 / np.sqrt(var + 1e-5), rtol=2e-5, atol=0)
    # the fused pair (GEMM with statistics + apply) equals the separate-pass InstanceNorm
    want = ops.instnorm_act(out[:M].contiguous(), offs, len(lens), slope=0.1)
    got = ops.instnorm_apply(out[:M].contiguous(), offs, len(lens), stats, slope=0.1)
    assert float((got - want).abs().max()) <= 5e-6


def N_(t):
    return t.detach().cpu().numpy()


@pytest.mark.parametrize('N,K', [(32, 64), (32, 480), (64, 960), (128, 32), (128, 64), (256, 64)])
def test_gemm_persistent_tiles_vs_float64(N, K):
    """Launches of several waves walk their tiles persistently (tile loop per CTA, barrier phases running across
    tiles, the next tile's loads in flight under the epilogue): bias / residual / ReLU, a device-side row count that ends inside
    a tile, InstanceNorm partials of two clouds, all against float64; repeated calls bit-identical."""
    from regtr_b200 import ops
    rng = np.random.default_rng(N * 1000 + K)
    cap, M = 46000, 44321                                      # 360 row tiles > 2 x 132 SMs; the last real tile is partial
    a = np.zeros((cap, K), dtype=np.float32)
    a[:M] = rng.normal(size=(M, K)) * 0.9 + 0.2
    a[M:] = 7e2
    w = (rng.normal(size=(N, K)) / np.sqrt(K)).astype(np.float32)
    b = rng.normal(size=N).astype(np.float32)
    res = rng.normal(size=(cap, N)).astype(np.float32)
    lens = [20000, M - 20000]
    offs = ops.make_offsets(lens, DEV)
    m_dev = offs[2:3]
    hi, lo = ops.split_weight(G(w))
    A, Rr, Bb = G(a), G(res), G(b)
    c64 = a[:M].astype(np.float64) @ w.astype(np.float64).T
    tol = 1e-5 * np.abs(c64).max() * max(1.0, (K / 256) ** 0.5)
    out = ops.gemm(A, hi, lo, bias=Bb, residual=Rr, relu=True, m_dev=m_dev)
    want = np.maximum(c64 + b.astype(np.float64) + res[:M].astype(np.float64), 0.0)
    assert np.abs(N_(out)[:M] - want).max() <= tol + 1e-6
    out2 = ops.gemm(A, hi, lo, bias=Bb, residual=Rr, relu=True, m_dev=m_dev)
    assert torch.equal(out[:M], out2[:M])
    c, stats = ops.gemm_instats(A, hi, lo, offs, 2, m_dev=m_dev)
    assert np.abs(N_(c)[:M] - c64).max() <= tol
    st = N_(stats)
    for ci, (s0, s1) in enumerate(((0, lens[0]), (lens[0], M))):
        blk = c64[s0:s1]
        np.testing.assert_allclose(st[ci, :, 0], blk.mean(0), rtol=0, atol=2e-6 * max(1.0, np.abs(c64).max()))
        np.testing.assert_allclose(st[ci, :, 1], 1.0 / np.sqrt(blk.var(0) + 1e-5), rtol=2e-5, atol=0)


# ------------------------------------------------- N1 + N2 through the GPU once (SURVEY.md 8f)

def test_benchmark_loop_on_real_sample_pairs_through_graph_executor(tmp_path):
    """The reference's test loop (generic_reg_model.py:130-183 -> benchmark_predator.py:285-375) on the two shipped
    sample pairs that belong to the 3DMatch benchmark: `ThreeDMatchPairs` (files as the dataset stores them:
    float64 .pth) -> `PairStream` (pinned read-ahead) -> `GraphedRegTR` -> `EstLogWriter` -> `benchmark_3dmatch`
    against their real gt.log / gt.info entries.  Random weights: the recall is meaningless, but the est.log
    must parse, hold the eager forward's poses and be scored; loader throughput is printed beside the model's."""
    import json
    import os
    import pickle
    import time
    from conftest import GOLDEN
    from regtr_b200 import data as D, eval as E
    from regtr_b200.config import get_config
    from regtr_b200.regtr import GraphedRegTR, RegTR
    from regtr_b200.weights import random_state_dict
    rows = json.load(open(os.path.join(GOLDEN, 'real', 'test_3DMatch_info_rows.json')))
    infos = dict(rot=[], trans=[], src=[], tgt=[], overlap=[])
    for r in rows:                                   # rebuild the on-disk layout: data/indoor/test/<scene>/cloud_bin_<i>.pth
        inp = np.load(os.path.join(GOLDEN, 'real', r['fixture'] + '_input.npz'))
        for rel in (r['src'], r['tgt']):
            which = 'src_xyz' if os.path.basename(rel) == os.path.basename(str(inp['src_file'])) else 'tgt_xyz'
            path = tmp_path / 'indoor' / rel
            os.makedirs(path.parent, exist_ok=True)
            torch.save(inp[which].astype(np.float64), path)
        infos['rot'].append(np.array(r['rot'])); infos['trans'].append(np.array(r['trans']))
        infos['src'].append(r['src']); infos['tgt'].append(r['tgt']); infos['overlap'].append(r['overlap'])
    with open(tmp_path / 'info.pkl', 'wb') as f:
        pickle.dump(infos, f)
    ds = D.ThreeDMatchPairs(str(tmp_path / 'indoor'), str(tmp_path / 'info.pkl'), pin=True)
    assert len(ds) == 2
    cfg = get_config('3dmatch')
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(random_state_dict(cfg, 41), strict=True)
    runner = GraphedRegTR(model)
    gt_dir = os.path.join(GOLDEN, 'real', 'benchmarks', '3DMatch')
    t0 = time.perf_counter()
    res = E.run_3dmatch_benchmark(D.PairStream(ds, [[0], [1]], workers=2), lambda b: runner(b), str(tmp_path / 'log'),
                                  '3DMatch', gt_dir)
    torch.cuda.synchronize()
    t_all = time.perf_counter() - t0
    t0 = time.perf_counter()
    n_loaded = sum(1 for _ in D.PairStream(ds, [[0], [1]] * 8, workers=4))
    t_load = time.perf_counter() - t0
    print(f'loader {n_loaded / t_load:.0f} pairs/s (pinned, 4 threads); loop incl. graph capture {t_all:.2f} s')
    assert set(res['per_scene']) == {'7-scenes-redkitchen', 'sun3d-hotel_umd-maryland_hotel3'}
    assert 'Mean median RRE' in res['summary'] and (np.isnan(res['recall']) or 0.0 <= res['recall'] <= 1.0)   # random weights
    assert 'reg_success_final' in res['metrics']
    for k, r in enumerate(rows):                     # est.log holds the eager forward's final-layer pose of each pair
        scene = r['src'].split('/')[1]
        pairs, traj = E.read_trajectory(os.path.join(str(tmp_path / 'log'), '3DMatch', scene, 'est.log'))
        assert len(pairs) == 1 and traj.shape == (1, 4, 4)
        item = ds[k]
        want = model({'src_xyz': [item['src_xyz'].to(DEV)], 'tgt_xyz': [item['tgt_xyz'].to(DEV)]})['pose'][-1, 0].cpu().numpy()
        assert np.abs(traj[0, :3] - want).max() <= 5e-5
        assert np.allclose(traj[0, 3], [0, 0, 0, 1])


# ------------------------------------------------- fp32-accurate wgmma attention core (3xTF32, TMA-fed, P in registers)

@pytest.mark.parametrize('lens', [[410, 339], [130, 7, 300, 129], [64, 64], [1, 200, 65, 3]])
def test_tf32_tcgen05_attention_block_vs_float64(lens):
    """Split-epilogue in-projection + regtr_mha_tf32_tc_fwd on ragged self and cross problems (unaligned key ranges,
    partial tiles, 1- and 3-token clouds) against a float64 in-projection + softmax attention: fp32-accurate."""
    from regtr_b200 import ops
    from regtr_b200.transformer import AttentionPlan
    rng = np.random.default_rng(sum(lens))
    E, H = 256, 8
    n = sum(lens)
    x = (rng.normal(size=(n, E)) * 0.8).astype(np.float32)
    W = (rng.normal(size=(3 * E, E)) / np.sqrt(E) * 1.5).astype(np.float32)
    b = (rng.normal(size=3 * E) * 0.1).astype(np.float32)
    plan = AttentionPlan(lens, DEV)
    qkv = x.astype(np.float64) @ W.astype(np.float64).T + b
    q64, k64, v64 = qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:]
    starts = np.concatenate([[0], np.cumsum(lens)])
    B = len(lens) // 2
    for cross in (False, True):
        ks, kl = (plan.xk_start, plan.xk_len) if cross else (plan.q_start, plan.q_len)
        ref = np.zeros((n, E))
        for c in range(len(lens)):
            o = (c + B if c < B else c - B) if cross else c
            qq = q64[starts[c]:starts[c + 1]].reshape(-1, H, 32).transpose(1, 0, 2)
            kk = k64[starts[o]:starts[o + 1]].reshape(-1, H, 32).transpose(1, 0, 2)
            vv = v64[starts[o]:starts[o + 1]].reshape(-1, H, 32).transpose(1, 0, 2)
            sc = qq @ kk.transpose(0, 2, 1) / np.sqrt(32)
            w = np.exp(sc - sc.max(-1, keepdims=True)); w /= w.sum(-1, keepdims=True)
            ref[starts[c]:starts[c + 1]] = (w @ vv).transpose(1, 0, 2).reshape(-1, E)
        got = N(ops.mha_tf32_tc(G(x), G(W), G(b), plan.q_start, plan.q_len, ks, kl, plan.max_len, H))
        assert np.isfinite(got).all()
        assert np.abs(got - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max()), (cross, np.abs(got - ref).max())
        dplan = AttentionPlan.from_device(ops.make_offsets(lens, DEV), B, n + 300)    # linear 128-query tile table
        ks2, kl2 = (dplan.xk_start, dplan.xk_len) if cross else (dplan.q_start, dplan.q_len)
        lin = N(ops.mha_tf32_tc(G(x), G(W), G(b), dplan.q_start, dplan.q_len, ks2, kl2, dplan.max_len, H,
                                tiles=dplan.tiles128))
        assert np.array_equal(lin, got)


def test_forward_with_tf32_tcgen05_attention_vs_reference_golden():
    """Full forward with attention_impl='tf32_tc' (both MHA contractions on wgmma, fed by TMA) against the
    unmodified reference: features 1e-4, pose 1e-4 -- the parity mode on the tensor cores."""
    case = 'fwd_3dmatch_small_b2'
    cfg, sd, src, tgt = make_case(case)
    cfg.attention_impl = 'tf32_tc'
    out, meta = _run_model(cfg, sd, src, tgt)
    check_forward_against_golden(out, meta, load_golden(case), len(src), feat_rtol=1e-4, corr_atol=1e-4,
                                 logit_atol=2e-4, pose_atol=1e-4)
    # and capacity-shaped inside a CUDA graph
    from regtr_b200.regtr import GraphedRegTR, RegTR
    model = RegTR(cfg).to(DEV).eval()
    model.load_state_dict(sd, strict=True)
    runner = GraphedRegTR(model, bucket=16384)
    batch = {'src_xyz': [G(a) for a in src], 'tgt_xyz': [G(a) for a in tgt]}
    got = runner(batch)
    assert runner.fallbacks == 0
    assert float((got['pose'] - out['pose']).abs().max()) <= 5e-5


# ------------------------------------------------- voxel sub-sampling without a library sort

def test_scan_state_is_clean_across_differently_sized_calls():
    """The prefix-sum state is laid out per call (tile count): sizes alternate on ONE stream and every call must still
    equal the oracle -- stale aggregates of a previous layout once aliased counters / flags of the next."""
    from oracle import pre
    from regtr_b200 import ops
    rng = np.random.default_rng(11)
    cases = [[42000, 40000], [700, 900], [9000, 11000], [38000, 37000], [300], [20000, 100], [42000, 40000]]
    for lens in cases * 2:
        n = sum(lens)                                            # extents inside the dense-grid cell budget
        pts = _pre_inputs(n + int(rng.integers(1, 1000)), lens, scale=0.6 if n < 5000 else (1.0 if n < 30000 else 2.0))
        offs = ops.make_offsets(lens, DEV)
        status = ops.new_status(DEV)
        sub, so = ops.grid_subsample(G(pts), offs, len(lens), 0.05, status)
        assert int(status.item()) == 0
        want_sub, want_len = pre.grid_subsample(pts, lens, 0.05)
        assert np.array_equal(np.diff(N(so)), want_len) and np.array_equal(N(sub)[:int(so[-1])], want_sub)
        # cell list + radius search over the sub-sampled level (the scan of the cell list has its own state)
        grid = ops.CellGrid(sub, so, len(lens), 0.125, status)
        i32, _ = ops.ball_query(sub, so, sub, so, grid, 20, 0.125, want64=False)
        want_idx = pre.ball_query(want_sub, want_len, want_sub, want_len, 20, 0.125)
        assert int(status.item()) == 0
        assert np.array_equal(N(i32)[:len(want_sub)], want_idx)


def test_dense_grid_subsample_equals_sorted_variant_and_falls_back_when_sparse():
    """The dense-grid counting sort (hand-written kernels, own single-pass prefix sum) and the sort-based variant
    give bit-identical barycentres and offsets; a cloud whose bounding box exceeds the cell budget raises
    REGTR_STATUS_GRID, and the pre-processor then takes the sort-based path on its own (same result as the oracle)."""
    from oracle import pre
    from regtr_b200 import ops
    from regtr_b200.config import get_config
    from regtr_b200.kpconv import PreprocessorGPU
    for lens in ([900, 1100], [1, 2000, 0, 37], [30000, 28000]):
        pts = _pre_inputs(sum(lens) + 1, lens, scale=0.6 if sum(lens) < 5000 else 1.5)
        offs = ops.make_offsets(lens, DEV)
        out = []
        for dense in (True, True, False):                       # twice dense: the self-cleaning state is reused
            status = ops.new_status(DEV)
            sub, so = ops.grid_subsample(G(pts), offs, len(lens), 0.05, status, dense=dense)
            assert int(status.item()) == 0
            out.append((N(sub)[:int(so[-1])], N(so)))
        for a in out[1:]:
            assert np.array_equal(out[0][0], a[0]) and np.array_equal(out[0][1], a[1])
        want_sub, want_len = pre.grid_subsample(pts, lens, 0.05)
        assert np.array_equal(out[0][0], want_sub) and np.array_equal(np.diff(out[0][1]), want_len)
    # sparse: 3000 points over a 120 m cube at 5 cm voxels -> 1.4e10 cells
    rng = np.random.default_rng(4)
    sparse = rng.uniform(-60, 60, size=(3000, 3)).astype(np.float32)
    status = ops.new_status(DEV)
    ops.grid_subsample(G(sparse), ops.make_offsets([3000], DEV), 1, 0.05, status)
    assert int(status.item()) & 4
    sub2, so2 = ops.grid_subsample(G(pts), offs, len(lens), 0.05, ops.new_status(DEV))      # state still clean afterwards
    assert np.array_equal(N(sub2)[:int(so2[-1])], out[0][0])
    cfg = get_config('3dmatch')
    big = (rng.uniform(-40, 40, size=(4000, 3))).astype(np.float32)
    big[:2000] = rng.uniform(-1, 1, size=(2000, 3))             # a dense core so that the pyramid is not trivial
    meta = PreprocessorGPU(cfg)([G(big[:2500]), G(big[2500:])])
    want = pre.preprocess(cfg, [big[:2500], big[2500:]])
    for key in ('points', 'neighbors', 'pools', 'stack_lengths'):
        for lvl, (a, b) in enumerate(zip(meta[key], want[key])):
            assert np.array_equal(N(a), b), f'{key}[{lvl}]'
