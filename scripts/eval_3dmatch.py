"""3DMatch / 3DLoMatch registration recall of a checkpoint on the CUDA path (the reference's `test.py`):

    python scripts/eval_3dmatch.py --root <data/indoor> --info <test_3DMatch_info.pkl> \
        --gt <datasets/3dmatch/benchmarks/3DMatch> --ckpt <model.pth> --out logs/3DMatch [--icp R [--icp_iters N]
        [--icp_method point_to_plane|generalized [--normal_radius NR] [--normal_max_nn 30] [--icp_epsilon 1e-3]
        [--icp_loss l2|huber|cauchy|gm|tukey --icp_loss_k K]
        [--icp_voxels V1,V2,... [--icp_radii R1,...] [--icp_level_iters I1,...]]]]
        [--ransac R [--ransac_iters 100000] [--ransac_confidence 0.999] [--ransac_n 3] [--ransac_edge 0.9]
         [--ransac_dist D] [--ransac_overlap 0.5] [--ransac_seed 0]]
        [--fgr [--fgr_dist 0.025] [--fgr_iters 64] [--fgr_tuple_test] [--fgr_overlap 0.5] ...]
    python scripts/eval_3dmatch.py --root <data/indoor> --info <test_3DMatch_info.pkl> \
        --gt <datasets/3dmatch/benchmarks/3DMatch> --fpfh V [--fpfh_radius FR] [--fpfh_max_nn 100] [--fpfh_no_mutual]
        [--ransac R ... | --fgr [--fgr_dist D] [--fgr_no_tuple_test] ...] [--icp R ...] --out logs/3DMatch_fpfh

--icp R refines every final pose by ICP on the full clouds (`ops.icp`, max correspondence distance R; point-to-point,
or point-to-plane against target normals from `ops.estimate_normals` at NR, default 2 R, or generalized ICP on the
normals of both clouds, optionally under a robust loss; --icp_voxels runs multi-scale ICP over a voxel pyramid of the
clouds, `eval.icp_refine`'s voxels / radii / level_iters): est.log then holds the
refined poses, and the metrics report both (`rot_err_deg` / `trans_err` refined, `*_coarse` the network's).
--ransac R replaces every network pose by RANSAC over the network's correspondences with predicted overlap above
--ransac_overlap (`ops.ransac`, max correspondence distance R, validated on the full clouds); with --icp as well, ICP
starts from the RANSAC pose, and the metrics also report `*_ransac`.
--fgr replaces them by Fast Global Registration over the same correspondences instead (`ops.fgr`, --fgr_* options;
`*_fgr` with --icp).
--fpfh V (no --ckpt) scores the classical baseline instead of a network: `eval.fpfh_forward`, FPFH features of the
clouds downsampled at V matched in feature space, then RANSAC (radius --ransac, default 1.5 V), and ICP after it with
--icp (the metrics then also report `*_fpfh`); with --fgr, FGR over the mutual feature matches replaces RANSAC
(--fgr_dist defaulting to 0.5 V).
Needs the dataset and trained weights (neither is available offline: SURVEY.md 8f N1)."""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from regtr_b200 import data as D, eval as E
from regtr_b200.config import get_config
from regtr_b200.regtr import GraphedRegTR, RegTR


def parser():
    ap = argparse.ArgumentParser()
    ap.add_argument('--root', required=True); ap.add_argument('--info', required=True); ap.add_argument('--gt', required=True)
    ap.add_argument('--ckpt'); ap.add_argument('--out', default='logs'); ap.add_argument('--benchmark', default='3DMatch')
    ap.add_argument('--batch', type=int, default=1); ap.add_argument('--workers', type=int, default=4)
    E.add_icp_arguments(ap, 'Refine the poses by ICP with this max correspondence distance')
    E.add_ransac_arguments(ap, 'Replace the poses by RANSAC over the predicted correspondences, max correspondence '
                               'distance R (before ICP with --icp; with --fpfh 1.5 V)')
    E.add_fgr_arguments(ap, 'Replace the poses by Fast Global Registration over the predicted correspondences (with '
                            '--fpfh: over the FPFH matches) instead of RANSAC; before ICP with --icp')
    E.add_fpfh_arguments(ap)
    return ap


def network_forward(args):
    """The checkpoint's forward on the CUDA graph, with RANSAC or FGR and / or ICP after it as the flags ask."""
    dev = torch.device('cuda:0')
    cfg = get_config('3dmatch')
    model = RegTR(cfg).to(dev).eval()
    state = torch.load(args.ckpt, map_location='cpu')
    model.load_state_dict(state.get('state_dict', state), strict=False)      # torch_helpers.py:222
    runner = GraphedRegTR(model)
    if args.ransac is not None:
        return E.ransac_forward(lambda b: runner(b), args.ransac, **E.ransac_kwargs(args), icp_radius=args.icp,
                                icp_kwargs=E.icp_kwargs(args))
    if args.fgr:
        return E.fgr_forward(lambda b: runner(b), args.fgr_overlap, icp_radius=args.icp, icp_kwargs=E.icp_kwargs(args),
                             **E.fgr_kwargs(args))
    return (lambda b: runner(b)) if args.icp is None else E.icp_forward(
        lambda b: runner(b), args.icp, args.icp_iters, method=args.icp_method, normal_radius=args.normal_radius,
        normal_max_nn=args.normal_max_nn, epsilon=args.icp_epsilon, loss=args.icp_loss, loss_k=args.icp_loss_k,
        voxels=args.icp_voxels, radii=args.icp_radii, level_iters=args.icp_level_iters)


def main(argv=None):
    ap = parser()
    args = ap.parse_args(argv)
    E.check_fgr_arguments(ap, args)
    E.check_fpfh_arguments(ap, args)
    E.check_icp_arguments(ap, args)
    E.check_ransac_arguments(ap, args)
    ds = D.ThreeDMatchPairs(args.root, args.info, pin=True)
    batches = [list(range(i, min(i + args.batch, len(ds)))) for i in range(0, len(ds), args.batch)]
    if args.fpfh is not None:
        forward = E.fpfh_forward(args.fpfh, icp_radius=args.icp, icp_kwargs=E.icp_kwargs(args), **E.fpfh_kwargs(args))
    else:
        forward = network_forward(args)
    res = E.run_3dmatch_benchmark(D.PairStream(ds, batches, workers=args.workers), forward, args.out,
                                  args.benchmark, args.gt)
    print(res['summary']); print('registration recall', res['recall'])
    print({k: float(v) for k, v in res['metrics'].items() if not k.endswith('hist')})


if __name__ == '__main__':
    main()
