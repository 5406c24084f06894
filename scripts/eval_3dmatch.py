"""3DMatch / 3DLoMatch registration recall of a checkpoint on the CUDA path (the reference's `test.py`):

    python scripts/eval_3dmatch.py --root <data/indoor> --info <test_3DMatch_info.pkl> \
        --gt <datasets/3dmatch/benchmarks/3DMatch> --ckpt <model.pth> --out logs/3DMatch

Needs the dataset and trained weights (neither is available offline: SURVEY.md 8f N1)."""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from regtr_b200 import data as D, eval as E
from regtr_b200.config import get_config
from regtr_b200.regtr import GraphedRegTR, RegTR

ap = argparse.ArgumentParser()
ap.add_argument('--root', required=True); ap.add_argument('--info', required=True); ap.add_argument('--gt', required=True)
ap.add_argument('--ckpt', required=True); ap.add_argument('--out', default='logs'); ap.add_argument('--benchmark', default='3DMatch')
ap.add_argument('--batch', type=int, default=1); ap.add_argument('--workers', type=int, default=4)
args = ap.parse_args()
dev = torch.device('cuda:0')
cfg = get_config('3dmatch')
model = RegTR(cfg).to(dev).eval()
state = torch.load(args.ckpt, map_location='cpu')
model.load_state_dict(state.get('state_dict', state), strict=False)      # torch_helpers.py:222
runner = GraphedRegTR(model)
ds = D.ThreeDMatchPairs(args.root, args.info, pin=True)
batches = [list(range(i, min(i + args.batch, len(ds)))) for i in range(0, len(ds), args.batch)]
res = E.run_3dmatch_benchmark(D.PairStream(ds, batches, workers=args.workers), lambda b: runner(b), args.out,
                              args.benchmark, args.gt)
print(res['summary']); print('registration recall', res['recall'])
print({k: float(v) for k, v in res['metrics'].items() if not k.endswith('hist')})
