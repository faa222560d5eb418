"""Worker of tests/test_ema_gpu.py's two-rank test (launched with torch.distributed.run, one rank per GPU): trains a few alternating
steps with a moving average of the weights on this rank's shard of a fixed global batch, with the NCCL all-reduce of AdversarialLearner,
then saves its parameters and their averages."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
from unsupervised_detection_b200.step_graph import CISGraph  # noqa: E402


def main():
    out = sys.argv[1]
    rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
    torch.cuda.set_device(local)
    dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    blob = torch.load(os.path.join(out, 'inputs.pt'))
    GB, H, W, ph, pw = blob['GB'], blob['H'], blob['W'], blob['ph'], blob['pw']
    b = GB // world
    g = CISGraph(H, W, b, device='cuda:%d' % local, global_batch=GB, with_pwc=True, pwc_hw=(ph, pw), ema_decay=blob['decay'])
    g.load_params(blob['params'])
    sl = slice(rank * b, (rank + 1) * b)
    g.img1.copy_(blob['img1'][sl])
    g.img2.copy_(blob['img2'][sl])
    ar = lambda t: dist.all_reduce(t)
    for mode in blob['modes']:
        g.train_step(mode, allreduce=ar, use_graph=True)
    torch.cuda.synchronize()
    torch.save({k: v.cpu() for k, v in g.export_params().items() if not k.startswith('pwcnet')}, os.path.join(out, 'rank%d.pt' % rank))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
