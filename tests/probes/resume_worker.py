"""Worker of tests/test_resume_gpu.py: runs training command lines one after another in this one process, each through its script's
main() with the flags reset, so a batch of runs pays the interpreter, torch and CUDA start-up once.  Each job is [script, args, out]: the
script's stdout goes to `out`, and a SystemExit (a usage error) is written there as a last line 'EXIT <message>'.
Usage: python resume_worker.py jobs.json"""
import contextlib
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
# all three scripts are imported before any job runs, so that every job sees the same set of defined flags
import pretrain_recover  # noqa: E402
import train  # noqa: E402
import train_flow  # noqa: E402
from unsupervised_detection_b200.common_flags import FLAGS  # noqa: E402

SCRIPTS = {'train.py': train, 'pretrain_recover.py': pretrain_recover, 'train_flow.py': train_flow}


def main():
    for script, args, out in json.load(open(sys.argv[1])):
        FLAGS.unparse_flags()
        with open(out, 'w') as f, contextlib.redirect_stdout(f):
            try:
                SCRIPTS[script].main([script] + args)
            except SystemExit as e:
                print('EXIT %s' % (e.code,))
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
