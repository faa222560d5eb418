"""The learner-level step schedule on the GPU, as train.py, pretrain_recover.py and bench.py's end-to-end arm drive it:
step(batch, next_batch=...) mixes pipelined steps (the flow network of the next batch on a second stream, its upload on the copy stream),
summary steps (sequential, with the summary pre-pass) and batches prefetched into a staging slot and handed over on the device.  Whatever
the schedule, every step must train on its own frame pair, so the pipelined schedule, the sequential one (CIS_PIPELINE=0) and eager
launches without CUDA graphs end with bit-identical parameters and losses.  The same holds for pretrain_step."""
import pytest
import torch

from unsupervised_detection_b200.common_flags import Config
from unsupervised_detection_b200.data.synthetic import SyntheticReader
from unsupervised_detection_b200.models import adversarial_learner as AL

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

STEPS = 9        # summary_freq 3: steps 3, 6 and 9 take the sequential summary path between pipelined steps; steps 4 and 8 train the recover net


@pytest.fixture(scope='module')
def batches():
    rd = SyntheticReader(seed=5)
    return [rd.batch(2) for _ in range(STEPS + 1)]


def _run(monkeypatch, batches, pretrain, pipeline, use_graph):
    monkeypatch.setattr(AL, 'PIPELINE', pipeline)
    L = AL.AdversarialLearner()
    L.config = Config(img_height=64, img_width=96, batch_size=2, dataset='SYNTHETIC', flow_ckpt='synthetic', summary_freq=3)
    if pretrain:
        L.build_pretrain_graph()
    else:
        L.build_train_graph()
    g = L.graph
    start = {k: v.cpu() for k, v in g.export_params().items()}
    results = []
    for t in range(STEPS):
        if pretrain:
            results.append(L.pretrain_step(batches[t], next_batch=batches[t + 1], fetch_losses=True, use_graph=use_graph))
        else:
            results.append(L.step(batches[t], fetch_losses=True, use_graph=use_graph, next_batch=batches[t + 1], summarize=True))
    g.pipeline_drain()
    torch.cuda.synchronize()
    params = {k: v.cpu() for k, v in g.export_params().items()}
    assert ('pipe_pwc' in g.graphs) == (pipeline and use_graph)
    assert any(not torch.equal(params[k], start[k]) for k in start if k.startswith('FlownetS/'))
    return params, results


@pytest.mark.parametrize('pretrain', [False, True], ids=['step', 'pretrain_step'])
def test_pipelined_sequential_and_eager_schedules_are_bit_identical(monkeypatch, batches, pretrain):
    runs = [_run(monkeypatch, batches, pretrain, pipeline, use_graph) for pipeline, use_graph in ((True, True), (False, True), (True, False))]
    assert len(runs[0][1]) == STEPS and all('loss_recover' in r for r in runs[0][1])
    for params, results in runs[1:]:
        assert results == runs[0][1], (results, runs[0][1])
        diff = [k for k in params if not torch.equal(params[k], runs[0][0][k])]
        assert not diff, diff[:5]
