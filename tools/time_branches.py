"""Developer tool: GPU time of the two branches of the pipelined step on their own (CUDA-graph replays, events on the launching stream)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from unsupervised_detection_b200.common_flags import Config
from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner

L = AdversarialLearner()
L.config = Config(img_height=256, img_width=448, batch_size=4, dataset='SYNTHETIC', flow_ckpt='synthetic', summary_freq=10 ** 9)
L.build_train_graph()
b = L.reader.batch(4)
L.feed(b[0], b[1])
g = L.graph
for m in 'GR':
    g.train_step(m, use_graph=True, pipeline=True)
torch.cuda.synchronize()


def t(fn, reps=10):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


G = g.graphs
print('flow network (PWC-Net 384x640 + resizes) alone      : %.3f ms' % t(G['pipe_pwc'].replay))
for m in 'RG':
    print('train branch %s (generator+recover fwd, loss, bwd) : %.3f ms' % (m, t(G['pipe_rest_' + m].replay)))
    print('optimiser + re-pack %s                              : %.3f ms' % (m, t(G['pipe_adam_' + m].replay)))
for m in 'RG':
    print('pipelined step %s                                   : %.3f ms' % (m, t(lambda: g.train_step(m, use_graph=True, pipeline=True))))
    print('sequential step %s                                  : %.3f ms' % (m, t(lambda: g.train_step(m, use_graph=True))))

# ---- where the train branch spends its time: forward, backward main lane (data gradients) and side lane (weight gradients) on their own
from unsupervised_detection_b200.engine import Plan


def sub(plan, keep):
    q = Plan(plan.name + '.sub')
    q.ops = [op for op in plan.ops if keep(op)]
    q.keep = plan.keep
    return q


print('train branch forward only                          : %.3f ms' % t(g._capture_plans('tb_fwd', [g._pipe_rest]).replay))
for m in 'RG':
    bw = g.bwd[m]
    both = g._capture_plans('tb_bwd_' + m, [bw])
    main = g._capture_plans('tb_bwd_main_' + m, [sub(bw, lambda op: op[4] == 0)])
    side = g._capture_plans('tb_bwd_side_' + m, [sub(bw, lambda op: op[4] == 1 or op[0] is None)])
    print('backward %s: both lanes %.3f ms | main lane alone %.3f ms | side lane alone %.3f ms' % (m, t(both.replay), t(main.replay), t(side.replay)))
