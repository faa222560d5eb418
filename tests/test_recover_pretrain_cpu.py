"""Recover-net pretraining on box-shaped occlusions, host side: the box draw of cis_box_masks restated in Python integers, the launch plans of
a CISGraph(masks='boxes'), the pretraining loop with the GPU parts stubbed, the recover-only checkpoint and the flags of pretrain_recover.py.
box_draw / box_masks below are also the reference of the GPU test (test_recover_pretrain_gpu.py)."""
import os

import numpy as np
import pytest
import torch

from unsupervised_detection_b200.common_flags import FLAG_NAMES, Config
from unsupervised_detection_b200.step_graph import CISGraph, box_sides

M64 = (1 << 64) - 1
BOX_DOMAIN = 0x426f784d61736b73


def hash32(x):
    """64-bit MurmurHash3 finaliser, truncated to 32 bits (the counter hash of csrc/misc_kernels.cu)."""
    x &= M64
    x ^= x >> 33
    x = (x * 0xff51afd7ed558ccd) & M64
    x ^= x >> 33
    x = (x * 0xc4ceb9fe1a85ec53) & M64
    x ^= x >> 33
    return x & 0xffffffff


def box_draw(seed, t, g, box, H, W):
    """Box of global sample g at Adam step t -> (y0, x0, bh, bw), as cis_box_masks draws it."""
    lo_h, hi_h, lo_w, hi_w = box
    r = [hash32(seed ^ BOX_DOMAIN ^ ((t << 40) & M64) ^ ((g << 2) & M64) ^ k) for k in range(4)]
    bh = lo_h + r[0] % (hi_h - lo_h + 1)
    bw = lo_w + r[1] % (hi_w - lo_w + 1)
    return r[2] % (H - bh + 1), r[3] % (W - bw + 1), bh, bw


def box_masks(seed, t, sample_offset, B, box, H, W):
    """fp32 [B,H,W,1]: 1 inside sample (sample_offset + b)'s box."""
    m = torch.zeros(B, H, W, 1)
    for b in range(B):
        y0, x0, bh, bw = box_draw(seed, t, sample_offset + b, box, H, W)
        m[b, y0:y0 + bh, x0:x0 + bw] = 1.0
    return m


def test_box_draws_stay_inside_the_image_with_sides_in_range():
    seen_h, seen_w = set(), set()
    for H, W in ((37, 53), (256, 448), (5, 3)):
        box = box_sides(0.1, 0.5, H, W)
        for seed in (8964, 0, 2 ** 63 + 5):
            for t in (0, 1, 7, 12345):
                for g in range(20):
                    y0, x0, bh, bw = box_draw(seed, t, g, box, H, W)
                    assert box[0] <= bh <= box[1] and box[2] <= bw <= box[3]
                    assert 0 <= y0 and y0 + bh <= H and 0 <= x0 and x0 + bw <= W
                    if (H, W) == (256, 448):
                        seen_h.add(bh)
                        seen_w.add(bw)
    # 240 draws over 103 heights / 180 widths: most of the range is hit
    assert min(seen_h) < 40 and max(seen_h) > 110 and min(seen_w) < 70 and max(seen_w) > 200


def test_box_draws_change_with_step_and_sample():
    box = box_sides(0.1, 0.5, 256, 448)
    draws = {box_draw(8964, t, g, box, 256, 448) for t in range(8) for g in range(8)}
    assert len(draws) == 64
    m = box_masks(8964, 3, 0, 4, box, 256, 448)
    assert set(m.unique().tolist()) <= {0.0, 1.0}
    for b in range(4):
        y0, x0, bh, bw = box_draw(8964, 3, b, box, 256, 448)
        assert int(m[b].sum()) == bh * bw


def test_rank_local_draws_equal_the_global_batch_draws():
    box = box_sides(0.1, 0.5, 37, 53)
    GB, world = 8, 4
    full = box_masks(77, 5, 0, GB, box, 37, 53)
    B = GB // world
    for r in range(world):
        assert torch.equal(box_masks(77, 5, r * B, B, box, 37, 53), full[r * B:(r + 1) * B])
    assert not torch.equal(full[:B], full[B:2 * B])          # ranks do not repeat each other's boxes


def test_box_sides_from_fractions():
    assert box_sides(0.1, 0.5, 256, 448) == (25, 128, 44, 224)
    assert box_sides(0.001, 0.002, 64, 96) == (1, 1, 1, 1)           # lo >= 1, hi >= lo
    assert box_sides(1.0, 1.0, 37, 53) == (37, 37, 53, 53)
    for bad in ((0.0, 0.5), (0.6, 0.5), (0.1, 1.5), (-0.1, 0.2)):
        with pytest.raises(ValueError):
            box_sides(bad[0], bad[1], 64, 96)


# ------------------------------------------------------------------------------------------------ the boxes graph
@pytest.fixture(scope='module')
def boxes_graph():
    return CISGraph(64, 96, 2, device='cpu', masks='boxes', pwc_hw=(128, 192), box=(6, 32, 9, 48), sample_offset=4)


def test_boxes_graph_forward_has_no_generator(boxes_graph):
    g = boxes_graph
    names = [op[2] for op in g.fwd.ops]
    assert 'cis_flow_stats' not in names and 'cis_pack_generator_input' not in names and 'cis_mask_bwd' not in names
    gen_layers = {id(L) for L in g.gen.all_layers()}
    convs = [op for op in g.fwd.ops if op[2] == 'cis_conv_igemm']
    assert len(convs) > 0
    # no generator layer was ever placed: their forward operands were never set up
    assert all(L.fwd_pack is None for L in g.gen.all_layers()) and len(gen_layers) == 17
    assert g.pack_gen.ops == []
    assert names.count('cis_box_masks') == 1 and names.count('cis_mask_apply') == 1


def test_box_kernel_runs_in_the_main_lane_part_of_the_forward(boxes_graph):
    g = boxes_graph
    names = [op[2] for op in g.fwd.ops]
    i = names.index('cis_box_masks')
    assert g._pwc_ops > 0 and names[g._pwc_ops] == 'take_stage'
    assert i > g._pwc_ops and g.fwd.ops[i][4] == 0
    assert i < names.index('cis_mask_apply')
    args = g.fwd.ops[i][1]
    assert args[0] == g.mask.data_ptr() and args[1:8] == (2, 64, 96, 6, 32, 9, 48)
    assert args[8] == 4 and args[9] == g.step_state.data_ptr() and args[10] == g.seed
    # the pipelined schedule: the side-stream prefix never contains it, the main-lane rest does
    assert 'cis_box_masks' not in names[:g._pwc_ops]


def test_boxes_graph_trains_the_recover_net_only(boxes_graph):
    g = boxes_graph
    assert sorted(g.bwd) == ['R'] and sorted(g.adam) == ['R']
    adam = [op for op in g.adam['R'].ops if op[2] == 'cis_clip_adam']
    assert len(adam) == 1 and adam[0][1][13] == 0                       # can_change = 0
    assert adam[0][1][0] == g.rec_store.flat.data_ptr()
    assert 'cis_grad_avg_abs' not in [op[2] for op in g.adam['R'].ops]
    assert [op[2] for op in g.bwd['R'].ops][0] == 'cis_cis_loss_bwd' and g.bwd['R'].ops[0][1][11] == 0   # d recover_loss
    with pytest.raises(ValueError):
        g.train_step('G')


def test_boxes_graph_without_pwc_and_bad_arguments():
    g = CISGraph(32, 48, 1, device='cpu', masks='boxes', with_pwc=False)
    names = [op[2] for op in g.fwd.ops]
    assert g._pwc_ops == 0 and names.index('cis_box_masks') > 0 and g.box == box_sides(0.1, 0.5, 32, 48)
    with pytest.raises(ValueError):
        CISGraph(32, 48, 1, device='cpu', masks='box', with_pwc=False)
    with pytest.raises(ValueError):
        CISGraph(32, 48, 1, device='cpu', masks='boxes', with_pwc=False, box=(4, 40, 4, 8))       # hi_h > H
    with pytest.raises(ValueError):
        CISGraph(32, 48, 1, device='cpu', masks='boxes', with_pwc=False, box=(0, 4, 4, 8))        # lo < 1


def test_generator_graph_keeps_both_steps():
    g = CISGraph(32, 48, 1, device='cpu', with_pwc=False)
    names = [op[2] for op in g.fwd.ops]
    assert 'cis_box_masks' not in names and 'cis_flow_stats' in names and sorted(g.bwd) == ['G', 'R']


# ------------------------------------------------------------------------------------------------ loop, checkpoint, flags
def test_pretrain_loop_control_flow_on_cpu(capsys, tmp_path):
    """AdversarialLearner.pretrain_recover with the GPU parts stubbed: every batch is consumed once and in order, the next batch is
    handed over for the overlapped upload, epochs end after num_samples_train/batch_size steps, recover-<epoch> is saved every
    save_freq epochs and after the last one, and the loss scalars go to the console and the event file every summary_freq steps."""
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    from unsupervised_detection_b200.summary import read_events

    class Reader(object):
        def __init__(self):
            self.n = 0

        def batch(self, b):
            self.n += 1
            return ('img1_%d' % self.n, 'img2_%d' % self.n, None, [])

    class Store(object):
        def real_count(self):
            return 77

    class Graph(object):
        box = (1, 2, 3, 4)
        rec_store = Store()

    class Stub(AdversarialLearner):
        def build_pretrain_graph(self):
            self.rank, self.world, self.local_batch = 0, 1, 2
            self.reader, self.graph = Reader(), Graph()
            self.train_steps_per_epoch = 3
            self.calls, self.saved = [], []

        def pretrain_step(self, batch, next_batch=None, fetch_losses=False, use_graph=True):
            self.global_step += 1
            self.calls.append((batch[0], next_batch[0], fetch_losses))
            r = {'global_step': self.global_step}
            if fetch_losses:
                r.update(loss_recover=1.5, reconstruction_loss=2.5, reconstruction_compl_loss=3.5)
            return r

        def save_recover(self, checkpoint_dir, epoch):
            self.saved.append((checkpoint_dir, epoch, len(self.calls)))

    L = Stub()
    L.pretrain_recover(Config(max_epochs=5, save_freq=2, summary_freq=4, checkpoint_dir=str(tmp_path)))
    assert [c[0] for c in L.calls] == ['img1_%d' % i for i in range(1, 16)]           # 5 epochs x 3 steps, each batch once, in order
    assert [c[1] for c in L.calls] == ['img1_%d' % i for i in range(2, 17)]
    assert [i + 1 for i, c in enumerate(L.calls) if c[2]] == [4, 8, 12]
    assert L.saved == [(str(tmp_path), 2, 6), (str(tmp_path), 4, 12), (str(tmp_path), 5, 15)]
    out = capsys.readouterr().out
    assert 'Pretraining completed successfully' in out and out.count('loss_recover') == 3 and 'Number of recover params: 77' in out
    L.summary_writer.close()
    ev = read_events(L.summary_writer.path)[1:]
    assert [e['step'] for e in ev] == [4, 8, 12]
    assert [(v['tag'], v['simple_value']) for v in ev[0]['values']] == [('recover', 1.5), ('reconstruction_loss', 2.5),
                                                                         ('reconstruction_compl_loss', 3.5)]


def test_recover_checkpoint_holds_exactly_the_flownets_variables(tmp_path):
    from unsupervised_detection_b200 import checkpoint as ckpt_io, params_init
    from unsupervised_detection_b200.models.adversarial_learner import AdversarialLearner
    g = CISGraph(32, 48, 1, device='cpu', masks='boxes', with_pwc=False)
    p = params_init.init_generator()
    p.update(params_init.init_recover())
    g.load_params(p)
    L = AdversarialLearner()
    L.rank, L.graph, L.global_step = 0, g, 17
    L.save_recover(str(tmp_path), 3)
    prefix = str(tmp_path / 'recover-3')
    rec = L._names('FlownetS')
    assert sorted(v[0] for v in ckpt_io.list_variables(prefix)) == sorted(ckpt_io.to_tf_name(n) for n in rec)
    assert ckpt_io.latest_checkpoint(str(tmp_path)) == prefix
    for path in (prefix, prefix + '.pt'):
        got, gs = AdversarialLearner._read_ckpt(path, rec)
        assert sorted(got) == sorted(rec)
        for n in rec:
            assert torch.equal(got[n].reshape(-1), p[n].reshape(-1).float()), n
        with pytest.raises(KeyError):
            AdversarialLearner._read_ckpt(path, L._names('MaskNet'))
    assert AdversarialLearner._read_ckpt(prefix, rec)[1] is None                         # recover_saver stores no global_step
    assert torch.load(prefix + '.pt')['global_step'] == 17


def test_pretrain_flags(monkeypatch, tmp_path):
    import pretrain_recover as PR
    from unsupervised_detection_b200.common_flags import FLAGS
    assert len(FLAG_NAMES) == 31 and 'box_min' not in FLAG_NAMES and 'box_max' not in FLAG_NAMES
    assert FLAGS['box_min'].default == 0.1 and FLAGS['box_max'].default == 0.5
    seen = []
    monkeypatch.setattr(PR, 'run', lambda cfg: seen.append((cfg.box_min, cfg.box_max, cfg.dataset)))
    ck = '--checkpoint_dir=%s' % tmp_path

    def main(*args):
        FLAGS.unparse_flags()              # every call parses from the defaults, as a fresh process would
        PR.main(['pretrain_recover.py'] + list(args))
    try:
        main('--dataset=SYNTHETIC', ck)
        main('--box_min=0.25', '--box_max=0.25', ck)
        assert seen == [(0.1, 0.5, 'SYNTHETIC'), (0.25, 0.25, 'DAVIS2016')]
        for bad in (['--box_min=0', '--box_max=0.5'], ['--box_min=0.6', '--box_max=0.5'], ['--box_max=1.5'], ['--box_min=-0.2']):
            with pytest.raises(SystemExit):
                main(ck, *bad)
        with pytest.raises(SystemExit):
            main()                         # no --checkpoint_dir
        with pytest.raises(SystemExit):
            main('--no_such_flag=1', ck)
    finally:
        FLAGS.unparse_flags()
    assert len(seen) == 2 and len(FLAG_NAMES) == 31


def test_box_rule_matches_a_numpy_restatement():
    """The integer draw does not depend on Python's big integers: the same arithmetic in numpy uint64 gives the same boxes."""
    box = box_sides(0.1, 0.5, 256, 448)
    for seed, t, g in ((8964, 0, 0), (8964, 9, 5), (1, 2 ** 20, 3000)):
        ks = []
        for k in range(4):
            with np.errstate(over='ignore'):
                x = np.uint64(seed) ^ np.uint64(BOX_DOMAIN) ^ (np.uint64(t) << np.uint64(40)) ^ (np.uint64(g) << np.uint64(2)) ^ np.uint64(k)
                x ^= x >> np.uint64(33)
                x *= np.uint64(0xff51afd7ed558ccd)
                x ^= x >> np.uint64(33)
                x *= np.uint64(0xc4ceb9fe1a85ec53)
                x ^= x >> np.uint64(33)
            ks.append(int(x & np.uint64(0xffffffff)))
        bh, bw = box[0] + ks[0] % (box[1] - box[0] + 1), box[2] + ks[1] % (box[3] - box[2] + 1)
        assert box_draw(seed, t, g, box, 256, 448) == (ks[2] % (256 - bh + 1), ks[3] % (448 - bw + 1), bh, bw)
