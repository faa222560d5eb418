"""Oracle restatement of models/utils/loss_utils.py, flow_utils.py:5-12 and the loss/step algebra of
models/adversarial_learner.py:72-258,376-409 (test infra only)."""
import math
import torch
from . import tf_ops as T
from .nets import generator_net, recover_net
from .pwcnet import predict_from_img_pairs


def preprocess_flow_batch(flow):
    """flow_utils.py:5-12: per-sample/channel zero-mean, unit population variance, NO epsilon."""
    mean = flow.mean(dim=(1, 2), keepdim=True)
    var = ((flow - mean) ** 2).mean(dim=(1, 2), keepdim=True)
    return (flow - mean) / torch.sqrt(var)


def charbonnier_loss(gt_flows, pred_flows, masks, cbn=0.5):
    """loss_utils.py:34-51 -> [B]."""
    lp = (gt_flows - pred_flows) ** 2 + 0.001 ** 2
    lp = torch.pow(lp, cbn) * masks
    return lp.sum(dim=(1, 2, 3))


def resize_inputs(image_384, flow_384, h, w, flow_normalizer=80.0):
    """adversarial_learner.py:87-97."""
    image = T.resize_bilinear_legacy(image_384, h, w)
    flow = T.resize_bilinear_legacy(flow_384, h, w) / flow_normalizer
    return image, flow


def adversarial_losses(image, flow, p, cbn=0.5, epsilon=75.0, global_batch=None):
    """adversarial_learner.py:99-204 given the resized image [B,H,W,3] and normalised flow [B,H,W,2].
    `global_batch` = config.batch_size used in num_pixels (defaults to the local batch)."""
    m = generator_net(image, preprocess_flow_batch(flow), p)          # :101-105
    mc = 1.0 - m                                                      # :107
    flow_masked = flow * (1.0 - m)                                    # :109
    flow_compl = flow * (1.0 - mc)                                    # :110
    pred = recover_net(image, flow_masked, m, p)                      # :114
    pred_c = recover_net(image, flow_compl, mc, p)                    # :120
    pred_i = recover_net(image, torch.zeros_like(flow), torch.ones_like(m), p)  # :127
    out = dict(masks=m, pred=pred, pred_c=pred_c, pred_i=pred_i)
    out.update(loss_head(flow, m, pred, pred_c, pred_i, cbn, epsilon, global_batch))
    return out


def loss_head(flow, mask, pred, pred_c, pred_i, cbn=0.5, epsilon=75.0, global_batch=None):
    """adversarial_learner.py:141-204 from the networks' outputs on: flow [B,H,W,2], mask [B,H,W,1] and the three recovered
    flows [B,H,W,2] -> the loss scalars, the per-sample terms, and `sums` [B,5] = the per-sample Charbonnier sums in the order
    the step graph accumulates them: {rec, rec_c, prior, den - epsilon, den_c - epsilon}.  Runs in the dtype of its inputs."""
    b, h, w, _ = flow.shape
    gb = global_batch or b
    m = mask
    mc = 1.0 - m                                                      # :107
    rec = charbonnier_loss(flow, pred, m, cbn)                        # :144
    rec_c = charbonnier_loss(flow, pred_c, mc, cbn)                   # :149
    prior_b = charbonnier_loss(flow, pred_i, torch.ones_like(flow), cbn)
    prior = prior_b.sum()                                             # :161-165
    recover_loss = (rec.sum() + rec_c.sum() + prior) / float(w * h * gb)        # :167-172
    den_s = charbonnier_loss(flow, pred_i, m, cbn)
    den = den_s + epsilon                                             # :179-182
    rr = (1.0 - rec / den).sum() / gb                                 # :183-184 (mean over the global batch)
    den_cs = charbonnier_loss(flow, pred_i, mc, cbn)
    den_c = den_cs + epsilon                                          # :186-189
    rr_c = (1.0 - rec_c / den_c).sum() / gb                           # :190-191
    return dict(generator=rr + rr_c, recover=recover_loss, red_rate=rr, red_rate_compl=rr_c, rec=rec, rec_c=rec_c, den=den,
                den_c=den_c, sums=torch.stack([rec, rec_c, prior_b, den_s, den_cs], dim=1))


def clip_or_noise(grads, clip=0.2, can_change=False, gen=None):
    """loss_utils.py:12-32: elementwise clip to +-clip; generator only: if the mean over variables of
    mean|g| < 1e-5, replace every grad by |U(-clip, clip)|."""
    if can_change:
        avg = torch.stack([g.abs().mean() for g in grads]).mean()
        if avg < 1e-5:
            return [torch.empty_like(g).uniform_(-clip, clip, generator=gen).abs() for g in grads], True
    return [g.clamp(-clip, clip) for g in grads], False


class TFAdam(object):
    """tf.train.AdamOptimizer(1e-4, beta1, 0.999, 1e-8), adversarial_learner.py:216-217.
    One optimizer object is shared by both train ops => the beta-power accumulators advance on every
    apply_gradients of either network (App. A.14)."""

    def __init__(self, lr=1e-4, beta1=0.9, beta2=0.999, eps=1e-8):
        self.lr, self.b1, self.b2, self.eps = lr, beta1, beta2, eps
        self.t = 0
        self.m, self.v = {}, {}

    def apply(self, params, names, grads):
        self.t += 1
        lr_t = self.lr * math.sqrt(1.0 - self.b2 ** self.t) / (1.0 - self.b1 ** self.t)
        with torch.no_grad():
            for n, g in zip(names, grads):
                if n not in self.m:
                    self.m[n] = torch.zeros_like(g)
                    self.v[n] = torch.zeros_like(g)
                self.m[n].mul_(self.b1).add_(g, alpha=1 - self.b1)
                self.v[n].mul_(self.b2).addcmul_(g, g, value=1 - self.b2)
                params[n].sub_(lr_t * self.m[n] / (self.v[n].sqrt() + self.eps))


def is_recover_step(step, iters_rec=1, iters_gen=3):
    """adversarial_learner.py:386-389."""
    return (step % (iters_rec + iters_gen)) < iters_rec


def train_step(p, opt, step, img1, img2, h, w, cfg=None, precomputed_flow=None):
    """One iteration of the loop body adversarial_learner.py:380-409 on explicit tensors.
    Returns dict(kind, loss_generator, loss_recover, grads(clipped), names)."""
    cfg = cfg or {}
    with torch.no_grad():
        flow384 = precomputed_flow if precomputed_flow is not None else predict_from_img_pairs(img1, img2, p)
        image, flow = resize_inputs(img1, flow384, h, w, cfg.get('flow_normalizer', 80.0))
    rec_step = is_recover_step(step, cfg.get('iters_rec', 1), cfg.get('iters_gen', 3))
    scope = 'FlownetS/' if rec_step else 'MaskNet/'
    names = [n for n in p if n.startswith(scope)]
    for n in names:
        p[n].requires_grad_(True)
    L = adversarial_losses(image, flow, p, cfg.get('cbn', 0.5), cfg.get('epsilon', 75.0), cfg.get('batch_size'))
    loss = L['recover'] if rec_step else L['generator']
    grads = torch.autograd.grad(loss, [p[n] for n in names])
    for n in names:
        p[n].requires_grad_(False)
    clipped, noised = clip_or_noise(list(grads), 0.2, can_change=not rec_step)
    opt.apply(p, names, clipped)
    return dict(kind='recover' if rec_step else 'generator', loss_generator=float(L['generator']),
                loss_recover=float(L['recover']), grads=list(grads), clipped=clipped, names=names, noised=noised,
                masks=L['masks'].detach())
