"""Variable-name map between this package's parameter dict and the reference's TF1 graph  (SURVEY 8f-1).

Internal names (oracle/params.py, engine.ParamStore) attach a generator layer's batch-norm scale/offset to the conv layer
(`MaskNet/conv3/gamma`).  The reference's graph names them the way TF1 does:

  * `tf.name_scope("MaskNet") as scope` hands the *string* "MaskNet/" to `tf.variable_scope(scope)`
    (models/adversarial_learner.py:99-104, models/nets.py:17), so variables are expected under `MaskNet//...` (double slash);
    the same for "FlownetS/" (:112-117, nets.py:60).  The single-slash spelling is accepted on import as well.
  * `tf.layers.batch_normalization(x)` is unnamed (models/utils/convolution_utils.py:49) -> `batch_normalization`,
    `batch_normalization_1`, ... numbered per enclosing variable scope in creation order; `gen_deconv` opens its own scope
    (convolution_utils.py:68-73), so its conv is `<name>/<name>_conv` and its BN is `<name>/batch_normalization`.
  * recover-net layers are `model_variable('weights' / 'biases')` under the layer scope (convolution_utils.py:78-83).
  * PWC-Net variables already carry their TF names (`pwcnet/featpyr/conv1a/kernel`, models/PWCNet/model_pwcnet.py:154-166,478-504,
    561-574,284-286).
  * `global_step` is a `tf.Variable` created inside `tf.name_scope("train_op")` (adversarial_learner.py:206-208) -> `train_op/global_step`.

These spellings are derived from TF1's naming rules, not from a real checkpoint (none is available offline): `import_params`
therefore tries the candidates in order and reports the checkpoint's own keys when nothing matches.
"""
import numpy as np


GEN_SCOPE, REC_SCOPE, PWC_SCOPE = 'MaskNet', 'FlownetS', 'pwcnet'
GLOBAL_STEP_NAMES = ('train_op/global_step', 'global_step')
EMA_SUFFIX = '/ExponentialMovingAverage'


# creation order of generator_net's layers (models/nets.py:19-37); kept equal to models.nets.GEN_LAYERS by tests/test_tf_bundle.py
GEN_LAYER_NAMES = ('conv1', 'conv2_downsample', 'conv3', 'conv4_downsample', 'conv5', 'conv6', 'conv7_atrous', 'conv8_atrous',
                   'conv9_atrous', 'conv10_atrous', 'conv11', 'conv12', 'conv13_upsample', 'conv14', 'conv15_upsample', 'conv16',
                   'conv17')


def generator_tf_names(sep='//'):
    """internal name -> TF name for every generator variable."""
    out, bn = {}, 0
    for name in GEN_LAYER_NAMES:
        pre = GEN_SCOPE + sep
        if name.endswith('_upsample'):
            conv = '%s%s/%s_conv' % (pre, name, name)
            bnn = '%s%s/batch_normalization' % (pre, name)
        else:
            conv = pre + name
            bnn = pre + ('batch_normalization' if bn == 0 else 'batch_normalization_%d' % bn)
            bn += 1
        out['%s/%s/kernel' % (GEN_SCOPE, name)] = conv + '/kernel'
        out['%s/%s/bias' % (GEN_SCOPE, name)] = conv + '/bias'
        out['%s/%s/gamma' % (GEN_SCOPE, name)] = bnn + '/gamma'
        out['%s/%s/beta' % (GEN_SCOPE, name)] = bnn + '/beta'
    return out


def ema_name(internal):
    """The name of a variable's moving average: tf.train.ExponentialMovingAverage's shadow name, `<var>/ExponentialMovingAverage`."""
    return internal + EMA_SUFFIX


def to_tf_name(internal, sep='//', _cache={}):
    if internal.endswith(EMA_SUFFIX):
        return to_tf_name(internal[:-len(EMA_SUFFIX)], sep) + EMA_SUFFIX
    if internal.startswith(GEN_SCOPE + '/'):
        if sep not in _cache:
            _cache[sep] = generator_tf_names(sep)
        return _cache[sep][internal]
    if internal.startswith(REC_SCOPE + '/'):
        return REC_SCOPE + sep + internal[len(REC_SCOPE) + 1:]
    return internal


def export_params(params, global_step=None, sep='//'):
    """{internal name: tensor/array} -> {TF name: numpy array} ready for tf_bundle.write_bundle."""
    out = {}
    for k, v in params.items():
        a = v.detach().cpu().numpy() if hasattr(v, 'detach') else np.asarray(v)
        out[to_tf_name(k, sep)] = np.ascontiguousarray(a, dtype=np.float32)
    if global_step is not None:
        out[GLOBAL_STEP_NAMES[0]] = np.asarray(global_step, dtype=np.int32)
    return out


def import_params(tf_vars, wanted, strict=True):
    """Pick the `wanted` internal names out of a checkpoint's {TF name: array}.

    Returns ({internal: array}, global_step or None).  Both scope spellings are tried per variable; optimizer slots and
    anything else in the file are ignored (a PWC-Net checkpoint also holds Adam moments and its own global_step)."""
    out, missing = {}, []
    for k in wanted:
        for sep in ('//', '/'):
            t = to_tf_name(k, sep)
            if t in tf_vars:
                out[k] = tf_vars[t]
                break
        else:
            missing.append(k)
    if missing and strict:
        have = sorted(tf_vars)
        raise KeyError('checkpoint lacks %d of %d variables (first: %s -> tried %s); checkpoint holds %d keys, e.g. %s'
                       % (len(missing), len(wanted), missing[0], [to_tf_name(missing[0], s) for s in ('//', '/')],
                          len(have), have[:6]))
    gs = None
    for n in GLOBAL_STEP_NAMES:
        if n in tf_vars:
            gs = int(np.asarray(tf_vars[n]).reshape(-1)[0])
            break
    return out, gs


def normalize_prefix(path):
    """Accept `<prefix>`, `<prefix>.index` or `<prefix>.data-00000-of-00001` (scripts/test_DAVIS2016_raw.sh:11 passes the latter)."""
    if path.endswith('.index'):
        return path[:-6]
    i = path.rfind('.data-')
    if i >= 0 and '-of-' in path[i:]:
        return path[:i]
    return path
