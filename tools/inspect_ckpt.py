"""List the variables of a TF V2 checkpoint (like TensorFlow's inspect_checkpoint) and check them against the name map this
package expects -- the first thing to run when a real `model.best` / `pwcnet.ckpt-595000` is available (DESIGN.md section 5:
the bundle reader and the `MaskNet//...` name map are not pinned against a TF-written file yet).  --check also reports which PWC-Net
option set (use_dense_cx, use_res_cx, search_range) the checkpoint's pwcnet/* shapes match: the tfoptflow 'lg' and 'sm' networks differ
in them, and the matching values go into model_pwcnet._DEFAULT_PWCNET_TEST_OPTIONS.
Usage: python tools/inspect_ckpt.py <prefix | prefix.index | prefix.data-00000-of-00001> [--check]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from unsupervised_detection_b200 import checkpoint as ck  # noqa: E402
from unsupervised_detection_b200.checkpoint import tf_names  # noqa: E402


def pwcnet_variable_names(options=None):
    """Names of the PWC-Net variables this package loads for an option set (models/PWCNet/model_pwcnet.py of the reference: featpyr
    conv{l}{a,aa,b}, predict_flow conv{l}_{0..4} + flow{l}, ctxt dc_conv{l}{1..7} (levels 6..3 only with use_res_cx), upsample
    up_flow{l} / up_feat{l}; pyramid levels 6..2)."""
    return [e[0] for e in pwcnet_shapes(options)]


def pwcnet_shapes(options=None):
    """[(name, shape)] of the pwcnet/* variables of an option set, in checkpoint layout."""
    from unsupervised_detection_b200.engine import ParamStore
    from unsupervised_detection_b200.models.PWCNet.model_pwcnet import PWCNetBuilder
    st = ParamStore('cpu')
    PWCNetBuilder(st, options=options)
    return [(e[0], tuple(e[1])) for e in st.entries]


def detect_pwc_options(shapes):
    """{name: shape} of a checkpoint -> (options dict or None, message).  The Cin of predict_flow/conv6_0 is (2r+1)^2, conv6_1 reads
    conv6_0's 128 channels alone without dense connections and 128 + (2r+1)^2 with them, and ctxt/dc_conv61 exists only with the
    context network on every level."""
    get = lambda n: shapes.get('pwcnet/' + n + '/kernel')
    s0, s1 = get('predict_flow/conv6_0'), get('predict_flow/conv6_1')
    if s0 is None or s1 is None:
        return None, 'no pwcnet/predict_flow/conv6_0 or conv6_1 kernel'
    nd = int(s0[2])
    r = int(round((nd ** 0.5 - 1) / 2))
    if (2 * r + 1) ** 2 != nd:
        return None, 'predict_flow/conv6_0 has Cin %d, not a (2r+1)^2 correlation width' % nd
    if int(s1[2]) == 128:
        dense = False
    elif int(s1[2]) == 128 + nd:
        dense = True
    else:
        return None, 'predict_flow/conv6_1 has Cin %d: neither 128 (no dense connections) nor %d (dense)' % (int(s1[2]), 128 + nd)
    opts = {'use_dense_cx': dense, 'use_res_cx': get('ctxt/dc_conv61') is not None, 'search_range': r}
    if r not in (1, 2, 3, 4):
        return None, 'search_range %d (from conv6_0 Cin %d) is outside the supported 1..4' % (r, nd)
    want = pwcnet_shapes(opts)
    bad = [(n, shp, shapes.get(n)) for n, shp in want if tuple(shapes.get(n, ())) != shp]
    if bad:
        n, shp, got = bad[0]
        return None, '%s suggests %s, but %d of %d variables differ (first %s: expected %s, found %s)' % (
            'conv6_0 / conv6_1 / dc_conv61', opts, len(bad), len(want), n, shp, got)
    return opts, 'all %d pwcnet/* variables match use_dense_cx=%s, use_res_cx=%s, search_range=%d' % (
        len(want), opts['use_dense_cx'], opts['use_res_cx'], opts['search_range'])


def main(argv):
    prefix = ck.normalize_prefix(argv[1])
    rows = ck.list_variables(prefix)
    for name, shape, dtype in rows:
        print('%-70s %-18s %s' % (name, tuple(shape), getattr(dtype, '__name__', dtype)))
    print('%d variables, %d parameters' % (len(rows), sum(int(__import__("numpy").prod(s)) if s else 1 for _, s, _ in rows)))
    if '--check' in argv:
        have = set(n for n, _, _ in rows)
        from unsupervised_detection_b200 import params_init
        shapes = {n: tuple(int(d) for d in shp) for n, shp, _ in rows}        # PWC-Net variables keep their TF names (tf_names.py)
        opts, msg = detect_pwc_options(shapes)
        print('pwcnet    options: %s' % msg)
        want = list(params_init.init_generator()) + list(params_init.init_recover()) + pwcnet_variable_names(opts)
        for scope in ('MaskNet', 'FlownetS', 'pwcnet'):
            names = [k for k in want if k.startswith(scope + '/')]
            hit = {sep: sum(tf_names.to_tf_name(k, sep) in have for k in names) for sep in ('//', '/')}
            print('%-9s %3d variables expected; found with "//" spelling: %3d, with "/" spelling: %3d' % (scope, len(names), hit['//'], hit['/']))
            miss = [k for k in names if not any(tf_names.to_tf_name(k, s) in have for s in ('//', '/'))]
            for k in miss[:10]:
                print('   missing: %s  (tried %s)' % (k, [tf_names.to_tf_name(k, s) for s in ('//', '/')]))


if __name__ == '__main__':
    main(sys.argv)
