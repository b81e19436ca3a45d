"""Launches of the bi-LSTM recurrence (lstm_cluster.cu: lstm_cluster_kernel) and the layouts lstm_layer gives them (no GPU
needed).

* model_launches -- every recurrence launch of the model at one batch (any in tc_cases.ACCEPTED_BATCHES, 1 .. 1024): the
                    eval forward (model.cu forward_rnn), the training forward (train_step.cu) and TTA (hn_model_infer_tta:
                    up to 64 views in one forward), each with both layers at T = 256;
* abi_launches   -- hn_lstm_layer takes any T >= 1: T = 1 (no exchange at all), 2 (one exchange, no re-arming) and 3
                    (an odd T);
* plan / variant_key -- hn_lstm_plan and the paths of the kernel a layout takes: one or two 8-column groups per cluster,
                    more than one cluster per direction, a last cluster that runs one group while the others run two, a
                    partial last group, clusters beyond what the device co-schedules (a second wave), and the T class;
* CASES          -- the -m gpu unit cases of test_lstm_variants.py, one per key, named by it; batch_for gives the
                    smallest batch that reaches a key on a device with a given number of co-resident clusters.

The number of co-resident 16-CTA clusters decides the layout.  An H100 SXM (132 SMs) co-schedules 7; the 114-SM H100 PCIe
has not been measured, so the census takes every count from 2 (the least hn_lstm_layer accepts) to 8."""
import ctypes

from horizonnet_b200 import _lib
from tc_cases import ACCEPTED_BATCHES

PLAN_FIELDS = ('max_clusters', 'ngroups', 'gpc', 'clusters', 'last_cluster_groups', 'last_group_cols', 'waves')
KEY_FIELDS = ('gpc', 'multi_cluster', 'last_cluster_one_group', 'partial_group', 'second_wave', 'T')
MAX_CLUSTERS = tuple(range(2, 9))
MODEL_T = 256
T_CLASSES = ('1', '2', 'odd', 'even')
# the T each unit case runs at: odd T = 5 is the first odd T whose waits reuse a barrier phase (step 3 waits for h_2 on
# parity 0 in phase 1); the even class runs at the model's T
T_FOR_CLASS = {'1': 1, '2': 2, 'odd': 5, 'even': MODEL_T}


def model_launches(B):
    return [dict(name=f'{path} bi_rnn layer {layer}', T=MODEL_T, B=B)
            for path in ('eval forward', 'training forward', 'TTA') for layer in (1, 2)]


def abi_launches(B):
    return [dict(name=f'hn_lstm_layer T={T}', T=T, B=B) for T in (1, 2, 3)]


def plan(T, B, max_clusters):
    """hn_lstm_plan as a dict of PLAN_FIELDS, or None where the library rejects the arguments."""
    out = (ctypes.c_int * len(PLAN_FIELDS))()
    if _lib.lib().hn_lstm_plan(T, B, max_clusters, out) != 0:
        return None
    return dict(zip(PLAN_FIELDS, out))


def t_class(T):
    return '1' if T == 1 else '2' if T == 2 else 'odd' if T % 2 else 'even'


def variant_key(T, p):
    return (p['gpc'], p['clusters'] > 2, p['gpc'] == 2 and p['last_cluster_groups'] == 1, p['last_group_cols'] < 8,
            p['waves'] > 1, t_class(T))


def key_dict(k):
    return dict(zip(KEY_FIELDS, k))


def key_name(k):
    gpc, multi, last_one, partial, wave2, tc = k
    return '-'.join([f'g{gpc}', 'multi' if multi else 'single', 'last1' if last_one else 'lastfull',
                     'partial' if partial else 'full', 'wave2' if wave2 else 'wave1', f'T{tc}'])


def check_plan(T, B, p):
    """The clusters of a plan own every column 0..B-1 exactly once, as lstm_cluster_kernel assigns them: cluster pair c
    (one per direction) runs groups c*gpc .. c*gpc + ng - 1, ng = min(gpc, ngroups - c*gpc), and group g columns
    8g .. min(8g + 8, B) - 1."""
    assert p['ngroups'] == -(-B // 8) and p['gpc'] in (1, 2) and p['clusters'] % 2 == 0, p
    owner = [0] * B
    ng = nb = 0
    for c in range(p['clusters'] // 2):
        ng = min(p['gpc'], p['ngroups'] - c * p['gpc'])
        assert ng >= 1, (T, B, p)
        for g in range(c * p['gpc'], c * p['gpc'] + ng):
            nb = min(8, B - 8 * g)
            assert nb >= 1, (T, B, p)
            for col in range(8 * g, 8 * g + nb):
                owner[col] += 1
    assert owner == [1] * B, (T, B, p, owner)
    assert ng == p['last_cluster_groups'] and nb == p['last_group_cols'], (T, B, p)
    assert p['waves'] == -(-p['clusters'] // p['max_clusters']), (T, B, p)


# One unit case per layout and T class.  The layouts, in the order of the batch that reaches them on 7 clusters:
LAYOUTS = [
    # gpc, more than one cluster per direction, last cluster runs one of two groups, partial last group, second wave
    (1, False, False, True, False),      # B = 1: the smallest launch
    (1, False, False, False, False),     # B = 8: one full group per direction
    (1, True, False, True, False),       # B = 9 (4+ clusters): a full group and a 1-column group on separate clusters
    (1, True, False, False, False),      # B = 16 (4+ clusters)
    (2, False, False, True, False),      # B = 9 (2-3 clusters): both groups on one cluster, the second has one column
    (2, False, False, False, False),     # B = 16 (2-3 clusters)
    (2, True, True, True, False),        # B = 33 (6-8 clusters): the last cluster runs one 1-column group
    (2, True, True, False, False),       # B = 40 (6-8 clusters)
    (2, True, False, True, False),       # B = 25 (4-7 clusters)
    (2, True, False, False, False),      # B = 32 (4-7 clusters): the benchmark's batch
    # a second wave (8 clusters: from B = 65 on), its last cluster one 1-column group
    (2, True, True, True, True),         # B = 49 (6-7 clusters; 8: B = 65)
    (2, True, True, False, True),        # B = 56 (6-7 clusters; 8: B = 72)
    (2, True, False, True, True),        # B = 57 (6-7 clusters; 8: B = 73)
    (2, True, False, False, True),       # B = 64 (6-7 clusters; 8: B = 80)
]
CASES = [key_name(lay + (tc,)) for lay in LAYOUTS for tc in T_CLASSES]
CASE_KEYS = {key_name(lay + (tc,)): lay + (tc,) for lay in LAYOUTS for tc in T_CLASSES}


def batch_for(key, max_clusters):
    """The smallest batch (1 .. 1024) whose layout at the key's T has the key on a device with max_clusters co-resident
    clusters, or None when no batch of the model reaches it there."""
    T = T_FOR_CLASS[key[5]]
    for B in ACCEPTED_BATCHES:
        p = plan(T, B, max_clusters)
        if p is not None and variant_key(T, p) == key:
            return B
    return None
