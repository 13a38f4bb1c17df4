"""Deterministic roidbs for the proposal-recall tests: hand-built edge cases and random ones.  Each case is (name, roidb, area, limit,
thresholds); entries carry the ground truth first and the proposals after it, as JsonDataset.get_roidb(gt=True, proposal_file=) does."""
import numpy as np


def entry(gt, props, classes=None, crowd=None, areas=None):
    gt = np.asarray(gt, np.float32).reshape(-1, 4)
    props = np.asarray(props, np.float32).reshape(-1, 4)
    G, P = len(gt), len(props)
    classes = np.ones(G, np.int32) if classes is None else np.asarray(classes, np.int32)
    crowd = np.zeros(G, bool) if crowd is None else np.asarray(crowd, bool)
    areas = ((gt[:, 2] - gt[:, 0] + 1) * (gt[:, 3] - gt[:, 1] + 1)) if areas is None else np.asarray(areas, np.float32)
    return {'boxes': np.vstack([gt, props]).astype(np.float32), 'gt_classes': np.r_[classes, np.zeros(P, np.int32)].astype(np.int32),
            'is_crowd': np.r_[crowd, np.zeros(P, bool)], 'seg_areas': np.r_[areas, np.zeros(P)].astype(np.float32)}


def random_entry(rng, P, G, crowd_frac=0.1, jitter=8.0):
    xy = rng.uniform(-20, 600, (G, 2))
    wh = np.exp(rng.uniform(np.log(2), np.log(700), (G, 2)))
    gt = np.hstack([xy, xy + wh]).astype(np.float32)
    src = gt[rng.randint(0, max(G, 1), P)] if G else rng.uniform(0, 600, (P, 4))
    props = (src + rng.normal(0, jitter, (P, 4)) * rng.uniform(0, 3, (P, 1))).astype(np.float32)
    props[rng.rand(P) < 0.1] = props[0] if P else 0            # repeated proposals: argmax ties
    areas = (wh[:, 0] * wh[:, 1] * rng.uniform(0.3, 1.0, G)).astype(np.float32)
    return entry(gt, props, rng.randint(1, 81, G), rng.rand(G) < crowd_frac, areas)


def edge_cases():
    rng = np.random.RandomState(7)
    C = []
    same = [[10, 10, 50, 50]] * 4
    C.append(("identical_proposals", [entry([[12, 8, 48, 52], [0, 0, 40, 40]], same)], 'all', None, None))
    C.append(("equal_cover", [entry([[0, 0, 9, 9], [20, 0, 29, 9]], [[0, 0, 9, 4], [20, 0, 29, 4], [0, 0, 9, 9]])], 'all', None, None))
    C.append(("p_lt_g", [random_entry(rng, 3, 9, 0)], 'all', None, None))
    C.append(("p_gt_g", [random_entry(rng, 200, 4, 0)], 'all', None, None))
    C.append(("limit_below_g", [random_entry(rng, 60, 12, 0)], 'all', 5, None))
    C.append(("limit_zero", [random_entry(rng, 60, 6, 0)], 'all', 0, None))
    C.append(("degenerate_boxes", [entry([[10, 10, 10, 30], [5, 5, 40, 40], [30, 30, 20, 50]],
                                         [[10, 10, 10, 30], [30, 30, 20, 50], [40, 5, 5, 40], [5, 5, 40, 40], [9.5, 10, 9.25, 30],
                                          [5, 5, 5, 5]])], 'all', None, None))
    C.append(("negative_coords", [entry([[-50, -40, 10, 20], [-5, -5, -1, -1]], [[-48, -41, 12, 18], [-6, -4, 0, 0], [-100, -100, -60, -60]])],
              'all', None, None))
    on_edges = [32 ** 2, 96 ** 2, 128 ** 2, 256 ** 2, 512 ** 2, 0, 1e10]
    e = random_entry(rng, 40, len(on_edges), 0)
    e['seg_areas'][:len(on_edges)] = on_edges
    for a in ('all', 'small', 'medium', 'large', '96-128', '128-256', '256-512', '512-inf'):
        C.append(("areas_on_bounds_" + a, [e], a, None, None))
    C.append(("crowd_only", [random_entry(rng, 30, 5, 1.0), random_entry(rng, 30, 3, 0)], 'all', None, None))
    C.append(("no_proposals", [random_entry(rng, 0, 5, 0), random_entry(rng, 30, 3, 0)], 'all', None, None))
    C.append(("no_gt", [random_entry(rng, 30, 0), random_entry(rng, 30, 4, 0)], 'all', None, None))
    C.append(("custom_thresholds", [random_entry(rng, 80, 10, 0)], 'all', 50, np.array([0.0, 0.1, 0.33, 0.7, 1.0])))
    C.append(("big_2000x120", [random_entry(rng, 2000, 120, 0.05, jitter=20.0)], 'all', None, None))
    C.append(("mixed_small", [random_entry(rng, int(rng.randint(0, 300)), int(rng.randint(0, 15))) for _ in range(40)], 'small', 100, None))
    return C


def random_roidb(seed, n_images=30):
    rng = np.random.RandomState(seed)
    return [random_entry(rng, int(rng.randint(0, 1200)), int(rng.randint(0, 25)), jitter=float(rng.uniform(2, 30))) for _ in range(n_images)]
