"""Inputs and the replay recipe of the batched LocalMapping searches (borb_search_for_triangulation_batch, borb_fuse_batch).
Test tooling."""
import dataclasses

import numpy as np

from orb_slam2_b200.matcher import FeatureVector
from tests import match_fixtures as mf


def flip_bits(rng, d, p):
    flip = rng.random((len(d), 32, 8)) < p
    return d ^ np.packbits(flip, axis=2, bitorder="little").reshape(len(d), 32)


def neighbourhood(v, voc, n_neighbours=6, levelsup=2):
    """A keyframe (the left view) and n_neighbours keyframes that re-observe the right view: each its own descriptor noise,
    MapPoint mask and stereo coordinates, FeatureVectors from the vocabulary."""
    kf1, _ = mf.keyframe_views(v, voc, 9, levelsup=levelsup, mp_frac=0.3)
    rng = np.random.default_rng(3)
    out = []
    for i in range(n_neighbours):
        _, kf2 = mf.keyframe_views(v, voc, 20 + i, levelsup=levelsup, mp_frac=0.2 + 0.05 * i)
        d = flip_bits(rng, kf2.mDescriptors, 0.005 * (i + 1))
        _, weight, node = voc.transform_raw(d, levelsup)
        out.append(dataclasses.replace(kf2, mDescriptors=d, mFeatVec=FeatureVector.from_nodes(node, weight > 0)))
    return kf1, out


def accept(pairs):
    """The simulated triangulation of the replay: every second pair gets a MapPoint."""
    return pairs[::2, 0]


def sequential(search, kf1, kf2s):
    """LocalMapping::CreateNewMapPoints as the reference runs it: neighbour i sees the MapPoints the earlier ones created."""
    hm = kf1.has_mp.copy()
    out = []
    for kf2 in kf2s:
        p = search(dataclasses.replace(kf1, has_mp=hm.copy()), kf2)
        out.append(p)
        hm[accept(p)] = 1
    return out


def replay(entry_pairs, has_mp):
    """The same from one search per neighbour with kf1's entry mask: neighbour i drops every idx1 an earlier one gave a MapPoint."""
    hm = has_mp.copy()
    out = []
    for p in entry_pairs:
        p = p[hm[p[:, 0]] == 0]
        out.append(p)
        hm[accept(p)] = 1
    return out
