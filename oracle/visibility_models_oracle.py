"""numpy restatements of the Biasutti and depth-map visibility models (oracle; test
infrastructure -- see oracle/__init__.py; never imported by the product path).

  image_knn / biasutti_alpha / biasutti_visibility <- visibility.py:1396-1500 (k_nn_image_system,
                                                      visibility_biasutti)
  depth_map_visibility                             <- visibility.py:1361-1392
  project_any / model_visibility                   <- visibility.py:478-538, 1694-1757, 1779-1799

Pinned on tests/golden/visibility_model_{biasutti_*,depth_*}.npz (oracle/make_golden_visibility.py).
Projection, features and the C restatement of the numba loops come from oracle/visibility_oracle.py.
"""
import numpy as np

from oracle.visibility_oracle import pose_to_rotation_matrix, postprocess_features, project_camera, project_equirect


def image_knn(x_proj, y_proj, k=75, x_margin=None, x_width=None, exact_below=20000):
    """k_nn_image_system (visibility.py:1396-1460) with an exact search: the search set is the n
    projections, then the left-margin copies (x <= x_margin, + float32(x_width)), then the
    right-margin copies (x >= x_width - x_margin, - float32(x_width)); rows = the n queries, ascending
    (d2, search-set index) with d2 = dx*dx + dy*dy in float32; k clamped to the search-set size;
    copies mapped back to their original index.  Search sets up to `exact_below` points are brute
    forced (neighborhood_oracle.knn_bruteforce with z = 0); larger ones take float64 candidates from
    scipy's cKDTree, re-ranked in float32 (d2, index), and a row is brute forced whenever the
    candidates cannot be shown to contain every point tied with or closer than its k-th."""
    from oracle.neighborhood_oracle import knn_bruteforce
    f32 = np.float32
    xp, yp = np.asarray(x_proj), np.asarray(y_proj)
    n = xp.shape[0]
    xy = np.stack([xp.astype(f32), yp.astype(f32)], axis=1)
    wrap = x_margin is not None and x_margin > 0 and x_width is not None and x_width > 0
    if wrap:
        left = np.nonzero(xp <= x_margin)[0]
        right = np.nonzero(xp >= (x_width - x_margin))[0]
        off = np.array([f32(x_width), 0], dtype=f32)
        search = np.concatenate([xy, xy[left] + off, xy[right] - off]).astype(f32)
        orig = np.concatenate([np.arange(n), left, right])
    else:
        search, orig = xy, np.arange(n)
    m = search.shape[0]
    k = min(int(k), m)
    pos = np.concatenate([search, np.zeros((m, 1), f32)], axis=1)
    if m <= exact_below:
        nbr, d2 = knn_bruteforce(pos, k)
        return orig[nbr[:n]], d2[:n]
    return _knn_candidates(search, n, k, orig)


def _knn_candidates(search, n, k, orig):
    from scipy.spatial import cKDTree
    f32 = np.float32
    m = search.shape[0]
    kc = min(m, k + 32)
    s64 = search.astype(np.float64)
    dist64, cand = cKDTree(s64).query(s64[:n], k=kc)
    cand = np.sort(cand.reshape(n, kc), axis=1)               # index order first: ties stay by index
    d = search[cand] - search[:n, None, :]
    d2 = d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]
    o = np.argsort(d2, axis=1, kind="stable")[:, :k]
    nbr = np.take_along_axis(cand, o, axis=1)
    d2k = np.take_along_axis(d2, o, axis=1)
    # a point outside the candidates is at float64 distance >= the farthest candidate's; the float32
    # d2 is within a few ulps of it, so rows whose k-th d2 is clearly below that bound are exact
    far = dist64.reshape(n, kc)[:, -1] ** 2
    ok = (kc == m) | (d2k[:, -1].astype(np.float64) * (1 + 1e-5) + 1e-30 < far)
    for i in np.nonzero(~ok)[0]:
        dd = search - search[i]
        dd2 = dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]
        oi = np.argsort(dd2, kind="stable")[:k]
        nbr[i], d2k[i] = oi, dd2[oi]
    return orig[nbr], d2k


def biasutti_alpha(dist, neighbors):
    """alpha = exp(-((d - d_min) / (d_max - d_min)) ** 2) over each row of neighbours, float32
    (visibility.py:1485-1489); NaN where every neighbour has the same depth.  exp is evaluated in
    float64 and rounded, i.e. within half an ulp of the exact value."""
    f32 = np.float32
    d = np.asarray(dist, f32)
    dnn = d[np.asarray(neighbors)]
    dmin, dmax = dnn.min(axis=1), dnn.max(axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = ((d - dmin) / (dmax - dmin)).astype(f32)
        return np.exp(-(r * r).astype(np.float64)).astype(f32)


def biasutti_visibility(x_proj, y_proj, dist, img_size, k=75, margin=None, threshold=None, neighbors=None):
    """visibility_biasutti (visibility.py:1463-1500) -> (indices, alpha, threshold): kept where
    alpha >= threshold, ascending; threshold None = float64 mean of alpha rounded to float32."""
    if neighbors is None:
        neighbors, _ = image_knn(x_proj, y_proj, k, margin, img_size[0])
    alpha = biasutti_alpha(dist, neighbors)
    thr = np.float32(alpha.astype(np.float64).mean()) if threshold is None else np.float32(threshold)
    return np.nonzero(alpha >= thr)[0], alpha, thr


def depth_map_visibility(x_proj, y_proj, dist, depth_map, depth_threshold=0.05):
    """visibility_from_depth_map (visibility.py:1361-1392): kept where
    |depth_map[int(x), int(y)] - dist| <= depth_threshold in float32, ascending."""
    f32 = np.float32
    dm = np.asarray(depth_map, f32)
    real = dm[np.asarray(x_proj).astype(np.int64), np.asarray(y_proj).astype(np.int64)]
    return np.nonzero(np.abs(real - np.asarray(dist, f32)) <= f32(depth_threshold))[0]


def project_any(xyz, img_xyz, img_opk=None, img_extrinsic=None, img_intrinsic_pinhole=None,
                img_intrinsic_fisheye=None, img_size=(1024, 512), crop_top=0, crop_bottom=0, r_max=30, r_min=0.5,
                camera="s3dis_equirectangular", **kwargs):
    """camera_projection_cpu (visibility.py:478-538) -> (indices, dist, x_proj, y_proj)."""
    xyz = np.ascontiguousarray(xyz, np.float32)
    img_xyz = np.asarray(img_xyz, np.float32)
    W, H = int(img_size[0]), int(img_size[1])
    if camera == "s3dis_equirectangular":
        R = pose_to_rotation_matrix(np.asarray(img_opk, np.float32))
        dist, xp, yp, keep = project_equirect(xyz, img_xyz, R, W, H, crop_top, crop_bottom, r_min, r_max)
    else:
        intr = img_intrinsic_fisheye if camera == "kitti360_fisheye" else img_intrinsic_pinhole
        dist, xp, yp, keep = project_camera(xyz, img_xyz, camera, img_extrinsic, np.asarray(intr), W, H, crop_top,
                                            crop_bottom, r_min, r_max)
    idx = np.nonzero(keep)[0]
    return idx, dist[idx], xp[idx], yp[idx]


def model_visibility(method, xyz, img_xyz, linearity=None, planarity=None, scattering=None, normals=None,
                     depth_map=None, **params):
    """BiasuttiVisibility / DepthBasedVisibility .__call__ (VisibilityModel.__call__,
    visibility.py:1694-1757): projection -> visibility -> the idx / x / y / depth / features dict.
    x and y are the kept float64 projections (:1499, :1392)."""
    img_size = tuple(int(v) for v in params.get("img_size", (1024, 512)))
    r_max, r_min = params.get("r_max", 30), params.get("r_min", 0.5)
    idx_1, dist, xp, yp = project_any(xyz, img_xyz, **params)
    if idx_1.size == 0:
        e = np.zeros(0, np.int64)
        return dict(idx=e, x=e.copy(), y=e.copy(), depth=np.zeros(0, np.float32), features=np.zeros(0, np.float32))
    if method == "BiasuttiVisibility":
        idx_2, _, _ = biasutti_visibility(xp, yp, dist, img_size, params.get("k", 75), params.get("margin"),
                                          params.get("threshold"))
    elif method == "DepthBasedVisibility":
        idx_2 = depth_map_visibility(xp, yp, dist, depth_map, params.get("depth_threshold", 0.05))
    else:
        raise ValueError(method)
    idx = idx_1[idx_2]
    pick = lambda a: None if a is None else np.asarray(a)[idx]  # noqa: E731
    feats = postprocess_features(np.asarray(xyz, np.float32)[idx] - np.asarray(img_xyz, np.float32), yp[idx_2],
                                 dist[idx_2], pick(linearity), pick(planarity), pick(scattering), pick(normals),
                                 img_size, r_max, r_min)
    return dict(idx=idx, x=xp[idx_2], y=yp[idx_2], depth=dist[idx_2], features=feats)
