"""GPU parity for the "next" rows (SURVEY.md §8f): candidate search, cloud assembly (transformPcd + submap merge +
pcl::VoxelGrid) and the batched performLoopClosure driver, against the CPU oracle."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def seq(synth):
    return synth.make_sequence(7, 140, pts_per_keyframe=6000, spacing=3.0, speed=8.0)


@pytest.fixture(scope="module")
def store(ctx, seq):
    kf = ctx.keyframes()
    for c, T, t in zip(seq["clouds"], seq["poses"], seq["stamps"]):
        kf.add(c, T, t)
    yield kf
    kf.destroy()


def test_fetch_closest_equals_oracle(store, oracle, seq):
    pos = seq["poses"][:, :3, 3]
    queries = np.arange(len(pos), dtype=np.int32)
    got = store.fetch_closest(queries, 35.0, 30.0)
    want = np.array([oracle.fetch_closest(pos, seq["stamps"], q, 35.0, 30.0) for q in queries])
    assert np.array_equal(got, want)
    assert (want >= 0).sum() > 10 and (want < 0).sum() > 10


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def test_assemble_quatro_and_submap_modes(ctx, store, oracle, seq):
    import b200reg
    pairs = [(137, 3), (139, 70), (120, 55)]
    src_idx = [p[0] for p in pairs]
    dst_idx = [p[1] for p in pairs]
    for quatro, submap in ((1, 0), (0, 0), (1, 1)):
        cfg = b200reg.default_loop_config()
        cfg.enable_quatro, cfg.enable_submap_matching = quatro, submap
        sc, dc = store.assemble(src_idx, dst_idx, cfg, n_keyframes=140)
        for k, (si, di) in enumerate(pairs):
            os_, od_ = oracle.set_src_and_dst_cloud(seq["clouds"], seq["poses"], si, di, submap_range=5, voxel_res=0.3,
                                                    enable_quatro=bool(quatro), enable_submap_matching=bool(submap), n_keyframes=140)
            for cloud, want in ((sc[k], os_), (dc[k], od_)):
                got = ctx.cloud_points(cloud)
                assert got.shape[0] == want.shape[0], "voxel count must match pcl::VoxelGrid's"
                # same voxel order (linear voxel index), same fp32 sums in the same order: bit-identical centroids
                assert np.array_equal(_bits(got), _bits(want[:, :3]))
        for c in sc + dc:
            c.destroy()


def test_perform_loop_closure_matches_oracle(ctx, store, oracle, synth, seq):
    import b200reg
    queries = np.array([137, 139, 20, 118], np.int32)
    closest = store.fetch_closest(queries)
    assert closest[2] == -1 and (closest[[0, 1, 3]] >= 0).all()
    res, qi = store.perform_loop_closure(queries, closest)
    assert not res[2]["valid"] and np.array_equal(res[2]["T"], np.eye(4))  # dummy output (loop_closure.cpp:201-204)
    for k in (0, 1, 3):
        q, c = int(queries[k]), int(closest[k])
        src, dst = oracle.set_src_and_dst_cloud(seq["clouds"], seq["poses"], q, c, n_keyframes=q + 1)
        if qi[k]["valid"]:
            o = oracle.coarse_to_fine(src, dst, quatro_T=qi[k]["T"])
            rot, tr = synth.se3_error(res[k]["T"], o["T"])
            assert rot < 3e-4 and tr < 3e-3, (k, rot, tr)  # same clouds bit for bit; the registrations reduce in other orders
            # the loop closure undoes the accumulated odometry drift between the two keyframes
            drift = seq["true_poses"][c] @ np.linalg.inv(seq["poses"][c]) @ seq["poses"][q] @ np.linalg.inv(seq["true_poses"][q])
            # T maps src (map frame by odom) onto dst: T ~= D_c * inv(D_q) with D = odom * inv(true)
            Dq = seq["poses"][q] @ np.linalg.inv(seq["true_poses"][q])
            Dc = seq["poses"][c] @ np.linalg.inv(seq["true_poses"][c])
            rot, tr = synth.se3_error(res[k]["T"], Dc @ np.linalg.inv(Dq))
            assert rot < 2e-2 and tr < 0.3, ("ground truth", k, rot, tr)
    # GICP-only mode (scan-to-submap, loop_closure.cpp:94-105)
    cfg = b200reg.default_loop_config()
    cfg.enable_quatro = 0
    res2, _ = store.perform_loop_closure(queries[:2], closest[:2], cfg)
    for k in range(2):
        q, c = int(queries[k]), int(closest[k])
        src, dst = oracle.set_src_and_dst_cloud(seq["clouds"], seq["poses"], q, c, enable_quatro=False, n_keyframes=q + 1)
        o = oracle.gicp_align(src, dst)
        rot, tr = synth.se3_error(res2[k]["T"], o["T"])
        assert rot < 3e-4 and tr < 3e-3, (k, rot, tr)


def test_loop_factors_close_the_loop(ctx, store, oracle, synth, seq):
    """Result consumption (fast_lio_sam_qn.cpp:220-237): the factor records of a batch equal the oracle's, and applying
    the measurement brings the drifted latest keyframe back onto the truth relative to the matched one."""
    queries = np.array([137, 20, 118], np.int32)
    closest = store.fetch_closest(queries)
    raw, _ = store.perform_loop_closure(queries, closest, raw=True)
    facs = store.loop_factors(queries, closest, raw)
    assert facs[1]["to_idx"] == -1 and not facs[1]["valid"]  # no candidate: nothing for the graph
    for k in (0, 2):
        q, c = int(queries[k]), int(closest[k])
        f = facs[k]
        assert (f["from_idx"], f["to_idx"]) == (q, c) and f["valid"] == bool(raw[k].valid)
        T = np.array(raw[k].pose_between).reshape(4, 4)  # RegistrationOutput::pose_between_eig_ is what the factor is built from
        M, var = oracle.loop_factor(T, seq["poses"][q], seq["poses"][c], raw[k].fitness)
        assert np.abs(f["measurement"] - M).max() < 1e-12 and np.array_equal(f["variances"], var)
        # the measured relative pose is the TRUE relative pose of the two keyframes (drift removed)
        true_rel = np.linalg.inv(seq["true_poses"][q]) @ seq["true_poses"][c]
        rot, tr = synth.se3_error(f["measurement"], true_rel)
        assert rot < 2e-2 and tr < 0.3, (k, rot, tr)


def test_batched_queries_see_their_own_keyframe_count(ctx, store, oracle, seq):
    """A batch replays several loopTimerFunc ticks: the sub-map bound `i < keyframes.size() - 1` (loop_closure.cpp:72,79,100)
    is evaluated with size = query + 1 PER QUERY, so a batch equals the one-by-one replay -- also for the non-maximal
    queries, whose merged clouds must not reach past (or onto) their own query keyframe."""
    import b200reg
    cfg = b200reg.default_loop_config()
    cfg.enable_submap_matching = 1
    # closest keyframes chosen within the sub-map range of their query so that the bound actually bites
    queries = np.array([60, 100, 139], np.int32)
    closest = np.array([57, 97, 136], np.int32)
    sc, dc = store.assemble(queries, closest, cfg, n_keyframes=queries + 1)
    for k in range(3):
        q, c = int(queries[k]), int(closest[k])
        os_, od_ = oracle.set_src_and_dst_cloud(seq["clouds"], seq["poses"], q, c, submap_range=5, voxel_res=0.3,
                                                enable_quatro=True, enable_submap_matching=True, n_keyframes=q + 1)
        for cloud, want in ((sc[k], os_), (dc[k], od_)):
            got = ctx.cloud_points(cloud)
            assert got.shape[0] == want.shape[0], (k, got.shape, want.shape)
            assert np.array_equal(_bits(got), _bits(want[:, :3])), k
    # the batch-wide bound (the old behaviour: size = max(query) + 1) gives DIFFERENT clouds for the non-maximal queries
    sc2, dc2 = store.assemble(queries, closest, cfg, n_keyframes=int(queries.max()) + 1)
    assert sc2[0].n != sc[0].n and sc2[2].n == sc[2].n
    # and the batched driver equals the one-by-one replay bit for bit
    res, _ = store.perform_loop_closure(queries, closest, cfg)
    for k in range(3):
        single, _ = store.perform_loop_closure(queries[k:k + 1], closest[k:k + 1], cfg)
        assert np.array_equal(res[k]["T"], single[0]["T"]) and res[k]["fitness"] == single[0]["fitness"]
    for c in sc + dc + sc2 + dc2:
        c.destroy()


def test_pose_pcd_ingest_matches_oracle(ctx, oracle, synth, seq):
    """Row f4: the PosePcd constructor (pose_pcd.hpp:21-43) as a device step -- the world-frame scan FAST-LIO publishes goes into
    the LiDAR frame with pose_eig_.inverse(), the pose comes from the odometry quaternion -- against the oracle, and a keyframe
    ingested that way registers exactly like one added in the LiDAR frame."""
    from b200reg import io as bio
    kf = ctx.keyframes()
    worst = 0.0
    for k in (3, 70, 137):
        T = seq["poses"][k]
        lidar = seq["clouds"][k]
        world = synth.to_map_frame(lidar, T)  # what FAST-LIO publishes (world frame)
        q = bio._rot_to_quat(T[:3, :3])
        q = q * 1.0000001  # odometry quaternions are never exactly unit: tf's setRotation divides by |q|^2
        idx = kf.add_world(world, T[:3, 3], q, seq["stamps"][k])
        got, pose, ts = kf.get(idx)
        want, opose = oracle.pose_pcd_ingest(world, T[:3, 3], q)
        assert np.abs(pose - opose).max() < 1e-15 and ts == seq["stamps"][k]
        assert np.array_equal(got[:, 3], want[:, 3])                       # intensity carried
        # two different 4x4 inverses (cofactors vs Gauss-Jordan) differ by ~1e-16 relative, i.e. ~1e-14 m in the translation:
        # the float results are at most one ulp apart (or 1e-12 m where a coordinate is nearly zero)
        ulp = np.maximum(np.spacing(np.maximum(np.abs(want[:, :3]), np.abs(got[:, :3])).astype(np.float32)), 1e-12)
        assert (np.abs(got[:, :3] - want[:, :3]) <= ulp).all()
        assert (got[:, :3] == want[:, :3]).mean() > 0.99  # measured 0.9988: cond([R|t]) ~ 1e4 amplifies the inverses' round-off
        worst = max(worst, np.abs(got[:, :3] - lidar[:, :3]).max())
    assert worst < 2e-5  # back in the LiDAR frame: the original scan up to the float round trip through the world frame
    kf.destroy()


def test_keyframe_store_slabs_and_reserve(ctx, synth):
    """Keyframes live in slabs apart from the scratch pool: a reservation that runs out rolls over to a new slab, and
    every keyframe reads back exactly as it was added, before and after registration calls used the scratch pool."""
    seq = synth.make_sequence(3, 9, pts_per_keyframe=4000, spacing=5.0)
    kf = ctx.keyframes()
    kf.reserve(2 * 4000 + 100)  # room for two keyframes and a bit: the third one opens a new slab
    for c, T, t in zip(seq["clouds"], seq["poses"], seq["stamps"]):
        kf.add(c, T, t)
    kf.reserve(0)
    q = np.array([8], np.int32)
    kf.perform_loop_closure(q, np.array([0], np.int32))
    for i, (c, T, t) in enumerate(zip(seq["clouds"], seq["poses"], seq["stamps"])):
        pts, pose, ts = kf.get(i)
        assert np.array_equal(pts, c[:, :4].astype(np.float32)) and np.array_equal(pose, T) and ts == t
    kf.destroy()


# ---- k_assemble point for point --------------------------------------------------------------------------------
SUBMAP_SIZES = (1, 255, 256, 257, 3001)  # segment boundaries inside and on the edges of 256-thread blocks


@pytest.fixture(scope="module")
def ragged_store(ctx, seq):
    """40 keyframes with the sequence's (non-identity) poses and point counts cycling through SUBMAP_SIZES."""
    kf = ctx.keyframes()
    clouds = [seq["clouds"][k][:SUBMAP_SIZES[k % len(SUBMAP_SIZES)]] for k in range(40)]
    for k, c in enumerate(clouds):
        kf.add(c, seq["poses"][k], seq["stamps"][k])
    yield kf, clouds, seq["poses"][:40]
    kf.destroy()


def test_assemble_point_for_point(ctx, oracle, ragged_store):
    """At a 1 mm leaf every merged cloud (but a lone 1-point keyframe) trips VoxelGrid's int32 guard, so the call returns
    k_assemble's merged cloud itself: it must be the concatenation of oracle.transform_pcd over the sub-map, bit for bit.
    num_submap_keyframes = 15 merges up to 31 keyframes; centres at 0 and at n_keyframes - 1; n_keyframes per pair."""
    import b200reg
    kf, clouds, poses = ragged_store
    leaf, rng = 1e-3, 15
    src = np.array([0, 39, 20, 21], np.int32)
    dst = np.array([39, 0, 22, 3], np.int32)
    nks = np.array([40, 40, 40, 22], np.int32)
    cfg = b200reg.default_loop_config()
    cfg.num_submap_keyframes, cfg.voxel_res = rng, leaf
    nseg = []
    for quatro, submap in ((1, 1), (0, 0), (1, 0)):
        cfg.enable_quatro, cfg.enable_submap_matching = quatro, submap
        sc, dc = kf.assemble(src, dst, cfg, n_keyframes=nks)
        for k in range(len(src)):
            for centre, cloud, merged in ((src[k], sc[k], submap), (dst[k], dc[k], submap or not quatro)):
                ids = [i for i in range(centre - rng, centre + rng + 1) if 0 <= i < nks[k] - 1] if merged else [centre]
                nseg.append(len(ids))
                want = np.concatenate([oracle.transform_pcd(clouds[i], poses[i]) for i in ids])
                assert np.array_equal(_bits(oracle.voxelize(want, leaf)), _bits(want))  # the guard trips (or one point)
                got = ctx.cloud_points(cloud)
                assert np.array_equal(_bits(got), _bits(want[:, :3])), (quatro, submap, k, centre)
        for c in sc + dc:
            c.destroy()
    assert max(nseg) == 2 * rng + 1 and min(nseg) == 1
    cfg.num_submap_keyframes = 16  # 33 keyframes > MAXSEG
    with pytest.raises(b200reg.B200RegError, match="error -1:"):
        kf.assemble(src, dst, cfg, n_keyframes=nks)


# ---- k_fetch_closest at its edges ------------------------------------------------------------------------------
def _fetch(ctx, oracle, pos, stamps, queries, radius, tdiff):
    """Single-point keyframes at `pos`; the device answer for `queries`, checked against the oracle."""
    kf = ctx.keyframes()
    for p, t in zip(pos, stamps):
        T = np.eye(4)
        T[:3, 3] = p
        kf.add(np.ones((1, 4), np.float32), T, float(t))
    got = kf.fetch_closest(np.asarray(queries, np.int32), radius, tdiff)
    kf.destroy()
    want = np.array([oracle.fetch_closest(pos, stamps, q, radius, tdiff) for q in queries])
    assert np.array_equal(got, want), (got, want)
    return got


def test_fetch_closest_ties_go_to_the_lowest_index(ctx, oracle):
    """Equidistant candidates in the same lane (idx mod 32) and in different lanes; four scenes 1 km apart, queried by
    keyframes 96..99.  The distances are exact (integer offsets), so the ties are exact."""
    n = 100
    pos = np.zeros((n, 3))
    pos[:, 1] = 5000.0 + 10.0 * np.arange(n)  # fillers: out of reach of every query
    stamps = np.arange(n, dtype=np.float64)
    scenes = [  # (candidate idx, offset); the answer
        ([(5, (3, 4, 0)), (37, (0, 3, 4))], 5),                      # same lane 5
        ([(33, (0, -5, 0)), (12, (5, 0, 0))], 12),                   # lane 12 holds the lower index than lane 1
        ([(40, (4, 3, 0)), (8, (0, 0, -5)), (70, (-3, 0, 4))], 8),   # three lanes, two of them the same
        ([(9, (3, 4, 0)), (41, (0, 4, 3)), (90, (4.999, 0, 0))], 90),  # strictly closer beats the lower index
    ]
    for a, (cands, _) in enumerate(scenes):
        o = np.array([1000.0 * (a + 1), 0.0, 0.0])
        pos[96 + a] = o
        for idx, off in cands:
            pos[idx] = o + np.array(off, np.float64)
    got = _fetch(ctx, oracle, pos, stamps, [96, 97, 98, 99], 35.0, 0.5)
    assert got.tolist() == [w for _, w in scenes]


def test_fetch_closest_bounds_are_strict(ctx, oracle):
    """radius > dist and tdiff < stamp gap: a candidate at exactly the radius and one exactly tdiff older are excluded."""
    pos = np.array([[3.0, 4.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 0.0]])  # keyframe 0 at distance 5, keyframe 1 at distance 1
    stamps = np.array([0.0, 98.0, 100.0])                                # keyframe 1 exactly 2 s before the query
    up, down = np.nextafter(5.0, np.inf), np.nextafter(2.0, -np.inf)
    assert _fetch(ctx, oracle, pos, stamps, [2, 0], 5.0, 2.0).tolist() == [-1, -1]
    assert _fetch(ctx, oracle, pos, stamps, [2], up, 2.0).tolist() == [0]
    assert _fetch(ctx, oracle, pos, stamps, [2], 5.0, down).tolist() == [1]
    assert _fetch(ctx, oracle, pos, stamps, [2], up, down).tolist() == [1]


def test_fetch_closest_query_sizes(ctx, oracle):
    """2001 keyframes on an integer lattice (ties and dist == radius everywhere), stamps 0.25 s apart so that the
    candidate exactly tdiff = 2 s older is excluded: queries with fewer candidates than a warp's lanes, exactly 32,
    just over, and 2000, in one batch; then every query."""
    rng = np.random.default_rng(5)
    pos = rng.integers(-8, 9, (2001, 3)).astype(np.float64)
    stamps = 0.25 * np.arange(2001)
    got = _fetch(ctx, oracle, pos, stamps, [0, 1, 31, 32, 33, 64, 2000], 5.0, 2.0)
    assert got[0] == -1 and got[1] == -1 and (got[3:] >= 0).all()
    every = _fetch(ctx, oracle, pos, stamps, np.arange(2001), 5.0, 2.0)
    d = np.linalg.norm(pos[:1992] - pos[2000], axis=1)
    assert (d == 5.0).any() and len(set(np.round(d, 9))) < 1992  # the boundary distance and ties occur
    assert (every >= 0).mean() > 0.9
