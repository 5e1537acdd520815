"""Trees for the compressor tests (tests/test_compress_cpu.py, tests/test_gpu_compress.py): seeded stand-ins and
small SH1 trees whose single point set is an adversarial case for the median cut."""
import numpy as np

from volrend_b200 import synth


def tree_dict(st) -> dict:
    """The npz dict ``SynthTree.save_npz`` writes, plus the training-time keys a trained tree carries."""
    z = dict(data_dim=np.int64(st.data_dim), data_format=np.array(st.data_format),
             invradius3=st.invradius3.astype(np.float32), offset=st.offset.astype(np.float32),
             child=st.child, data=st.data, parent_depth=np.zeros((st.capacity, 2), np.int32),
             n_internal=np.int64(st.capacity), depth_limit=np.int64(st.depth))
    if st.extra is not None:
        z["extra_data"] = st.extra.astype(np.float32)
    return z


def sh1_tree(points, sigma=None, pad_to=None) -> dict:
    """A flat SH1 tree (root node only, plus padding nodes) whose slots hold ``points`` (fp16 [M, 3]) with sigma 10
    (or ``sigma``), so the one point set at retain 0 is exactly ``points`` in slot order."""
    pts = np.asarray(points, np.float16).reshape(-1, 3)
    M = pts.shape[0]
    n = max(M, pad_to or 0, 8)
    cap = (n + 7) // 8
    data = np.zeros((cap * 8, 4), np.float16)
    data[:M, :3] = pts
    data[:M, 3] = 10.0 if sigma is None else sigma
    child = np.zeros((cap, 2, 2, 2), np.int32)
    return dict(data_dim=np.int64(4), data_format=np.array("SH1"), invradius3=np.full(3, 0.5, np.float32),
                offset=np.full(3, 0.5, np.float32), child=child, data=data.reshape(cap, 2, 2, 2, 4))


def adversarial_sets(rng=None):
    """name -> fp16 [M, 3] point set."""
    rng = rng or np.random.default_rng(7)
    h = np.float16
    sets = {
        "all_equal": np.full((37, 3), 0.25, h),
        "value_ties": rng.integers(-2, 3, (300, 3)).astype(h) * h(0.5),
        "mixed_zero": np.where(rng.random((200, 3)) < 0.5, h(0.0), h(-0.0)).astype(h),
        # x and y ranges both 2, z range 1: x wins the tie; the y order decides nothing
        "axis_tie": np.stack([rng.choice([-1.0, 0.0, 1.0], 64), rng.choice([-1.0, 1.0], 64), rng.random(64)], 1).astype(h),
        "one": np.array([[1.5, -2.0, 3.0]], h),
        "three": np.array([[3.0, 0.0, 0.0], [1.0, 0.0, 0.0], [2.0, 0.0, 0.0]], h),
    }
    # -65504 x 16392, then 1000 points of 2^-24 (the smallest step), then the even child's mirror: the even bucket's
    # sum exceeds 2^54 units, so a double running sum drops each small term; the exact sum keeps them
    k, t = 16392, 1000
    sets["big_sum"] = np.zeros((2 * (k + t), 3), h)
    sets["big_sum"][:k, 0] = -65504.0
    sets["big_sum"][k:k + t, 0] = 2.0 ** -24
    sets["big_sum"][k + t:, 0] = 65504.0
    z = sets["mixed_zero"]
    z[::7] = rng.standard_normal((len(z[::7]), 3)).astype(h)
    return sets
