"""Float32 restatement of LocalTrajectoryBuilder2D's per-point stages
(mapping/internal/2d/local_trajectory_builder_2d.cc): AddRangeData's loop (:163-186),
TransformRangeData and CropRangeData (sensor/range_data.cc:25-39), step by step in numpy float32
scalars with the reference's operation order."""
import numpy as np

from cartographer_b200.local_slam import rigid3f_apply

F = np.float32


def accumulate(hits, origins, origin_index, poses, pose_index, min_range, max_range,
               missing_data_ray_length):
    """-> (returns, misses) of one synchronized scan; poses are (t(3), q(4)) float32 tuples."""
    returns, misses = [], []
    for i, h in enumerate(np.asarray(hits, np.float32).reshape(-1, 3)):
        pose = poses[pose_index[i]]
        o = rigid3f_apply(pose, np.asarray(origins, np.float32)[origin_index[i]])
        p = rigid3f_apply(pose, h)
        d = [p[k] - o[k] for k in range(3)]
        rng = F(np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]))
        if rng >= F(min_range):
            if rng <= F(max_range):
                returns.append(p)
            else:
                s = F(missing_data_ray_length) / rng
                misses.append(tuple(o[k] + s * d[k] for k in range(3)))
    return (np.array(returns, np.float32).reshape(-1, 3), np.array(misses, np.float32).reshape(-1, 3))


def transform(points, rigid):
    return np.array([rigid3f_apply(rigid, p) for p in np.asarray(points, np.float32)],
                    np.float32).reshape(-1, 3)


def crop(points, min_z, max_z):
    p = np.asarray(points, np.float32).reshape(-1, 3)
    return p[(F(min_z) <= p[:, 2]) & (p[:, 2] <= F(max_z))]
