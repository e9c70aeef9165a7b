"""Seeded point clouds of the point-cloud tests (outlier removal, meshing, orientation).  Every generator draws from the
numpy Generator it is given, in a fixed order, so a cloud is a function of the seed and the arguments alone."""
import numpy as np

# corners 1e4 apart: coordinates large against the clusters' sizes
FAR = np.float32([[1e4, 1e4, 1e4], [-1e4, 1e4, -1e4], [1e4, -1e4, 0], [-1e4, -1e4, -1e4]])


def uniform(n, rng, lo=0.0, hi=1.0):
    """n points uniform in [lo, hi)^3, float32."""
    return rng.uniform(lo, hi, (n, 3)).astype(np.float32)


def sphere(n, rng, r=1.0, centre=(0.0, 0.0, 0.0), noise=0.0):
    """n points of the sphere, moved by Gaussian noise of std `noise` (drawn even when it is 0), float32, and their
    outward unit normals, float32."""
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (np.asarray(centre) + r * d + noise * rng.normal(size=(n, 3))).astype(np.float32), d.astype(np.float32)


def torus(n, rng, R0=1.0, r0=0.35):
    """n points of the torus around the z axis (ring radius R0, tube radius r0), float32; their outward unit normals,
    float32; and the nearest point of the ring to each, float64."""
    u, v = rng.uniform(0, 2 * np.pi, n), rng.uniform(0, 2 * np.pi, n)
    c = np.stack([np.cos(u), np.sin(u), np.zeros(n)], 1)
    nrm = np.cos(v)[:, None] * c + np.sin(v)[:, None] * np.array([0, 0, 1.0])
    return (R0 * c + r0 * nrm).astype(np.float32), nrm.astype(np.float32), R0 * c


def plane(n, rng, lo, hi, z, jitter=0.0):
    """n points uniform in [lo, hi)^2 at height z, plus Gaussian noise of std `jitter` in z when it is not 0, float32."""
    p = uniform(n, rng, lo, hi)
    p[:, 2] = np.float32(z) + rng.normal(0, jitter, n).astype(np.float32) if jitter else np.float32(z)
    return p


def lattice(m):
    """The m^3 integer points of [0, m)^3, float32, the first coordinate varying slowest."""
    g = np.arange(m, dtype=np.float32)
    return np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)


def clusters(rng, corners, counts, size):
    """counts[i] points uniform in the cube of side `size` at corners[i], one cube after the other, float32."""
    return np.concatenate([np.float32(c) + uniform(m, rng, 0.0, size) for c, m in zip(corners, counts)])


def dup_runs(n, rng, runs, gap):
    """n uniform points, then for every r in `runs` r copies of one point and `gap` more uniform points, shuffled,
    float32."""
    parts = [uniform(n, rng)]
    for r in runs:
        parts += [np.repeat(uniform(1, rng), r, 0), uniform(gap, rng)]
    p = np.concatenate(parts)
    return p[rng.permutation(p.shape[0])]
