"""Rotation <-> quaternion conversions of the CMR loaders, in float64 (w, x, y, z order; 4x4 homogeneous matrices).

The loaders convert with the "precise" branch of the classic trace / largest-diagonal method, and the mirrored pose goes
matrix -> flipped matrix -> quaternion, so the poses here are computed with the same operations in the same order: the
pose table and the items then agree with the reference loaders bit for bit."""
import math

import numpy as np

_TINY = np.finfo(float).eps * 4.0


def quaternion_matrix(quaternion):
    """Homogeneous 4x4 rotation matrix of a (not necessarily unit) quaternion (w, x, y, z)."""
    q = np.array(quaternion, dtype=np.float64, copy=True)
    norm2 = np.dot(q, q)
    if norm2 < _TINY:
        return np.identity(4)
    q *= math.sqrt(2.0 / norm2)
    p = np.outer(q, q)
    w, x, y, z = 0, 1, 2, 3
    m = np.identity(4)
    m[0, 0], m[0, 1], m[0, 2] = 1.0 - p[y, y] - p[z, z], p[x, y] - p[z, w], p[x, z] + p[y, w]
    m[1, 0], m[1, 1], m[1, 2] = p[x, y] + p[z, w], 1.0 - p[x, x] - p[z, z], p[y, z] - p[x, w]
    m[2, 0], m[2, 1], m[2, 2] = p[x, z] - p[y, w], p[y, z] + p[x, w], 1.0 - p[x, x] - p[y, y]
    return m


def quaternion_from_matrix(matrix, isprecise=True):
    """Quaternion (w, x, y, z, w >= 0) of a precise 4x4 homogeneous rotation matrix.  Only the precise method is
    provided: it is the one the loaders use."""
    if not isprecise:
        raise NotImplementedError('quaternion_from_matrix: only isprecise=True (the loaders\' method) is provided')
    M = np.asarray(matrix, dtype=np.float64)[:4, :4]
    q = np.empty(4)
    t = np.trace(M)
    if t > M[3, 3]:
        # w is the largest component
        q[0] = t
        q[1] = M[2, 1] - M[1, 2]
        q[2] = M[0, 2] - M[2, 0]
        q[3] = M[1, 0] - M[0, 1]
    else:
        # start from the largest diagonal entry i and its cyclic successors j, k
        i = 0
        if M[1, 1] > M[0, 0]:
            i = 1
        if M[2, 2] > M[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = M[i, i] - (M[j, j] + M[k, k]) + M[3, 3]
        q[1 + i] = t
        q[1 + j] = M[i, j] + M[j, i]
        q[1 + k] = M[k, i] + M[i, k]
        q[0] = M[k, j] - M[j, k]
    q *= 0.5 / math.sqrt(t * M[3, 3])
    if q[0] < 0.0:
        np.negative(q, q)
    return q
