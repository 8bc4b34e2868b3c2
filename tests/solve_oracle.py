"""NumPy restatement of the reference's rounding into the global frame (PGOAgent::getTrajectoryInGlobalFrame,
src/PGOAgent.cpp:500-519), the check of DistributedPGO.trajectory / dpgo_agent_trajectory_global."""
import numpy as np


def project_to_rotation(M: np.ndarray) -> np.ndarray:
    """ref projectToRotationGroup, src/DPGO_utils.cpp:463-477: U V^T, the last left singular vector flipped if det < 0."""
    U, _, Vt = np.linalg.svd(M)
    if np.linalg.det(U @ Vt) < 0:
        U[:, -1] = -U[:, -1]
    return U @ Vt


def trajectory_in_global_frame(X: np.ndarray, anchor: np.ndarray, d: int) -> np.ndarray:
    """X: r x (d+1)n lifted iterate, anchor: r x (d+1) = [Ya pa].  Per pose [proj(Ya^T Y_i)  Ya^T p_i - Ya^T pa]."""
    dh = d + 1
    Ya = anchor[:, :d]
    T = Ya.T @ X
    t0 = Ya.T @ anchor[:, d]
    for i in range(X.shape[1] // dh):
        T[:, i * dh:i * dh + d] = project_to_rotation(T[:, i * dh:i * dh + d])
        T[:, i * dh + d] -= t0
    return T
