from promp_b200.envs.base import MetaEnv, Box  # noqa: F401
from promp_b200.envs.normalized_env import normalize, NormalizedEnv  # noqa: F401
from promp_b200.envs.point_env_2d_corner import MetaPointEnvCorner  # noqa: F401
from promp_b200.envs.point_env_2d import MetaPointEnv  # noqa: F401
from promp_b200.envs.half_cheetah_rand_direc import HalfCheetahRandDirecEnv  # noqa: F401
from promp_b200.envs.half_cheetah_rand_vel import HalfCheetahRandVelEnv  # noqa: F401
from promp_b200.envs.point_env_2d_walls import MetaPointEnvWalls  # noqa: F401
from promp_b200.envs.point_env_2d_momentum import MetaPointEnvMomentum  # noqa: F401
from promp_b200.envs.walker2d_rand_vel import Walker2DRandVelEnv, Walker2DRandDirecEnv  # noqa: F401
from promp_b200.envs.swimmer_rand_vel import SwimmerRandVelEnv  # noqa: F401
from promp_b200.envs.cuda_env import CudaMetaEnv, CudaEnvProgram  # noqa: F401
