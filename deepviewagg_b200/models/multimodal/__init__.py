from .no3d import (No3D, No3DEncoder, No3DFeatureFusion, No3DImageFeatureFusion, No3DImageLogitFusion,  # noqa: F401
                   No3DLogitFusion)
from .sparseconv3d import APIModel, LateFeatureFusion, LateLogitFusion  # noqa: F401
