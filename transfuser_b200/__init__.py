"""transfuser_b200 — H100-native (sm_90a) TransFuser training hot path behind the reference's nn.Module contract."""
from .backbone import GeometricFusionBackbone, LateFusionBackbone, TransfuserBackbone, latentTFBackbone  # noqa: F401
from .model import LidarCenterNet  # noqa: F401
from .bev import lidar_to_histogram_features  # noqa: F401
