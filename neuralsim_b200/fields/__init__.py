"""Field objects the NeuS ray query drives: LoTD encoding, SDF / radiance networks, occupancy-grid accel, AABB space."""
from .encoding import LoTD, LoTDEncoding, gen_ngp_cfg, generate_meta  # noqa: F401
from .networks import MLP, DenseLayer, LoTDSDF, RadianceNet, SHEncoder, VarSingleMixLinear  # noqa: F401
from .accel import OccGridAccel, OccGridEma  # noqa: F401
from .space import AABBSpace  # noqa: F401
from .neus import LoTDNeuS, LoTDNeuSModel  # noqa: F401
from .occ_update import OccGridUpdate  # noqa: F401
