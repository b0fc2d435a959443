"""CPU oracle of the "SQfp16" shard (faiss IndexScalarQuantizer(QT_fp16) without lists): rows encoded to
fp16 with numpy (round to nearest even, overflow to +-inf -- what __float2half_rn and F16C vcvtps2ph do),
then the existing flat oracle over the decoded rows.  Its state is the engine's: "metric" and "codes16"."""
import numpy as np

from distributed_faiss_b200.index import factory_spec
from oracle import oracle as O
from tests.oracle_sq8 import oracle_engine_factory


def encode(x):
    """float32 rows -> their fp16 codes as uint16 (np.float16: round to nearest even, overflow to inf)"""
    with np.errstate(over="ignore"):
        return np.ascontiguousarray(np.asarray(x, dtype=np.float32).astype(np.float16)).view(np.uint16)


def decode(codes):
    """uint16 codes -> the float32 rows they stand for (exact)"""
    return np.ascontiguousarray(np.asarray(codes, dtype=np.uint16)).view(np.float16).astype(np.float32)


class OracleFlatSQ16(O.OracleFlat):
    """IndexScalarQuantizer(d, QT_fp16, metric): the flat oracle over the decoded rows"""

    kind = "flat_sq16"

    def __init__(self, d, metric=O.METRIC_IP):
        super().__init__(d, metric)
        self.codes16 = np.zeros((0, self.d), dtype=np.uint16)

    def add(self, x):
        c = encode(np.asarray(x, dtype=np.float32).reshape(-1, self.d))
        self.codes16 = np.concatenate([self.codes16, c], axis=0)
        self.xb = decode(self.codes16)

    def set_state(self, st):
        super().set_state(st)
        self.xb = decode(self.codes16)


def flat_sq16_engine_factory(cfg):
    """tests/oracle_sq8.oracle_engine_factory (builders and IVF factory strings), plus the factory string
    "SQfp16", as distributed_faiss_b200.index.default_engine_factory builds them"""
    spec = factory_spec(cfg)
    if spec is not None and spec.kind == "flat_sq16":
        return OracleFlatSQ16(cfg.dim, spec.metric)
    return oracle_engine_factory(cfg)
