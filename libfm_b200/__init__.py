"""libfm_b200 -- the libFM SGD training hot path, rebuilt for H100 (sm_90a).

Scope: the per-example loop of srendle/libfm (`fm_model::predict` + `fm_SGD`
driven by `fm_learn_sgd_element::learn`) as hand-written CUDA behind the C ABI
of include/fmb200.h, plus the host mirror needed to drive it.  See DESIGN.md.
"""
from .model import (Data, FmError, FmLearnSgdElement, FmModel, MODE_HOGWILD, MODE_INORDER, MODE_ORDERED,
                    RelationData, RelationJoin, TASK_CLASSIFICATION, TASK_REGRESSION)

__all__ = ["Data", "FmError", "FmLearnSgdElement", "FmModel", "MODE_HOGWILD", "MODE_INORDER", "MODE_ORDERED",
           "RelationData", "RelationJoin", "TASK_CLASSIFICATION", "TASK_REGRESSION"]
