"""oracle -- CPU checkers for the parity tests.  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
reference legs may import this package.  Three checkers:

  port  oracle/libfm_oracle.so        plain-C restatement (fm_oracle.c)
  ref   oracle/_ref/libfm_ref.so      the UNMODIFIED reference headers behind a
                                      C shim (ref_harness.cpp), built in place from
                                      /root/reference by oracle/Makefile
  rowlane_epoch_model                 fp64 numpy model of the reproducible row-lane HOGWILD
                                      epoch's windows (rowlane_model.py)
  rowgroup_epoch_model                fp64 numpy model of the free-running row-group HOGWILD epoch on
                                      data whose result no schedule can change (rowgroup_model.py)
  peer_model                          fp64 model of the per-epoch peer exchange: the mean and the
                                      mean-field combine with a per-element budget (peer_model.py)
"""
from .binding import Port, Ref, build, have_ref  # noqa: F401
from .rowgroup_model import concurrency, geometry, row_scores, rowgroup_epoch_model  # noqa: F401
from .rowlane_model import Budget, HParams, State, rowlane_epoch_model, ulp32  # noqa: F401
