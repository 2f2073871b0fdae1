"""CPU: the parts of `bin/libFM -method sgda` decided before a device is touched, and the step at which the
reference takes an epoch's last moments.

* -method sgda runs in -mode inorder | ordered only: in the default -mode hogwild the refusal is unchanged; without
  -validation, and with -gpus 2, it stops with an error before loading anything.
* the t* rule of launch_sgda_epoch (sgda_last_moments_step, fmb200_internal.h) against a direct statement of the
  reference's epoch loop (fm_learn_sgd_element_adapt_reg.h:298-310), at N <= V, N = V m and N = V m + 1."""
import os
import subprocess

import pytest

from libfm_b200 import build

HOGWILD_REFUSAL = "\nERROR: method 'sgda' is outside the libfm_b200 scope (SGD hot path only); use -method sgd\n"


@pytest.fixture(scope="module")
def cli():
    exe = build.cli_path()
    if not os.path.exists(exe):
        build.build_all()
    return exe


def _run(cli, args, cwd):
    return subprocess.run([cli] + args.split(), cwd=cwd, capture_output=True, text=True)


def test_hogwild_refusal_unchanged(cli, tmp_path):
    p = _run(cli, "-train missing.libfm -test missing.libfm -task r -method sgda -iter 1", tmp_path)
    assert p.returncode == 1 and p.stderr == HOGWILD_REFUSAL


def test_no_validation_refused(cli, tmp_path):
    p = _run(cli, "-train missing.libfm -test missing.libfm -task r -method sgda -mode inorder", tmp_path)
    assert p.returncode == 1 and "-method sgda needs a validation set (-validation)" in p.stderr
    assert "Loading train" not in p.stdout


def test_more_gpus_refused(cli, tmp_path):
    p = _run(cli, "-train missing.libfm -test missing.libfm -validation missing.libfm -task r -method sgda "
                  "-mode ordered -gpus 2", tmp_path)
    assert p.returncode == 1 and "-method sgda runs on one GPU: -gpus must be 1" in p.stderr
    assert "Loading train" not in p.stdout


def reference_last_moments_step(n_train, n_val, lambda_steps):
    """:298-310 step by step: update_means at the epoch's start, and before the lambda-step that finds the
    validation cursor at its end.  Returns the step of the last such call, 0 for the one at the start."""
    last = 0
    if not lambda_steps:
        return last
    cursor = 0  # validation->data->begin()
    for t in range(n_train):  # sgd_theta_step(t), then:
        if cursor == n_val:  # validation->data->end()
            last, cursor = t, 0
        cursor += 1  # sgd_lambda_step, validation->data->next()
    return last


def last_moments_step(n_train, n_val, lambda_steps):
    """sgda_last_moments_step (libfm_b200/csrc/fmb200_internal.h)"""
    if not lambda_steps or n_val == 0 or n_train <= n_val:
        return 0
    return (n_train - 1) // n_val * n_val


@pytest.mark.parametrize("n_val", [1, 2, 3, 7, 250])
@pytest.mark.parametrize("m", [1, 2, 5])
def test_t_star_rule(n_val, m):
    for n_train in (1, n_val - 1, n_val, n_val * m, n_val * m + 1, n_val * m + n_val - 1):
        if n_train < 1:
            continue
        for lam in (False, True):
            assert last_moments_step(n_train, n_val, lam) == reference_last_moments_step(n_train, n_val, lam), \
                (n_train, n_val, lam)
