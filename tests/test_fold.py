"""Folding of mirror-image chains in the model-specialised forward-dynamics program (csrc/rbd_codegen.cpp).

The left / right legs and arms of a humanoid run the same code with different model constants; the generator emits each such
pair's steps once per ABA pass, as a two-iteration loop.  CPU tier: the folded program's CPU flavour is bit-identical to the
straight-line form of the same trace, the bundled humanoids actually fold, and a pair whose chains differ in a joint's fast
class stays straight-line."""
import numpy as np
import pytest

import rigidbodydynamics.jl_b200 as rbd
from tests import hostsim
from tests.util import rand_inputs


def _check_bit_identical(mech, dtype, expect_fold):
    desc = mech.flatten()
    q, v, tau, _, _ = rand_inputs(mech, 16, 3)
    for has_out1 in (False, True):
        p0, p1 = (hostsim.SpecProgram(desc, "aba", dtype, True, has_out1, fold=fold) for fold in (False, True))
        st0, src1, st1 = p0.stats, p1.src, p1.stats
        assert st0["fold_loops"] == 0
        if expect_fold:
            assert st1["fold_loops"] > 0 and st1["fold_bodies"] > 0 and "rbd_it" in src1
        a, b = p0.run(q, v, tau), p1.run(q, v, tau)
        if has_out1:
            (a, qa), (b, qb) = a, b
        assert np.isfinite(a).all() and np.array_equal(a, b)
        if has_out1:
            assert np.array_equal(qa, qb)
    return st1


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", ["atlas", "valkyrie"])
def test_humanoid_program_folds_bit_identical(name, dtype):
    st = _check_bit_identical(rbd.load_model(name, floating=True), dtype, True)
    assert st["pairs"] == 2                       # legs and arms
    assert st["fold_loops"] >= 4 and st["fold_bodies"] >= 4 * 6


def _mirrored_tree(seed, spoil=False):
    """Floating base, a short random branch, and two revolute chains of 4 bodies hung from the base: the same axis-aligned
    joint axes and tree rotations, translations mirrored in y, independent random inertias.  `spoil`: one joint of the right
    chain gets an origin shift where its left twin has none (F_ZERO_R), so the two chains no longer run the same code."""
    rng = np.random.default_rng(seed)
    eye = np.eye(3)
    M = np.diag([1.0, -1.0, 1.0])
    mech = rbd.Mechanism(rbd.RigidBody("world"))
    base = rbd.RigidBody("base", rbd.SpatialInertia.rand(rng))
    mech.attach(mech.root_body, base, rbd.Joint("floating", rbd.QuaternionFloating()))
    spec = []
    for k in range(4):
        perm = rng.permutation(3)
        R = eye[:, perm] * rng.choice([-1.0, 1.0], 3)
        if np.linalg.det(R) < 0:
            R[:, 0] = -R[:, 0]
        axis = eye[int(rng.integers(3))] * rng.choice([-1.0, 1.0])
        trans = np.zeros(3) if k == 2 else rng.standard_normal(3)
        spec.append((R, axis, trans))
    for side in ("l", "r"):
        parent = base
        for k, (R, axis, trans) in enumerate(spec):
            if side == "r":
                trans = M @ trans
                if spoil and k == 2:
                    trans = np.array([0.0, 0.0, 0.1])
            body = rbd.RigidBody(f"{side}{k}", rbd.SpatialInertia.rand(rng))
            mech.attach(parent, body, rbd.Joint(f"{side}j{k}", rbd.Revolute(axis)), joint_pose=rbd.Transform3D(R, trans))
            parent = body
    body = rbd.RigidBody("torso", rbd.SpatialInertia.rand(rng))
    mech.attach(base, body, rbd.Joint("tj", rbd.Revolute(eye[2])), joint_pose=rbd.Transform3D(eye, rng.standard_normal(3)))
    mech.attach(body, rbd.RigidBody("head", rbd.SpatialInertia.rand(rng)), rbd.Joint("hj", rbd.Revolute(eye[0])),
                joint_pose=rbd.Transform3D(eye, rng.standard_normal(3)))
    return mech


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_mirrored_random_chains_fold_bit_identical(dtype):
    for seed in (1, 2):
        st = _check_bit_identical(_mirrored_tree(seed), dtype, True)
        assert st["pairs"] == 1 and st["fold_loops"] == 3 and st["fold_bodies"] == 3 * 4


def test_mismatched_fast_class_stays_straight_line():
    mech = _mirrored_tree(1, spoil=True)
    desc = mech.flatten()
    src0, st0 = hostsim.spec_source(desc, "aba", np.float32, fold=False)
    src1, st1 = hostsim.spec_source(desc, "aba", np.float32, fold=True)
    assert st1["pairs"] == 0 and st1["fold_loops"] == 0
    assert src0 == src1 and "rbd_it" not in src1 and "rbd_par_tab" not in src1
