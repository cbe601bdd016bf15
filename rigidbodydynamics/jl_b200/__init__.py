"""rigidbodydynamics.jl_b200 -- batched rigid-body dynamics on NVIDIA H100.

Drop-in for ONE path of RigidBodyDynamics.jl: ``dynamics!``, ``inverse_dynamics!``, ``mass_matrix!``, ``dynamics_bias!``
on ``Mechanism`` / ``MechanismState`` / ``DynamicsResult``, evaluated over a batch of states by hand-written sm_90a
kernels behind a C ABI (``include/rbd_b200.h``, ``csrc/librbd_b200.so``).  This Python package is the host side above
that ABI (Julia, the reference's language, is not available in the build image; ``julia/RBDB200.jl`` is the
equivalent shim).  Importing the package does not need a GPU; calling a dynamics function does.
"""
from .spatial import *          # noqa: F401,F403
from .joint_types import *      # noqa: F401,F403
from .mechanism import *        # noqa: F401,F403
from .mechanism import (DEFAULT_GRAVITATIONAL_ACCELERATION, Joint, Mechanism, ModelDesc, RigidBody,  # noqa: F401
                        rand_chain_mechanism, rand_floating_tree_mechanism, rand_tree_mechanism)
from .joint_types import (Fixed, Planar, Prismatic, QuaternionFloating, QuaternionSpherical, Revolute,  # noqa: F401
                          SinCosRevolute, SPQuatFloating)
from .urdf import (default_urdf_joint_types, load_description, load_model, mechanism_from_description,  # noqa: F401
                   parse_urdf, read_urdf)
from .state import (DynamicsResult, MechanismState, rand_, rand_configuration_, rand_velocity_, zero_,  # noqa: F401
                    zero_configuration_, zero_velocity_)
from .algorithms import (DimensionMismatch, dynamics_, dynamics_derivatives_, dynamics_dual_, dynamics_bias, dynamics_bias_, dynamics_ode_,  # noqa: F401
                         inverse_dynamics, inverse_dynamics_, mass_matrix, mass_matrix_, simulate_,
                         simulate_trajectory_)
from .kinematics import (TreePath, center_of_mass, geometric_jacobian, geometric_jacobian_,  # noqa: F401
                         gravitational_potential_energy, kinematics_, kinetic_energy, momentum, momentum_matrix,
                         momentum_matrix_, momentum_rate_bias, path, transforms_to_root, transforms_to_root_)
from .kinematics import (TaskFrame, point_acceleration, point_jacobian, point_velocity, relative_acceleration,  # noqa: F401
                         relative_transform, relative_twist, task_kinematics_)
from .contact import (ContactDesc, ContactPoint, HalfSpace3D, HuntCrossleyModel, SoftContactModel,  # noqa: F401
                      ViscoelasticCoulombModel, add_contact_point, add_environment_primitive, contact_desc, contact_dynamics_,
                      contact_points, dynamics_contact_, environment, hunt_crossley_hertz, num_contact_states,
                      simulate_contact_, simulate_contact_trajectory_)
from .loops import (LoopDesc, PDGains, SE3PDGains, constraint_wrench_subspace, default_constraint_stabilization_gains,  # noqa: F401
                    dynamics_loops_, loop_desc, num_constraints, simulate_loops_, simulate_loops_trajectory_)
from .mechanism import maximal_coordinates  # noqa: F401
from .mechanism import Bounds, effort_bounds  # noqa: F401
from .pd import JointPD, TaskPD, task_pd_torques  # noqa: F401
from . import autodiff  # noqa: F401  (rbd.autodiff.dynamics / inverse_dynamics: differentiable, kept out of this namespace)
from .autodiff import (dynamics_vjp_, integrate_contact_vjp_, integrate_pd_vjp_, integrate_task_pd_vjp_, integrate_vjp_,  # noqa: F401
                       inverse_dynamics_vjp_)
from ._cabi import RbdError, launch_info, load_library  # noqa: F401
