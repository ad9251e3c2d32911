"""Identify the mass of the Kuka iiwa's last link from the forces that hold its end effector in place (CUDA engine).

The "measurements" are the contact forces of the end-effector origin held by a bilateral position contact
(``compute_contact_dynamics``, position mode) on a model whose last link carries an extra payload.  A second model starts
from the URDF mass with that mass learnable, and Adam fits it to the measured forces through
``compute_contact_dynamics(..., differentiable=True)``: every step is one contact launch forward and the analytic adjoint
backward.

    python examples/identify_payload_from_contact_forces_iiwa.py [--batch 256] [--steps 300] [--payload 1.5]
"""
import argparse

import torch

from differentiable_robot_model_b200 import DifferentiableKUKAiiwa
from differentiable_robot_model_b200.rigid_body_params import UnconstrainedScalar

EE, LINK = "iiwa_link_ee", "iiwa_link_7"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--payload", type=float, default=1.5, help="extra mass of the last link in the measurements [kg]")
    ap.add_argument("--lr", type=float, default=0.05)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this example runs the CUDA engine and needs a GPU"
    dev = "cuda:0"
    torch.manual_seed(0)

    truth = DifferentiableKUKAiiwa(device=dev)
    mass0 = truth._bodies[truth._name_to_idx_map[LINK]].inertia.mass().detach().clone()
    urdf_mass, true_mass = float(mass0), float(mass0) + args.payload
    truth.make_link_param_learnable(LINK, "mass", UnconstrainedScalar(init_val=mass0 + args.payload))

    limits = truth.get_joint_limits()
    lo = torch.tensor([l["lower"] for l in limits], device=dev)
    hi = torch.tensor([l["upper"] for l in limits], device=dev)
    B, n = args.batch, truth._n_dofs
    q = lo + (hi - lo) * (0.2 + 0.6 * torch.rand(B, n, device=dev))
    qd = 0.3 * torch.randn(B, n, device=dev)
    f = 5.0 * torch.randn(B, n, device=dev)
    with torch.no_grad():
        measured = truth.compute_contact_dynamics(q, qd, f, [EE], position_only=True)
    keep = measured.solved

    model = DifferentiableKUKAiiwa(device=dev)
    mass = UnconstrainedScalar(init_val=mass0.clone())
    model.make_link_param_learnable(LINK, "mass", mass)
    opt = torch.optim.Adam(model.parameters(), lr=args.lr)
    for step in range(args.steps):
        opt.zero_grad()
        out = model.compute_contact_dynamics(q, qd, f, [EE], position_only=True, differentiable=True)
        loss = ((out.force - measured.force)[keep] ** 2).mean()
        loss.backward()
        opt.step()
        if step % 50 == 0 or step == args.steps - 1:
            print(f"step {step:4d}  loss {float(loss):.3e}  mass {float(mass.param):.4f}")
    got = float(mass.param)
    print(f"recovered mass {got:.4f} {true_mass:.4f} (URDF {urdf_mass:.4f})")


if __name__ == "__main__":
    main()
