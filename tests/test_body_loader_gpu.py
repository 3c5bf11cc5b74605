"""The engine's SMPL-X layer and the evaluation body models load through one builder: a malformed integer table of the
body-model dict is refused at mhmr_finalize with the message mhmr_body_create gives, before any kernel reads it."""
import pytest

import parity_util as pu

pytestmark = pytest.mark.gpu


def _parent_after_child(bm):
    bm["parents"] = bm["parents"].clone()
    bm["parents"][5] = 7


def _parent_out_of_range(bm):
    bm["parents"] = bm["parents"].clone()
    bm["parents"][5] = 55


def _extra_joint_past_the_mesh(bm):
    bm["extra_joints_idxs"] = bm["extra_joints_idxs"].clone()
    bm["extra_joints_idxs"][3] = bm["v_template"].shape[0]


def _landmark_corner_past_the_mesh(bm):
    bm["faces"] = bm["faces"].clone()
    bm["faces"][bm["lmk_faces_idx"][0], 1] = bm["v_template"].shape[0]


@pytest.mark.parametrize("corrupt, match", [
    (_parent_after_child, "must precede"),
    (_parent_out_of_range, "must precede"),
    (_extra_joint_past_the_mesh, "extra_joints_idxs out of range"),
    (_landmark_corner_past_the_mesh, "lmk_tri out of range"),
])
def test_finalize_rejects_bad_tables(corrupt, match, cuda_device):
    from multihmr_b200 import metrics

    case, sd, bm, _, _, _ = pu.build_inputs("s_224_S_forced")
    bm = dict(bm)
    corrupt(bm)
    m = pu.build_engine(case, sd, bm)
    with pytest.raises(AssertionError, match=match) as engine_err:
        m.finalize()
    with pytest.raises(AssertionError, match=match) as body_err:
        metrics.BodyModel(bm, "smplx", num_betas=10, max_persons=4, device=cuda_device)
    # "<entry> failed (code -2): <message>": the same message from both entries
    message = lambda e: str(e.value).split("): ", 1)[1]
    assert message(engine_err) == message(body_err)
