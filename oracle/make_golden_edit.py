"""TEST INFRASTRUCTURE - generates tests/golden/causal_edit_256x6_n16.npz by running the UNMODIFIED
reference's streaming step with point edits.

Needs a checkout of the reference (oracle/reference_loader.py, TAPNET_REFERENCE_ROOT):
  python -m oracle.make_golden_edit

A causal 256^2 x 6 clip with 16 points (weights, video and queries from the seeds of
`oracle/synth.py`, as the causal goldens of `oracle/make_golden.py`) is stepped frame by frame:
- frame 2: point 3 is re-targeted, the live demo's click (pytorch_live_demo.py:180-200): a
  one-frame get_feature_grids + get_query_features on the frame, then update_query_features;
- frame 2: 4 points are appended.  The reference has no append: their query features, sampled the
  same way, are concatenated along the point axis, and zero rows of construct_initial_causal_state's
  layout are appended to every state tensor;
- frame 4: points 0 and 9 are removed by an index-select of the features and every state tensor.
Each frame then runs the streaming step on its point set.  The fixture holds the per-frame tracks,
occlusion and expected distance, and the edits and per-frame counts in its meta.
"""
import json
import os

import numpy as np
import torch

from oracle import reference_loader, synth
from oracle.make_golden import GOLDEN_DIR

NAME = 'causal_edit_256x6_n16'
MODEL_KWARGS = dict(pyramid_level=1, use_casual_conv=True)
T, N, H, W = 6, 16, 256, 256
EDITS = dict(retarget_frame=2, retarget_idx=3, retarget_point=[0.0, 100.5, 37.25],
             add_frame=2, add_points=[[0.0, 20.0, 30.0], [0.0, 128.5, 200.25], [0.0, 250.0, 5.0],
                                      [0.0, 64.0, 64.0]],
             remove_frame=4, remove_idx=[0, 9])


def _np(x):
  return x.detach().cpu().numpy()


def run():
  sd = synth.make_state_dict(0, MODEL_KWARGS['pyramid_level'], True)
  model = reference_loader.build(sd, **MODEL_KWARGS)
  video = synth.make_video(T, H, W, seed=1)
  queries = synth.make_queries(N, T, H, W, seed=2, frame0_only=True)
  e = EDITS
  out = {}
  with torch.no_grad():
    g0 = model.get_feature_grids(video[:, :1], False)
    qf = model.get_query_features(video[:, :1], False, queries, g0)
    levels = len(qf.resolutions) - 1
    state = model.construct_initial_causal_state(N, levels)
    counts = []
    for t in range(T):
      frame = video[:, t:t + 1]
      if t == e['retarget_frame']:
        gf = model.get_feature_grids(frame, False)
        new = model.get_query_features(frame, False, torch.tensor([[e['retarget_point']]]), gf)
        qf, state = model.update_query_features(qf, new, np.array([e['retarget_idx']]),
                                                causal_state=state)
      if t == e['add_frame']:
        gf = model.get_feature_grids(frame, False)
        add = torch.tensor([e['add_points']])
        new = model.get_query_features(frame, False, add, gf)
        qf = type(qf)(tuple(torch.cat([a, b], 1) for a, b in zip(qf.lowres, new.lowres)),
                      tuple(torch.cat([a, b], 1) for a, b in zip(qf.hires, new.hires)),
                      qf.resolutions)
        zeros = model.construct_initial_causal_state(add.shape[1], levels)
        state = [{k: torch.cat([v, zeros[i][k]], 1) for k, v in d.items()}
                 for i, d in enumerate(state)]
      if t == e['remove_frame']:
        keep = torch.tensor([i for i in range(qf.lowres[0].shape[1]) if i not in e['remove_idx']])
        qf = type(qf)(tuple(x.index_select(1, keep) for x in qf.lowres),
                      tuple(x.index_select(1, keep) for x in qf.hires), qf.resolutions)
        state = [{k: v.index_select(1, keep) for k, v in d.items()} for d in state]
      g = model.get_feature_grids(frame, False)
      r = model.estimate_trajectories((H, W), False, g, qf, None, query_chunk_size=64,
                                      causal_context=state, get_causal_context=True)
      state = r['causal_context']
      out[f'online_tracks_{t}'] = _np(r['tracks'][-1][0])
      out[f'online_occlusion_{t}'] = _np(r['occlusion'][-1][0])
      out[f'online_expected_dist_{t}'] = _np(r['expected_dist'][-1][0])
      counts.append(int(qf.lowres[0].shape[1]))
  meta = dict(name=NAME, model_kwargs=MODEL_KWARGS, T=T, N=N, H=H, W=W, mode='causal_edit',
              weights_seed=0, video_seed=1, query_seed=2, edits=e, counts=counts,
              torch=torch.__version__)
  out['meta'] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
  return out


def main():
  os.makedirs(GOLDEN_DIR, exist_ok=True)
  out = run()
  path = os.path.join(GOLDEN_DIR, NAME + '.npz')
  np.savez_compressed(path, **out)
  print(NAME, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
  main()
