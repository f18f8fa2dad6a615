"""Dataset lookup with the reference's rule (datasets/__init__.py:18-20): alias -> module -> `Dataset`.

  synthetic_sequence  seeded synthetic pairs of the pair-file format (the default; no files needed)
  davis_sequence      the reference's DAVIS dataset: sequence .pt files + frames, same flags and items, plus --data_root
  shutterstock        the reference's Shutterstock dataset (integer --track_id), likewise
  video_frames        a video read from frames_midas/<track> + flow_pairs/<track>: pairs built in memory at construction
                      (flow_pairs.PairBuilder; raw flows resized and masked on the GPU), no per-pair files

Every train item is the batch dict the Model consumes, so `--resident` (datasets/resident.py) takes any of them."""
import importlib


def get_dataset(alias):
    return importlib.import_module(__name__ + '.' + (alias or 'synthetic_sequence')).Dataset
