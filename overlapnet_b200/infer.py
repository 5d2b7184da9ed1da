"""Drop-in replacement of the reference's ``Infer`` class (src/two_heads/infer.py:22-265).

Same constructor argument (the dict loaded from config/network.yml), same public attributes and
the same four entry points with the same argument meaning, return shapes/dtypes and error
behaviour; underneath, the Keras leg/head models are replaced by the CUDA kernels behind the C ABI
(include/ovn_b200.h) and the feature bank lives on the GPU instead of in a Python list that is
re-stacked on every query (infer.py:193,228).

Additions that the reference does not have (all optional): ``precision`` / ``device`` keyword
arguments, ``.npz`` weights, and ``encode_clouds`` / ``infer_one_raw`` which take raw ``.bin``
clouds through the fused projection kernels instead of preprocessed ``.npy`` files.
"""
import os

import numpy as np
import torch

from . import weights as _weights
from .config import check_model
from .engine import Engine, FEAT_C, check_probs


class _ModelShim:
  """Stands in for the ``keras.Model`` objects the reference exposes as ``Infer.leg`` /
  ``Infer.head`` (infer.py:101,111): ``predict`` on host arrays."""

  def __init__(self, fn):
    self._fn = fn

  def predict(self, x, **kwargs):
    return self._fn(x)


class Infer():
  """ A class used for inferring overlap and yaw-angle between LiDAR scans (infer.py:22). """

  def __init__(self, config, precision='f16_tc', device=None, max_batch_pairs=None):
    """ Args: config: A dict with configuration values, usually loaded from a yaml file
        (infer.py:26-122). """
    self.network_output_size = config['model']['leg_output_width']
    self.seq = config['infer_seqs']
    self.datasetpath = config['data_root_folder']

    # infer.py:36-59
    self.use_depth = config['use_depth'] if 'use_depth' in config else True
    self.use_normals = config['use_normals'] if 'use_normals' in config else True
    self.use_class_probabilities = config['use_class_probabilities'] \
        if 'use_class_probabilities' in config else False
    self.use_class_probabilities_pca = config['use_class_probabilities_pca'] \
        if 'use_class_probabilities_pca' in config else False
    self.use_intensity = config['use_intensity'] if 'use_intensity' in config else False

    # no channels for input -- read unguarded like infer.py:61-73 (all five keys are required)
    self.no_input_channels = 0
    if config['use_depth']:
      self.no_input_channels += 1
    if config['use_normals']:
      self.no_input_channels += 3
    if config['use_intensity']:
      self.no_input_channels += 1
    if config['use_class_probabilities']:
      if config['use_class_probabilities_pca']:
        self.no_input_channels += 3
      else:
        self.no_input_channels += 20

    # Input shape of model; mutates the config in place like infer.py:76-82
    self.inputShape = config['model']['inputShape']
    if len(self.inputShape) == 3:
      pass
    elif len(self.inputShape) == 2:
      self.inputShape.append(self.no_input_channels)
    else:
      self.inputShape[2] = self.no_input_channels

    self.batch_size = config['batch_size']

    model_cfg = config['model']
    check_model(model_cfg)                                   # infer.py:91-93 (getattr on generateNet)
    # the generators inject their defaults into the dict (generateNet.py:88-89,143-146)
    model_cfg.setdefault('strides_layer1', (2, 2))
    model_cfg.setdefault('additional_unsymmetric_layer3a', False)
    model_cfg.setdefault('conv1NetworkHead_conv1size', 15)

    use = {'use_depth': config['use_depth'], 'use_normals': config['use_normals'],
           'use_class_probabilities': config['use_class_probabilities'],
           'use_class_probabilities_pca': config['use_class_probabilities_pca'],
           'use_intensity': config['use_intensity']}
    self._engine = Engine(use=use, model=model_cfg, precision=precision, device=device,
                          max_batch_scans=max(1, int(self.batch_size)),
                          max_batch_pairs=int(max_batch_pairs or 2048),
                          proj_H=self.inputShape[0], proj_W=self.inputShape[1])
    self.leg = _ModelShim(self._leg_predict)
    self.head = _ModelShim(self._head_predict)

    # previous feature volumes: device-resident bank, exposed as a list on access
    self._bank = torch.empty((0, self.network_output_size, FEAT_C), dtype=torch.float32,
                             device=self._engine.device)
    self._bank_n = 0
    self._fv_as_array = False

    # Load weights from training (infer.py:115-122)
    pretrained_weightsfilename = config['pretrained_weightsfilename']
    if len(pretrained_weightsfilename) > 0:
      self._engine.load_weights(_weights.load(pretrained_weightsfilename))
    else:
      print('Pre-trained weights was not found in:', pretrained_weightsfilename)
      self._engine.load_weights(_weights.glorot_init(self.no_input_channels, model_cfg,
                                                     H=self.inputShape[0], W=self.inputShape[1]))

  # ---- the feature bank ----------------------------------------------------------------------
  @property
  def feature_volumes(self):
    """Host view of the bank: a list of (1,360,128) arrays after ``infer_multiple`` calls, an
    (n,1,360,128) array after ``infer_multiple_vs_multiple`` -- like infer.py:185,220."""
    host = self._bank[:self._bank_n].cpu().numpy()[:, None, :, :]
    return host if self._fv_as_array else list(host)

  @feature_volumes.setter
  def feature_volumes(self, value):
    arr = np.asarray(value, dtype=np.float32).reshape(-1, self.network_output_size, FEAT_C)
    self._set_bank(torch.from_numpy(arr).to(self._engine.device))
    self._fv_as_array = isinstance(value, np.ndarray)

  def _set_bank(self, fv):
    # the resident operand copies are keyed by the storage address: drop them before the old tensor can
    # be freed (and its address handed to another tensor by the caching allocator)
    self._engine.bank_release(None)
    self._bank = fv.contiguous()
    self._bank_n = int(fv.shape[0])
    if self._bank_n:
      self._engine.bank_prepare(self._bank, 0, self._bank_n)      # resident tensor-core operand copies

  def _append_bank(self, fv):
    n = int(fv.shape[0])
    if self._bank_n + n > self._bank.shape[0]:
      cap = max(1024, 2 * (self._bank_n + n))
      nb = torch.empty((cap, self.network_output_size, FEAT_C), dtype=torch.float32, device=self._engine.device)
      nb[:self._bank_n] = self._bank[:self._bank_n]
      self._engine.bank_release(None)                             # before the old storage is dropped
      self._bank = nb
      if self._bank_n:
        self._engine.bank_prepare(self._bank, 0, self._bank_n)    # new storage: rebuild the resident copies
    self._bank[self._bank_n:self._bank_n + n] = fv
    self._engine.bank_prepare(self._bank, self._bank_n, n)
    self._bank_n += n

  # ---- keras-model shims ---------------------------------------------------------------------
  def _leg_predict(self, x):
    x = x[0] if isinstance(x, (list, tuple)) else x
    xt = torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(self._engine.device)
    return self._engine.leg(xt).cpu().numpy()[:, None, :, :]

  def _head_predict(self, x):
    x1, x2 = x
    n = x1.shape[0]
    both = np.concatenate([np.asarray(x1, np.float32).reshape(n, -1, FEAT_C),
                           np.asarray(x2, np.float32).reshape(n, -1, FEAT_C)])
    bank = torch.from_numpy(both).to(self._engine.device)
    li = torch.arange(n, dtype=torch.int32)
    ov, _, corr = self._engine.heads(bank, li, li + n, want_corr=True)
    return [ov.cpu().numpy()[:, None], corr.cpu().numpy()]

  # ---- inference entry points ----------------------------------------------------------------
  def _run_heads(self, pair_indizes):
    """pairs[:,0] -> LEFT, pairs[:,1] -> RIGHT (ImagePairOverlapSequenceFeatureVolume.py:44-45).
    Returns model_outputs-like (overlap (n,1) f32, yaw (n,) int64)."""
    left = torch.from_numpy(np.ascontiguousarray(pair_indizes[:, 0], np.int32))
    right = torch.from_numpy(np.ascontiguousarray(pair_indizes[:, 1], np.int32))
    n = self._bank_n
    if len(pair_indizes) and (pair_indizes.min() < -n or pair_indizes.max() >= n):
      raise IndexError('index %d is out of bounds for axis 0 with size %d' % (int(pair_indizes.max()), n))
    left = torch.where(left < 0, left + n, left)               # numpy-style negative indices
    right = torch.where(right < 0, right + n, right)
    ov, yaw, _ = self._engine.heads(self._bank[:n], left, right)
    self._engine.check()                                       # deferred device errors -> exception, never garbage
    return ov.cpu().numpy()[:, None], yaw.cpu().numpy().astype(np.int64)

  def infer_one(self, filepath1, filepath2):
    """ Infer with one input pair (infer.py:124-160).  Returns [overlap (1,) f32, yaw (1,) int]. """
    if not filepath1.endswith('.bin') or not filepath2.endswith('.bin'):
      raise Exception('Please check the LiDAR file format, '
                      'this implementation currently only works with .bin files.')
    filename1 = os.path.basename(filepath1).replace('.bin', '')
    filename2 = os.path.basename(filepath2).replace('.bin', '')
    self.filenames = np.array([filename2, filename1])

    preprocess_data_folder = os.path.join(self.datasetpath, self.seq)
    if not os.path.isdir(preprocess_data_folder):
      raise Exception('Please first generate preprocessed input data.')

    fv = self._create_feature_volumes_device(self.filenames)
    ov, yaw, _ = self._engine.heads(fv, torch.tensor([0], dtype=torch.int32), torch.tensor([1], dtype=torch.int32))
    self._engine.check()
    overlap_out = ov.cpu().numpy()[:, None][0]                 # model_outputs[0][0]
    yaw_out = yaw.cpu().numpy().astype(np.int64)               # 180 - argmax, computed on device
    return overlap_out, yaw_out

  def infer_multiple(self, current_frame_id, reference_frame_id):
    """ Infer for loopclosing: the current frame versus old frames (infer.py:162-203). """
    filename = [str(current_frame_id).zfill(6)]
    self._append_bank(self._create_feature_volumes_device(filename)[:1])
    self._fv_as_array = False

    if len(reference_frame_id) > 0:
      pair_indizes = np.zeros((len(reference_frame_id), 2), dtype=int)
      pair_indizes[:, 1] = np.ones(len(reference_frame_id)) * current_frame_id
      pair_indizes[:, 0] = reference_frame_id
      overlap, yaw_out = self._run_heads(pair_indizes)
      overlap_out = overlap.squeeze()
      return overlap_out, yaw_out
    else:
      return None

  def infer_multiple_vs_multiple(self, file_names, first_idxs, second_idxs):
    """ Infer with multiple input pairs (infer.py:205-238). """
    if len(first_idxs) != len(second_idxs):
      raise Exception('Please make sure the first_idxs and second_idxs have the same size.')
    file_names = [os.path.basename(v).replace('.bin', '') for v in file_names]
    self._set_bank(self._create_feature_volumes_device(file_names))
    self._fv_as_array = True

    if len(second_idxs) > 0:
      pair_indizes = np.zeros((len(second_idxs), 2), dtype=int)
      pair_indizes[:, 1] = first_idxs
      pair_indizes[:, 0] = second_idxs
      overlap, yaw_out = self._run_heads(pair_indizes)
      overlap_out = overlap.squeeze()
      return overlap_out, yaw_out
    else:
      return None

  def create_feature_volumes(self, filenames):
    """ create feature volumes, thus execute the leg (infer.py:240-265).
        Returns: A n x 1 x 360 x 128 numpy array of feature volumes """
    return self._create_feature_volumes_device(filenames).cpu().numpy()[:, None, :, :]

  # ---- internals -----------------------------------------------------------------------------
  def _load_cue(self, sub, name, what):
    f = os.path.join(self.datasetpath, self.seq, sub, name + '.npy')
    try:
      return np.load(f)
    except IOError:
      if sub in ('probability', 'probability_pca', 'intensity'):
        # ImagePairOverlapOrientationSequence.py:183-191,201-205: second try with .npz
        return np.load(os.path.join(self.datasetpath, self.seq, sub, name + '.npz'))
      raise Exception('Could not read %s image %s' % (what, f))

  def _prepare_inputs(self, filenames):
    """Channel packing of prepareOneInput (ImagePairOverlapOrientationSequence.py:130-207):
    depth, normal, probabilities, intensity; raw values."""
    H, W = self.inputShape[0], self.inputShape[1]
    x = np.zeros((len(filenames), H, W, self.no_input_channels), dtype=np.float32)

    def load_one(i_name):
      i, name = i_name
      c = 0
      if self.use_depth:
        x[i, :, :, c] = self._load_cue('depth', name, 'depth')
        c += 1
      if self.use_normals:
        x[i, :, :, c:c + 3] = self._load_cue('normal', name, 'normal')
        c += 3
      if self.use_class_probabilities:
        if self.use_class_probabilities_pca:
          x[i, :, :, c:c + 3] = self._load_cue('probability_pca', name, 'probability')
          c += 3
        else:
          x[i, :, :, c:c + 20] = self._load_cue('probability', name, 'probability')
          c += 20
      if self.use_intensity:
        x[i, :, :, c] = self._load_cue('intensity', name, 'intensity')
        c += 1

    if len(filenames) <= 1:
      for item in enumerate(filenames):
        load_one(item)
    else:
      # the reference feeds predict_generator with 8 workers (infer.py:262); np.load releases the GIL in its
      # file reads, so a small thread pool keeps the GPU fed when thousands of scans are encoded (testing.py)
      from concurrent.futures import ThreadPoolExecutor
      with ThreadPoolExecutor(max_workers=min(8, len(filenames))) as ex:
        list(ex.map(load_one, enumerate(filenames)))     # list(): re-raise the first worker exception
    return x

  def _create_feature_volumes_device(self, filenames):
    outs = []
    bs = max(1, int(self.batch_size))
    filenames = list(filenames)
    for s in range(0, len(filenames), bs):
      x = self._prepare_inputs(filenames[s:s + bs])
      outs.append(self._engine.leg(torch.from_numpy(x).to(self._engine.device)))
    if not outs:
      return torch.empty((0, self.network_output_size, FEAT_C), dtype=torch.float32, device=self._engine.device)
    return torch.cat(outs)

  # ---- extensions: raw clouds in, no .npy round trip -----------------------------------------
  def encode_clouds(self, clouds, probs=None):
    """list of (N,4) float32 raw clouds -> device feature volumes [n,360,128] through the fused
    projection + normal + packing kernels, every cue as the reference's .npy files give it.  A config with class
    probabilities needs ``probs``: one (N, 20) -- (N, 3) with use_class_probabilities_pca -- float32 array per
    cloud, the per-point scores a .label file holds (gen_semantic_data.py:33); other configs refuse them."""
    n_prob = self._engine.n_prob
    if self.use_class_probabilities and probs is None:
      raise Exception('encode_clouds: semantic probabilities need per-point class scores (probs)')
    if probs is not None:
      if not self.use_class_probabilities:
        raise Exception('encode_clouds: class probabilities given, but the config does not use them')
      if len(probs) != len(clouds):
        raise Exception('encode_clouds: %d probability arrays for %d clouds' % (len(probs), len(clouds)))
      probs = [check_probs(p, np.shape(c)[0], n_prob, 'encode_clouds') for c, p in zip(clouds, probs)]
      probs = np.concatenate([np.asarray(p, np.float32) for p in probs]) if probs else np.zeros((0, n_prob), np.float32)
    batch = self._engine.upload_clouds(clouds)
    return self._engine.leg(self._engine.preprocess_cues(batch, probs))

  def infer_one_raw(self, filepath1, filepath2, labels1=None, labels2=None):
    """Like ``infer_one`` but reads the raw .bin scans (LEFT = file2, RIGHT = file1).  A config with class
    probabilities also reads each scan's .label file of per-point scores, as gen_semantic_data.py:33 does."""
    if not filepath1.endswith('.bin') or not filepath2.endswith('.bin'):
      raise Exception('Please check the LiDAR file format, '
                      'this implementation currently only works with .bin files.')
    clouds = [np.fromfile(p, dtype=np.float32).reshape((-1, 4)) for p in (filepath2, filepath1)]
    probs = None
    if labels1 is not None or labels2 is not None:
      if labels1 is None or labels2 is None:
        raise Exception('infer_one_raw: give the .label files of both scans')
      probs = [np.fromfile(p, dtype=np.float32).reshape((-1, self._engine.n_prob or 20)) for p in (labels2, labels1)]
    fv = self.encode_clouds(clouds, probs)
    ov, yaw, _ = self._engine.heads(fv, torch.tensor([0], dtype=torch.int32), torch.tensor([1], dtype=torch.int32))
    self._engine.check()
    return ov.cpu().numpy(), yaw.cpu().numpy().astype(np.int64)
