"""Image datasets of the reference's training/dataset.py (:26-250): Dataset and ImageFolderDataset, which the metrics read real images
through (calc_metrics.py names the class 'training.dataset.ImageFolderDataset').

ImageFolderDataset reads a directory or a zip of images: the file names sorted; with non_rebalance (the default) only names whose
last eight digits before the extension are below 140000 (FFHQ's originals, not its rebalanced copies); labels from
dataset_eric_orig.json, with the camera rows' y and z axes negated (OpenCV -> OpenGL: entries 1, 2, 5, 6, 9, 10).  Dataset applies
max_size (a RandomState(random_seed) subset, kept sorted) and then xflip (the items again, mirrored).
"""

import json
import os
import zipfile

import numpy as np
import PIL.Image
import torch

from .. import dnnlib

_OPENCV_TO_OPENGL = [1, 2, 5, 6, 9, 10]


class Dataset(torch.utils.data.Dataset):
    def __init__(self, name, raw_shape, max_size=None, use_labels=False, xflip=False, random_seed=0):
        self._name = name
        self._raw_shape = list(raw_shape)
        self._use_labels = use_labels
        self._raw_labels = None
        self._label_shape = None
        idx = np.arange(self._raw_shape[0], dtype=np.int64)
        if max_size is not None and idx.size > max_size:
            np.random.RandomState(random_seed).shuffle(idx)
            idx = np.sort(idx[:max_size])
        flip = np.zeros(idx.size, dtype=np.uint8)
        if xflip:
            idx, flip = np.tile(idx, 2), np.concatenate([flip, np.ones_like(flip)])
        self._raw_idx, self._xflip = idx, flip

    def _get_raw_labels(self):
        if self._raw_labels is None:
            labels = self._load_raw_labels() if self._use_labels else None
            if labels is None:
                labels = np.zeros([self._raw_shape[0], 0], dtype=np.float32)
            if not (isinstance(labels, np.ndarray) and labels.shape[0] == self._raw_shape[0] and labels.dtype in (np.float32, np.int64)):
                raise ValueError(f'dataset labels must be float32 or int64 with one row per image, got {getattr(labels, "shape", None)}')
            if labels.dtype == np.int64 and (labels.ndim != 1 or np.any(labels < 0)):
                raise ValueError('integer labels must be non-negative class indices')
            self._raw_labels = labels
        return self._raw_labels

    def close(self):
        pass

    def _load_raw_image(self, raw_idx):
        raise NotImplementedError

    def _load_raw_labels(self):
        raise NotImplementedError

    def __getstate__(self):
        return dict(self.__dict__, _raw_labels=None)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __len__(self):
        return self._raw_idx.size

    def __getitem__(self, idx):
        image = self._load_raw_image(self._raw_idx[idx])
        if not (isinstance(image, np.ndarray) and list(image.shape) == self.image_shape and image.dtype == np.uint8):
            raise ValueError(f'image {idx}: expected uint8 {self.image_shape}, got {getattr(image, "dtype", None)} {getattr(image, "shape", None)}')
        if self._xflip[idx]:
            image = image[:, :, ::-1]
        return image.copy(), self.get_label(idx)

    def get_label(self, idx):
        label = self._get_raw_labels()[self._raw_idx[idx]]
        if label.dtype == np.int64:
            onehot = np.zeros(self.label_shape, dtype=np.float32)
            onehot[label] = 1
            label = onehot
        return label.copy()

    def get_details(self, idx):
        raw = int(self._raw_idx[idx])
        return dnnlib.EasyDict(raw_idx=raw, xflip=int(self._xflip[idx]) != 0, raw_label=self._get_raw_labels()[raw].copy())

    @property
    def name(self):
        return self._name

    @property
    def image_shape(self):
        return list(self._raw_shape[1:])

    @property
    def num_channels(self):
        return self.image_shape[0]

    @property
    def resolution(self):
        if self.image_shape[1] != self.image_shape[2]:
            raise ValueError(f'images are not square: {self.image_shape}')
        return self.image_shape[1]

    @property
    def label_shape(self):
        if self._label_shape is None:
            raw = self._get_raw_labels()
            self._label_shape = [int(np.max(raw)) + 1] if raw.dtype == np.int64 else raw.shape[1:]
        return list(self._label_shape)

    @property
    def label_dim(self):
        return self.label_shape[0]

    @property
    def has_labels(self):
        return any(x != 0 for x in self.label_shape)

    @property
    def has_onehot_labels(self):
        return self._get_raw_labels().dtype == np.int64


class ImageFolderDataset(Dataset):
    def __init__(self, path, resolution=None, non_rebalance=True, **super_kwargs):
        self._path = path
        self._zipfile = None
        if os.path.isdir(path):
            self._type = 'dir'
            self._all_fnames = {os.path.relpath(os.path.join(root, f), start=path) for root, _dirs, files in os.walk(path) for f in files}
        elif self._file_ext(path) == '.zip':
            self._type = 'zip'
            self._all_fnames = set(self._get_zipfile().namelist())
        else:
            raise IOError('Path must point to a directory or zip')
        PIL.Image.init()
        fnames = sorted(f for f in self._all_fnames if self._file_ext(f) in PIL.Image.EXTENSION)
        if non_rebalance:
            fnames = [f for f in fnames if int(f[-12:-4]) < 140000]
        if not fnames:
            raise IOError('No image files found in the specified path')
        self._image_fnames = fnames
        raw_shape = [len(fnames)] + list(self._load_raw_image(0, resolution).shape)
        if resolution is not None and (raw_shape[2] != resolution or raw_shape[3] != resolution):
            raise IOError('Image files do not match the specified resolution')
        super().__init__(name=os.path.splitext(os.path.basename(path))[0], raw_shape=raw_shape, **super_kwargs)

    @staticmethod
    def _file_ext(fname):
        return os.path.splitext(fname)[1].lower()

    def _get_zipfile(self):
        if self._zipfile is None:
            self._zipfile = zipfile.ZipFile(self._path)
        return self._zipfile

    def _open_file(self, fname):
        if self._type == 'dir':
            return open(os.path.join(self._path, fname), 'rb')
        return self._get_zipfile().open(fname, 'r')

    def close(self):
        try:
            if self._zipfile is not None:
                self._zipfile.close()
        finally:
            self._zipfile = None

    def __getstate__(self):
        return dict(super().__getstate__(), _zipfile=None)

    def _load_raw_image(self, raw_idx, resolution=None):
        with self._open_file(self._image_fnames[raw_idx]) as f:
            image = PIL.Image.open(f)
            if resolution:
                image = image.resize((resolution, resolution))
            image = np.array(image)
        if image.ndim == 2:
            image = image[:, :, np.newaxis]
        return image.transpose(2, 0, 1)

    def _load_raw_labels(self):
        fname = 'dataset_eric_orig.json'
        if fname not in self._all_fnames:
            return None
        with self._open_file(fname) as f:
            labels = json.load(f)['labels']
        if labels is None:
            return None
        labels = dict(labels)
        labels = np.array([labels[f.replace('\\', '/')] for f in self._image_fnames])
        labels[:, _OPENCV_TO_OPENGL] *= -1
        return labels.astype({1: np.int64, 2: np.float32}[labels.ndim])
