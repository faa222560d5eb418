"""Host-side SegTrackV2 reader (SURVEY 8f-2): the reference's data/segtrackv2_data_utils.py:11-308 restated on top of the
DAVIS2016 reader's numpy/OpenCV pipeline (preprocessing, pair sampling, augmentation and test ordering are the same code in
the reference; only the folder layout differs and there is a single partition).

Folder contract: `<root>/ImageSets/all.txt` lists the sequences with one leading marker character per line (:25-26);
`ImageSets/<seq>.txt` lists the frame names after a header line (:56); frames are `JPEGImages/<seq>/<name>.png`, masks
`GroundTruth/<seq>/<name>.png`.
"""
import os

from .davis2016_data_utils import Davis2016Reader


class DirectoryIterator(object):
    """segtrackv2_data_utils.py:11-70."""

    def __init__(self, directory):
        self.directory = directory
        all_files = os.path.join(directory, 'ImageSets/all.txt')
        self.image_dirs = os.path.join(directory, 'JPEGImages')
        self.annotation_dir = os.path.join(directory, 'GroundTruth')
        if not os.path.isfile(all_files):
            raise IOError("Division file not found")
        with open(all_files) as f:
            self.components = [l.split()[0][1:] for l in f.read().splitlines() if l.strip()]
        self.samples = 0
        self.num_experiments = 0
        self.image_filenames, self.annotation_filenames = [], []
        for experiment in self.components:
            self._parse_experiment(experiment)
            self.num_experiments += 1
        if self.samples == 0:
            raise IOError("Did not find any file in the dataset folder")
        assert self.num_experiments == len(self.image_filenames), "Reading failed"
        print('Found {} images belonging to {} experiments.'.format(self.samples, self.num_experiments))

    def _parse_experiment(self, experiment):
        exp_file = os.path.join(self.directory, 'ImageSets', experiment + '.txt')
        assert os.path.isfile(exp_file), "Experiment {} not found".format(exp_file)
        with open(exp_file) as f:
            names = [l.split()[0] for l in f.read().splitlines()[1:] if l.strip()]
        cur_f, cur_a = [], []
        for n in names:
            cur_f.append(os.path.join(self.image_dirs, experiment, n + '.png'))
            assert os.path.isfile(cur_f[-1]), "Not found image {}".format(cur_f[-1])
            cur_a.append(os.path.join(self.annotation_dir, experiment, n + '.png'))
            assert os.path.isfile(cur_a[-1]), "Not found image {}".format(cur_a[-1])
            self.samples += 1
        self.image_filenames.append(cur_f)
        self.annotation_filenames.append(cur_a)


class SegTrackV2Reader(Davis2016Reader):
    """segtrackv2_data_utils.py:73-308 (no partitions: training and evaluation both walk the whole dataset)."""

    def __init__(self, root_dir, max_temporal_len=3, min_temporal_len=2, num_threads=6, seed=8964, flow_dir=''):
        Davis2016Reader.__init__(self, root_dir, max_temporal_len, min_temporal_len, num_threads, seed, flow_dir)

    def get_filenames_list(self, partition=None):
        it = DirectoryIterator(self.root_dir)
        self.val_samples = it.samples
        return it.image_filenames, it.annotation_filenames

    def image_inputs(self, batch_size=32, train_crop=1.0, num_threads=6, partition=None):
        return Davis2016Reader.image_inputs(self, batch_size=batch_size, partition=None, train_crop=train_crop)

    def test_inputs(self, batch_size=32, t_len=2, with_fname=False, test_crop=1.0, partition=None):
        return Davis2016Reader.test_inputs(self, batch_size=batch_size, partition=None, t_len=t_len, with_fname=with_fname,
                                           test_crop=test_crop)
