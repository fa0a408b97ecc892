"""mortal_b200.dataloader.batch_schedule against the reference's FileDatasetsIter restated over integer entries: load_files'
file-list shuffle, populate_buffer, the reserve_ratio split and the final shuffle, wrapped in torch's DataLoader. For the same
random.seed both give the same sample ids in the same batches, and leave `random` in the same state."""
import random

import pytest
import torch
from torch.utils.data import DataLoader, IterableDataset

from mortal_b200.dataloader import batch_schedule


class RefIter(IterableDataset):
    """mortal/dataloader.py FileDatasetsIter with populate_buffer appending the next `count(file)` integer ids"""

    def __init__(self, file_list, counts, file_batch_size, reserve_ratio, num_epochs, enable_augmentation, augmented_first):
        super().__init__()
        self.file_list, self.counts = file_list, counts
        self.file_batch_size, self.reserve_ratio, self.num_epochs = file_batch_size, reserve_ratio, num_epochs
        self.enable_augmentation, self.augmented_first = enable_augmentation, augmented_first
        self.next_id = 0
        self.iterator = None

    def build_iter(self):
        for _ in range(self.num_epochs):
            yield from self.load_files(self.augmented_first)
            if self.enable_augmentation:
                yield from self.load_files(not self.augmented_first)

    def load_files(self, augmented):
        random.shuffle(self.file_list)
        self.buffer = []
        for start_idx in range(0, len(self.file_list), self.file_batch_size):
            old_buffer_size = len(self.buffer)
            self.populate_buffer(self.file_list[start_idx:start_idx + self.file_batch_size], augmented)
            buffer_size = len(self.buffer)
            reserved_size = int((buffer_size - old_buffer_size) * self.reserve_ratio)
            if reserved_size > buffer_size:
                continue
            random.shuffle(self.buffer)
            yield from self.buffer[reserved_size:]
            del self.buffer[reserved_size:]
        random.shuffle(self.buffer)
        yield from self.buffer
        self.buffer.clear()

    def populate_buffer(self, file_list, augmented):
        for f in file_list:
            n = self.counts[f, augmented]
            self.buffer.extend(range(self.next_id, self.next_id + n))
            self.next_id += n

    def __iter__(self):
        if self.iterator is None:
            self.iterator = self.build_iter()
        return self.iterator


def _device_side(file_list, counts, file_batch_size, reserve_ratio, num_epochs, enable_augmentation, augmented_first, batch_size):
    """the order function fed as FileDatasetsIter feeds it: one pass per load_files, its file-list shuffle when it starts"""
    def one_pass(augmented):
        random.shuffle(file_list)
        for s in range(0, len(file_list), file_batch_size):
            yield sum(counts[f, augmented] for f in file_list[s:s + file_batch_size])

    def passes():
        for _ in range(num_epochs):
            yield one_pass(augmented_first)
            if enable_augmentation:
                yield one_pass(not augmented_first)

    return list(batch_schedule(passes(), reserve_ratio, batch_size))


CASES = [  # (files, file_batch_size, reserve_ratio, num_epochs, enable_augmentation, augmented_first, batch_size)
    (23, 4, 0, 1, False, False, 16),
    (23, 4, 0.3, 1, False, False, 7),
    (23, 4, 0.9, 2, False, False, 50),
    (23, 4, 1.5, 2, False, False, 13),
    (17, 5, 0.3, 2, True, False, 8),
    (17, 5, 0.9, 1, True, True, 1),
    (20, 20, 0, 2, True, True, 1000),
    (12, 3, 0.5, 2, False, False, 4),
]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("seed", [0, 1])
def test_schedule_equals_reference(case, seed):
    n_files, fbs, ratio, epochs, aug, aug_first, bs = case
    rng = random.Random(seed * 100 + n_files)
    # file sizes 0..40 with plenty of empty files, so that whole file batches come out empty too
    counts = {(f, a): (0 if rng.random() < 0.3 else rng.randrange(41)) for f in range(n_files) for a in (False, True)}
    for f in range(0, n_files, 3):
        counts[f, False] = counts[f, True] = 0
    random.seed(seed)
    files = list(range(n_files))
    ref = [b.tolist() for b in DataLoader(RefIter(files, counts, fbs, ratio, epochs, aug, aug_first), batch_size=bs,
                                          drop_last=False, num_workers=0)]
    state = random.getstate()
    random.seed(seed)
    files2 = list(range(n_files))
    got = _device_side(files2, counts, fbs, ratio, epochs, aug, aug_first, bs)
    assert got == ref
    assert files2 == files and random.getstate() == state
    total = sum(counts[f, a] for f in range(n_files) for a in ((False, True) if aug else (aug_first,))) * epochs
    assert sorted(i for b in got for i in b) == list(range(total))
    assert all(len(b) == bs for b in got[:-1]) and 0 < len(got[-1]) <= bs if got else total == 0


def test_empty_run_and_bad_batch_size():
    assert list(batch_schedule([[0, 0], []], 0.5, 4)) == []
    with pytest.raises(ValueError):
        list(batch_schedule([[1]], 0, 0))


def test_batches_are_cut_before_the_next_load():
    """a batch is handed out before the file batch that follows it is loaded (the reference's generator runs just as far)"""
    log = []

    def counts():
        for n in (8, 8):
            log.append(("load", n))
            yield n

    random.seed(3)
    for b in batch_schedule([counts()], 0, 4):
        log.append(("batch", len(b)))
    assert log == [("load", 8), ("batch", 4), ("batch", 4), ("load", 8), ("batch", 4), ("batch", 4)]


def test_collated_ids_match_tensor_collation():
    """DataLoader's collation of integer entries is what the reference's batches of ids look like"""
    b = next(iter(DataLoader(RefIter([0], {(0, False): 5, (0, True): 0}, 1, 0, 1, False, False), batch_size=3)))
    assert b.dtype == torch.int64 and len(b) == 3
