"""`QRec`: loads the data named by a ModelConf, partitions it and runs the model
(reference: QRec.py:8-118).  Model classes are resolved by name, model.rating first and then
model.ranking like the reference (QRec.py:51-56)."""
import importlib
import sys
from time import strftime, localtime, time

from .util.config import OptionConf
from .util.dataSplit import DataSplit
from .util.io import FileIO


def _model_class(name):
    try:
        mod = importlib.import_module('qrec_b200.model.rating.' + name)
    except ImportError:
        try:
            mod = importlib.import_module('qrec_b200.model.ranking.' + name)
        except ImportError as e:
            print('model %s is not available on the H100 engine (%s)' % (name, e))
            sys.exit(-1)
    return getattr(mod, name)


class QRec(object):
    def __init__(self, config):
        self.trainingData, self.testData, self.relation, self.measure = [], [], [], []
        self.config = config
        self.ratingConfig = OptionConf(config['ratings.setup'])
        if not self.config.contains('evaluation.setup'):
            print('Wrong configuration of evaluation!')
            sys.exit(-1)
        ev = self.evaluation = OptionConf(config['evaluation.setup'])
        binarized, bottom = ev.contains('-b'), float(ev['-b']) if ev.contains('-b') else 0
        load = lambda path, test=False: FileIO.loadDataSet(config, path, bTest=test, binarized=binarized, threshold=bottom)  # noqa: E731
        if ev.contains('-testSet'):
            self.trainingData = load(config['ratings'])
            self.testData = load(ev['-testSet'], True)
        elif ev.contains('-ap'):
            self.trainingData, self.testData = DataSplit.dataSplit(load(config['ratings']), test_ratio=float(ev['-ap']),
                                                                   binarized=binarized)
        elif ev.contains('-cv'):
            self.trainingData = load(config['ratings'])
        elif ev.contains('-predict'):
            self.trainingData = load(config['ratings'])
            self.testData = FileIO.loadUserList(ev['-predict'])
        if config.contains('social'):                                       # QRec.py:44-46
            self.socialConfig = OptionConf(self.config['social.setup'])
            self.relation = FileIO.loadRelationship(config, self.config['social'])
        print('Reading data and preprocessing...')

    def execute(self):
        cls = _model_class(self.config['model.name'])
        ev = self.evaluation
        if not ev.contains('-cv'):
            if self.config.contains('social'):                              # QRec.py:110-113
                self.measure = cls(self.config, self.trainingData, self.testData, self.relation).execute()
            else:
                self.measure = cls(self.config, self.trainingData, self.testData).execute()
            return self.measure
        k = int(ev['-cv'])
        if k < 2 or k > 10:
            print("k for cross-validation should not be greater than 10 or less than 2")
            sys.exit(-1)
        folds = []
        for n, (train, test) in enumerate(DataSplit.crossValidation(self.trainingData, k, binarized=ev.contains('-b')), 1):
            fold = '[' + str(n) + ']'
            model = (cls(self.config, train, test, self.relation, fold) if self.config.contains('social')
                     else cls(self.config, train, test, fold))
            folds.append(model.execute())                               # one GPU: folds run in turn
        self.measure = folds
        res = []
        for pos, line in enumerate(folds[0]):
            if line[:3] == 'Top':
                res.append(line)
                continue
            total = 0                                  # left-to-right `+=` like the reference (builtin sum() is compensated on 3.12)
            for f in folds:
                total += float(f[pos].split(':')[1])
            res.append(line.split(':')[0] + ':' + str(total / k) + '\n')
        stamp = strftime("%Y-%m-%d %H-%M-%S", localtime(time()))
        FileIO.writeFile(OptionConf(self.config['output.setup'])['-dir'],
                         self.config['model.name'] + '@' + stamp + '-' + str(k) + '-fold-cv' + '.txt', res)
        print('The result of %d-fold cross validation:\n%s' % (k, ''.join(res)))
        return res
