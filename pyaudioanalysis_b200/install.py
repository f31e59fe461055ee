"""Rebind the reference's module attributes to the GPU path.

Every caller in the reference looks the four functions up on the module object at call time
(MidTermFeatures.py:93-95; audioSegmentation.py:371,423,482,573,707,842,1137; audioTrainTest.py:
1081,1128; audioAnalysis.py:46,71,80), so setattr on the imported modules is the drop-in.
"""
_saved = {}


def install(pyaudioanalysis_pkg=None, precision=None):
    """Patch an importable ``pyAudioAnalysis``; returns the list of attributes rebound.  ``precision`` ("float32" /
    "float64", None: leave it as it is) sets the drop-ins' result contract (``precision.set_precision``)."""
    from . import ShortTermFeatures as ours_st, MidTermFeatures as ours_mt
    if precision is not None:
        from .precision import set_precision
        set_precision(precision)
    if pyaudioanalysis_pkg is None:
        import importlib
        ref_st = importlib.import_module("pyAudioAnalysis.ShortTermFeatures")
        ref_mt = importlib.import_module("pyAudioAnalysis.MidTermFeatures")
    else:
        ref_st, ref_mt = pyaudioanalysis_pkg.ShortTermFeatures, pyaudioanalysis_pkg.MidTermFeatures
    done = []
    for mod, ours, names in ((ref_st, ours_st, ("feature_extraction", "spectrogram", "chromagram")),
                             (ref_mt, ours_mt, ("mid_feature_extraction", "beat_extraction", "directory_feature_extraction",
                                                "multiple_directory_feature_extraction", "directory_feature_extraction_no_avg",
                                                "mid_feature_extraction_to_file", "mid_feature_extraction_file_dir"))):
        for n in names:
            _saved.setdefault((mod, n), getattr(mod, n))
            setattr(mod, n, getattr(ours, n))
            done.append("%s.%s" % (mod.__name__, n))
    return done


def install_training(audio_train_test=None):
    """Rebind an importable ``pyAudioAnalysis.audioTrainTest`` (or the module given) so that its evaluate_classifier runs
    the kNN model selection on the GPU (``audioTrainTest.evaluate_classifier`` here) and every other classifier, SMOTE
    and non-finite input through the saved original.  extract_features_and_train looks the function up on the module at
    call time (audioTrainTest.py:309), so it trains kNN models through the GPU unchanged.  train_random_forest and
    train_extra_trees and train_gradient_boosting, where the module has them, are rebound to the GPU trainers here
    (kernel 13): the final forest or boosting model extract_features_and_train fits and pickles is built on the GPU, tree
    for tree scikit-learn's.  Likewise, where the
    module has them, evaluate_regression (its "randomforest" model selection on the GPU, every other method through the
    saved original) and train_random_forest_regression, so feature_extraction_train_regression selects and fits its
    forest on the GPU.  Returns the attributes rebound."""
    from .audioTrainTest import dispatcher
    if audio_train_test is None:
        import importlib
        audio_train_test = importlib.import_module("pyAudioAnalysis.audioTrainTest")
    original = _saved.setdefault((audio_train_test, "evaluate_classifier"), audio_train_test.evaluate_classifier)
    audio_train_test.evaluate_classifier = dispatcher(original)
    done = ["%s.evaluate_classifier" % audio_train_test.__name__]
    from . import audioTrainTest as ours
    for n in ("train_random_forest", "train_extra_trees", "train_gradient_boosting"):
        if not hasattr(audio_train_test, n):
            continue
        _saved.setdefault((audio_train_test, n), getattr(audio_train_test, n))
        setattr(audio_train_test, n, getattr(ours, n))
        done.append("%s.%s" % (audio_train_test.__name__, n))
    if hasattr(audio_train_test, "evaluate_regression"):
        original = _saved.setdefault((audio_train_test, "evaluate_regression"), audio_train_test.evaluate_regression)
        audio_train_test.evaluate_regression = ours.regression_dispatcher(original)
        done.append("%s.evaluate_regression" % audio_train_test.__name__)
    if hasattr(audio_train_test, "train_random_forest_regression"):
        n = "train_random_forest_regression"
        _saved.setdefault((audio_train_test, n), getattr(audio_train_test, n))
        setattr(audio_train_test, n, ours.train_random_forest_regression)
        done.append("%s.%s" % (audio_train_test.__name__, n))
    return done


def install_segmentation(audio_segmentation=None):
    """Rebind an importable ``pyAudioAnalysis.audioSegmentation`` (or the module given) to the HMM segmentation here
    (``audioSegmentation``: training statistics and decode on the GPU, no hmmlearn needed at run time): the two
    trainers, hmm_segmentation, train_hmm_compute_statistics, and evaluate_segmentation_classification_dir through a
    dispatcher that sends the classifier methods to the saved original.  Returns the attributes rebound."""
    from . import audioSegmentation as ours
    if audio_segmentation is None:
        import importlib
        audio_segmentation = importlib.import_module("pyAudioAnalysis.audioSegmentation")
    done = []
    for n in ("train_hmm_compute_statistics", "train_hmm_from_file", "train_hmm_from_directory", "hmm_segmentation"):
        _saved.setdefault((audio_segmentation, n), getattr(audio_segmentation, n))
        setattr(audio_segmentation, n, getattr(ours, n))
        done.append("%s.%s" % (audio_segmentation.__name__, n))
    n = "evaluate_segmentation_classification_dir"
    original = _saved.setdefault((audio_segmentation, n), getattr(audio_segmentation, n))
    setattr(audio_segmentation, n, ours.dispatcher(original))
    return done + ["%s.%s" % (audio_segmentation.__name__, n)]


def install_diarization(audio_segmentation=None):
    """Rebind an importable ``pyAudioAnalysis.audioSegmentation`` (or the module given) to the speaker diarization here
    (``audioSegmentation.diarize``: the silhouette means on kernel 9, the HMM smoothing on kernel 7): speaker_diarization,
    speaker_diarization_evaluation and evaluate_speaker_diarization.  Returns the attributes rebound."""
    from . import audioSegmentation as ours
    if audio_segmentation is None:
        import importlib
        audio_segmentation = importlib.import_module("pyAudioAnalysis.audioSegmentation")
    done = []
    for n in ("speaker_diarization", "speaker_diarization_evaluation", "evaluate_speaker_diarization"):
        _saved.setdefault((audio_segmentation, n), getattr(audio_segmentation, n))
        setattr(audio_segmentation, n, getattr(ours, n))
        done.append("%s.%s" % (audio_segmentation.__name__, n))
    return done


def install_thumbnailing(audio_segmentation=None):
    """Rebind an importable ``pyAudioAnalysis.audioSegmentation`` (or the module given) to the music thumbnails here
    (``audioSegmentation.music_thumbnailing``: the similarity matrix, filter, masks, argmax and walk on kernel 10):
    music_thumbnailing and self_similarity_matrix.  Returns the attributes rebound."""
    from . import audioSegmentation as ours
    if audio_segmentation is None:
        import importlib
        audio_segmentation = importlib.import_module("pyAudioAnalysis.audioSegmentation")
    done = []
    for n in ("music_thumbnailing", "self_similarity_matrix"):
        _saved.setdefault((audio_segmentation, n), getattr(audio_segmentation, n))
        setattr(audio_segmentation, n, getattr(ours, n))
        done.append("%s.%s" % (audio_segmentation.__name__, n))
    return done


def uninstall():
    for (mod, n), fn in list(_saved.items()):
        setattr(mod, n, fn)
    _saved.clear()
