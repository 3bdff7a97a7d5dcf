"""The checks the CPU censuses share.  A census maps every key a product plan reaches (a code path of a kernel, keyed by the
fields that select it) to one place that reaches it, {key: where}, and every GPU parity case to the keys its plans reach,
{case id: keys}; the checks below then ask that every product key is reached by a case, and that each case a census added
reaches a key no other case reaches."""
import collections


def first_where(pairs):
    """{key: where} from (key, where) pairs: the first place that reaches each key."""
    found = collections.OrderedDict()
    for key, where in pairs:
        found.setdefault(key, where)
    return found


def _listing(keys):
    return '\n'.join('  %s  e.g. %s' % (tuple(k), where) for k, where in keys)


def assert_reached(what, keys, cases):
    """Every key of {key: where} is reached by a case of {case id: keys}."""
    reached = set().union(*cases.values())
    missing = [(k, where) for k, where in keys.items() if k not in reached]
    assert not missing, '%d %s are reached by no GPU parity case:\n%s' % (len(missing), what, _listing(missing))


def own_keys(name, keys, cases):
    """The keys of `keys` that case `name` reaches and no other case of {case id: keys} reaches."""
    others = set().union(*(ks for n, ks in cases.items() if n != name))
    return cases[name] & set(keys) - others


def assert_needed(names, levels):
    """Each case of the list `names` reaches a key of its own at one of the levels [(keys, cases)] it belongs to, so that
    deleting it fails the census.  A case listed twice has no key of its own."""
    for name in names:
        assert names.count(name) == 1 and any(own_keys(name, keys, cases) for keys, cases in levels if name in cases), \
            '%s reaches no key of its own' % name


def assert_unreached_listed(keys, cases, unreached):
    """Every key of {key: reason} is reached by a case and by no product plan, and every case key is a product key or listed."""
    prod, listed = set(keys), set(unreached)
    reached = set().union(*cases.values())
    assert not listed & prod, sorted(listed & prod)
    assert listed <= reached, sorted(listed - reached)
    unlisted = sorted((name, tuple(k)) for name, ks in cases.items() for k in ks - prod - listed)
    assert not unlisted, 'case keys no product reaches and the census does not list: %s' % unlisted
