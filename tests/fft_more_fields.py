"""Fr FFT constants of bls24-315, bls24-317, bw6-633 and bw6-761 for the oracle's FFT restatement (TEST INFRASTRUCTURE).

fr.Generator's rootOfUnity and maxOrderRoot (ecc/{bls24-315,bls24-317,bw6-633,bw6-761}/fr/generator.go:23-24) and
GeneratorFullMultiplicativeGroup (fr/fft/domain.go:59), in the layout of oracle.FFT_PARAMS.  `FFTDomain` is the oracle's
fft.Domain restatement (its DIF / DIT / coset transforms) built from these constants."""
from oracle import oracle as O

FFT_PARAMS = {
    "bls24315_fr": dict(root=1792993287828780812362846131493071959406149719416102105453370749552622525216, max_order=22, mult_gen=7),
    "bls24317_fr": dict(root=16532287748948254263922689505213135976137839535221842169193829039521719560631, max_order=60, mult_gen=7),
    "bw6633_fr": dict(root=4991787701895089137426454739366935169846548798279261157172811661565882460884369603588700158257,
                      max_order=20, mult_gen=13),
    "bw6761_fr": dict(root=32863578547254505029601261939868325669770508939375122462904745766352256812585773382134936404344547323199885654433,
                      max_order=46, mult_gen=15),
}


class FFTDomain(O.FFTDomain):
    """fft.Domain / NewDomain (domain.go:24-110) over one of the four fields above; the transforms are the oracle's"""

    def __init__(self, frname: str, m: int, shift: int = None):
        P = FFT_PARAMS[frname]
        self.q = O.FIELDS[frname].q
        x = 1
        while x < m:
            x <<= 1
        self.cardinality = x
        logx = x.bit_length() - 1
        if logx > P["max_order"]:
            raise ValueError("m (%d) is too big: the required root of unity does not exist" % m)
        self.generator = pow(P["root"], 1 << (P["max_order"] - logx), self.q)
        self.generator_inv = pow(self.generator, -1, self.q)
        self.cardinality_inv = pow(x, -1, self.q)
        self.shift = P["mult_gen"] if shift is None else shift % self.q
        self.shift_inv = pow(self.shift, -1, self.q)
