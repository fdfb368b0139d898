//go:build b200

package groth16_test

import (
	"testing"

	b200_groth16 "github.com/consensys/gnark/backend/accelerated/b200/groth16"
	"github.com/consensys/gnark/backend/witness"
	"github.com/consensys/gnark/frontend"
	"github.com/consensys/gnark/frontend/cs/r1cs"
	"github.com/consensys/gnark/test"
)

// Several witnesses of one circuit proven in one ProveBatch call, plain and committing: every proof verifies against its
// own public witness.
func TestProveBatch(t *testing.T) {
	for _, curve := range curves {
		assert := test.NewAssert(t)
		ccs, err := frontend.Compile(curve.ScalarField(), r1cs.NewBuilder, &circuit{})
		assert.NoError(err)
		pk, vk, err := b200_groth16.Setup(ccs)
		assert.NoError(err)
		var full, public []witness.Witness
		for i := 1; i <= 5; i++ {
			w, err := frontend.NewWitness(&circuit{A: i, B: i + 2, Res: i * (i + 2)}, curve.ScalarField())
			assert.NoError(err)
			pw, err := w.Public()
			assert.NoError(err)
			full, public = append(full, w), append(public, pw)
		}
		proofs, err := b200_groth16.ProveBatch(ccs, pk, full)
		assert.NoError(err)
		assert.Equal(len(full), len(proofs))
		for i, p := range proofs {
			assert.NoError(b200_groth16.Verify(p, vk, public[i]), curve.String(), i)
		}

		ccs, err = frontend.Compile(curve.ScalarField(), r1cs.NewBuilder, &commitCircuit{})
		assert.NoError(err)
		pk, vk, err = b200_groth16.Setup(ccs)
		assert.NoError(err)
		w, err := frontend.NewWitness(&commitCircuit{One: 1, Two: 2}, curve.ScalarField())
		assert.NoError(err)
		pw, err := w.Public()
		assert.NoError(err)
		proofs, err = b200_groth16.ProveBatch(ccs, pk, []witness.Witness{w, w, w})
		assert.NoError(err)
		for _, p := range proofs {
			assert.NoError(b200_groth16.Verify(p, vk, pw), curve.String())
		}
	}
}
